"""CPU checks of mnn_ref.py: the bounds are tight enough to catch a lost split term and loose enough for the split itself,
`admissible` rejects hand-made wrong answers, and filter_tau places the filter-border rows where test_gpu_mnn_edges.py needs
them."""
import pytest
import torch
import torch.nn.functional as F

from tests import mnn_ref as mr


def sets(kind, n1=400, n2=300, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "unit":
        return F.normalize(torch.randn(n1, 64, generator=g), dim=-1), F.normalize(torch.randn(n2, 64, generator=g), dim=-1)
    if kind == "x13":
        return torch.randn(n1, 64, generator=g) * 13, torch.randn(n2, 64, generator=g) * 13
    base = F.normalize(torch.randn(n1, 64, generator=g), dim=-1)
    return base, F.normalize(base[:n2] + 1e-4 * torch.randn(n2, 64, generator=g), dim=-1)


@pytest.mark.parametrize("kind", ["unit", "x13", "near"])
@pytest.mark.parametrize("abs_bound", [0.0, 1.0])
def test_bound_against_split_terms(kind, abs_bound):
    """split_ref.check_bound's rule, entry by entry: the three-term emulation stays within B / 5 everywhere, and leaving out
    any one term exceeds 5 B somewhere."""
    f1, f2 = sets(kind)
    if abs_bound and kind == "x13":
        abs_bound = 64.0
    sl = mr.scale_log2_for(abs_bound if abs_bound else max(float(f1.abs().max()), float(f2.abs().max())))
    s64 = f1.double() @ f2.double().t()
    B = mr.bound(1, sl)(f1, f2)
    three = float(((mr.emulate(f1, f2, sl) - s64).abs() / B).max())
    assert three <= 0.2, f"three-term error {three:.3f} B"
    for t in mr.TERMS[1:]:
        drop = float(((mr.emulate(f1, f2, sl, [u for u in mr.TERMS if u != t]) - s64).abs() / B).max())
        assert drop >= 5, f"dropping {t}: only {drop:.2f} B"
    drop_hh = float(((mr.emulate(f1, f2, sl, mr.TERMS[1:]) - s64).abs() / B).max())
    assert drop_hh >= 5
    print(f"{kind} abs_bound={abs_bound}: three-term {three:.3f} B")


@pytest.mark.parametrize("kind", ["unit", "x13"])
def test_fp32_bound_against_sequential_sum(kind):
    """Implementation 0's bound clears an fp32 sequential sum (each product and addition rounded) by 5x."""
    f1, f2 = sets(kind, 200, 150)
    acc = torch.zeros(200, 150, dtype=torch.float32)
    for k in range(64):
        acc = acc + f1[:, k:k + 1] * f2[None, :, k]
    s64 = f1.double() @ f2.double().t()
    r = float(((acc.double() - s64).abs() / mr.bound(0)(f1, f2)).max())
    assert r <= 0.2, r


def test_scale_rule():
    assert mr.scale_log2_for(1.0) == 13 and mr.scale_log2_for(0.999) == 14 and mr.scale_log2_for(0.5) == 14
    assert mr.scale_log2_for(13.0) == 10 and mr.scale_log2_for(0.0) == 0
    hi, lo = mr.split(torch.tensor([[0.1, -0.0, 2.0 ** -30, 2.0 ** -40]]), 13)
    assert float(hi[0, 0]) + float(lo[0, 0]) == pytest.approx(0.1 * 8192, rel=2 ** -22)
    assert str(float(hi[0, 1])) == "-0.0" and str(float(lo[0, 1])) == "0.0"      # -0 - (-0) = +0
    assert float(hi[0, 2]) == 2.0 ** -17                                          # an fp16 subnormal
    assert float(hi[0, 3]) == 0.0 and float(lo[0, 3]) == 0.0                      # 2^-27: below half the smallest one


def dyadic(n1=300, n2=260, seed=3):
    g = torch.Generator().manual_seed(seed)
    f1 = torch.randint(-4, 5, (n1, 64), generator=g).float() / 8
    f2 = torch.randint(-4, 5, (n2, 64), generator=g).float() / 8
    f2[:150] = f1[:150]
    f2[200] = f2[10]                   # duplicate column: row 10's tie goes to column 10
    return f1, f2


def test_reference_tie_rule():
    f1, f2 = dyadic()
    i, j = mr.reference(f1, f2, -1)
    s = f1.double() @ f2.double().t()
    assert 10 in i.tolist() and j[i.tolist().index(10)] == 10
    for a, b in zip(i.tolist(), j.tolist()):
        assert s[a, b] == s[a].max() and int((s[a] == s[a].max()).nonzero()[0]) == b
        assert s[a, b] == s[:, b].max() and int((s[:, b] == s[:, b].max()).nonzero()[0]) == a


def test_admissible_rejects_wrong_answers():
    f1, f2 = dyadic()
    st = mr.Stats(f1, f2, mr.bound(1, 14))
    w0, w1 = st.mutual()
    assert mr.admissible(w0, w1, st, -1, exact=True) == 0.0
    assert mr.admissible(w0, w1, st, -1) == 0.0
    # a swapped pair
    b1 = w1.clone()
    b1[3], b1[4] = w1[4], w1[3]
    with pytest.raises(AssertionError):
        mr.admissible(w0, b1, st, -1)
    # the tie of row 10 resolved to the later duplicate column
    k = w0.tolist().index(10)
    b1 = w1.clone()
    b1[k] = 200
    with pytest.raises(AssertionError):
        mr.admissible(w0, b1, st, -1, exact=True)
    # the threshold compared with >=: a pair whose value equals min_cossim kept
    s = (f1[w0].double() * f2[w1].double()).sum(1)
    thr = float(s[5])
    keep = s >= thr
    with pytest.raises(AssertionError):
        mr.admissible(w0[keep], w1[keep], st, thr, exact=True)
    keep = s > thr
    mr.admissible(w0[keep], w1[keep], st, thr, exact=True)
    # an unambiguous pair above the cut dropped
    sure = (~st.row_amb[w0] & ~st.col_amb[w1]).nonzero()[:, 0]
    drop = int(sure[len(sure) // 2])
    keep = torch.ones(len(w0), dtype=torch.bool)
    keep[drop] = False
    with pytest.raises(AssertionError):
        mr.admissible(w0[keep], w1[keep], st, -1)
    # ... or a pair kept well below the cut
    thr = float(s.max()) + 1.0
    with pytest.raises(AssertionError):
        mr.admissible(w0[:1], w1[:1], st, thr)


def test_admissible_allows_near_ties_only():
    """On near-duplicate descriptors, a partner within B of the maximum is accepted and one beyond it is not."""
    f1, f2 = sets("near", 300, 300, seed=5)
    st = mr.Stats(f1, f2, mr.bound(1, 14))
    w0, w1 = st.mutual()
    mr.admissible(w0, w1, st, -1)
    s = f1.double() @ f2.double().t()
    # the row whose runner-up is farthest from its maximum: returning the runner-up is wrong
    top = s.topk(2, 1)
    gaps = top.values[:, 0] - top.values[:, 1]
    r = int(gaps.argmax())
    k = (w0 == r).nonzero()
    if len(k):
        b1 = w1.clone()
        b1[int(k[0, 0])] = int(top.indices[r, 1])
        with pytest.raises(AssertionError):
            mr.admissible(w0, b1, st, -1)


def test_filter_tau_border_rows():
    """filter_border_sets puts, in both directions, one row whose hi-only arg-max is wrong with a gap between 1.0x and 2.1x the
    Cauchy-Schwarz term (re-scored only because of the factor 2.1), one more inside tau and two outside it, where the hi-only
    arg-max is the exact one."""
    f1, f2, rows = mr.filter_border_sets()
    for d, (a, b) in enumerate(((f1, f2), (f2, f1))):
        gap, tau, arg = mr.filter_rows(a, b, mr.BORDER_SCALE_LOG2, a.shape[0], b.shape[0])
        _, tau1, _ = mr.filter_rows(a, b, mr.BORDER_SCALE_LOG2, a.shape[0], b.shape[0], k=1.0)
        s = a.double() @ b.double().t()
        (r0, e0, h0), (r1, _, h1), (r2, _, h2), (r3, _, h3) = rows[d]
        assert tau1[r0] < gap[r0] < tau[r0] and int(arg[r0]) == h0 and int(s[r0].argmax()) == e0 != h0
        assert gap[r1] < tau[r1] and int(s[r1].argmax()) == int(arg[r1]) == h1
        for r, h in ((r2, h2), (r3, h3)):
            assert tau[r] < gap[r] < 1.5 * tau[r] and int(s[r].argmax()) == int(arg[r]) == h
