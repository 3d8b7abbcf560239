"""xfeat_refine and xfeat_refine_pairs against the float64 restatement (refine_ref.py) at the edges of their index arithmetic:
unequal set sizes (n_max != n1_max) with B >= 3, clamped / zero / overflowed counts, ragged 128-row MLP tiles and 1024-row
compaction chunks, the strict confidence cut, and pair tables.  Each case runs under the tensor-core schedule (conv impl 2) and the
fp32 CUDA-core schedule (conv impl 0), with every output pre-filled with a sentinel.

The inputs make every output row identify the slot it read.  kpts0 of slot s is the centre of a 16-pixel grid cell, so the refined
(x0, y0), at most 4 / 0.6 pixels away, still names s; kpts1 of image j, slot t is (t + 0.5, j + 0.25).  The descriptors are rows of
the asset pair's real coarse features, drawn per image, so a wrong pair or stride changes the logits; most coarse matches are the
mutual nearest neighbours of the two images' rows, so many rows are confident.

Bounds (stated once, used everywhere):
- kept sets are exact except for rows whose float64 confidence is within refine_ref.conf_band of the threshold (the band that the
  logit tolerance FINE_MATCHER_TOL allows);
- (x1, y1) bit-exact; (x0, y0) within SUBPIX_TOL * scale0 + 2 u (|x0| + 4 scale0), the offset tolerance plus the fp32 rounding of
  x0 + dx * s (u = 2^-24);
- rows past n_refined keep the sentinel; a negative count is passed through to n_refined.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from accelerated_features_b200 import _lib  # noqa: E402
from oracle import xfeat_oracle as orc  # noqa: E402
from tests import refine_ref as rr  # noqa: E402
from tests import split_ref as sr  # noqa: E402

SENT = -12345.5
NSENT = -777
U32 = 2.0 ** -24
IMPLS = [2, 0]
WORST = {}            # worst coordinate error / bound per schedule, printed at the end of each test


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat(device=0)


@contextlib.contextmanager
def conv_impl(xf, impl):
    old = xf._lib.xfeat_get_conv_impl()
    xf._lib.xfeat_set_conv_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_conv_impl(old)


@pytest.fixture(scope="module")
def pool(oracle_state, assets_vga):
    """The asset pair's 60 x 80 coarse features (2, 4800, 64), un-normalised, on the GPU."""
    ref, tgt = assets_vga
    with torch.inference_mode():
        feats = orc.backbone(oracle_state, torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0))["feats"]
    return feats.permute(0, 2, 3, 1).reshape(2, -1, 64).contiguous().cuda()


def grid_kpts(n):
    s = torch.arange(n)
    return torch.stack([(s % 128).float() * 16 + 8, (s // 128).float() * 16 + 8], 1)


def slot_of(xy):
    return ((xy[:, 0] - 8) / 16).round().long() + 128 * ((xy[:, 1] - 8) / 16).round().long()


def kpts1_code(j, n):
    return torch.stack([torch.arange(n).float() + 0.5, torch.full((n,), j + 0.25)], 1)


def draw(src, n, g):
    """n rows of src (4800, 64): distinct while n <= 4800."""
    i = torch.randperm(len(src), generator=g)[:n] if n <= len(src) else torch.randint(0, len(src), (n,), generator=g)
    return src[i.cuda()]


def coarse_matches(d0, d1, n_max, n1_max, g):
    """(idx0, idx1) (n_max,): the mutual nearest neighbours of d0 / d1 and the other rows of d0 with random partners, merged in a
    random order that favours the mutual ones early; idx0 is a permutation of n_max."""
    s = d0 @ d1.t()
    m12, m21 = s.argmax(1), s.argmax(0)
    mut = (m21[m12] == torch.arange(n_max, device=s.device)).cpu()
    a = torch.nonzero(mut)[:, 0]
    b = m12.cpu()[a]
    rest = torch.nonzero(~mut)[:, 0]
    a_all = torch.cat([a, rest])
    b_all = torch.cat([b, torch.randint(0, n1_max, (len(rest),), generator=g)])
    key = torch.rand(n_max, generator=g) + torch.cat([torch.zeros(len(a)), torch.full((len(rest),), 0.6)])
    o = torch.argsort(key)
    return a_all[o], b_all[o]


def make_case(pool, B, n_max, n1_max, seed, desc0=None, desc1=None, scales0=None, gain=None):
    g = torch.Generator().manual_seed(seed)
    if desc0 is None:
        desc0 = torch.stack([draw(pool[0], n_max, g) for _ in range(B)])
        desc1 = torch.stack([draw(pool[1], n1_max, g) for _ in range(B)])
    if gain is not None:
        desc0, desc1 = desc0 * gain.view(-1, 1, 1).cuda(), desc1 * gain.view(-1, 1, 1).cuda()
    if scales0 is None:
        scales0 = torch.where(torch.rand(B, n_max, generator=g) < 0.3, 1 / 0.6, 1 / 1.3).float()
    idx = [coarse_matches(desc0[p], desc1[p], n_max, n1_max, g) for p in range(B)]
    # desc1 / kpts1 sit at the front of buffers of B * max(n_max, n1_max) rows: a stride of n_max instead of n1_max then reads
    # other valid rows (wrong values the checks see) rather than past the allocation
    rows = B * max(n_max, n1_max)
    d1 = torch.full((rows, 64), 0.5, device="cuda")
    d1[:B * n1_max] = desc1.reshape(-1, 64)
    k1 = torch.full((rows, 2), -99.0, device="cuda")
    k1[:B * n1_max] = torch.stack([kpts1_code(j, n1_max) for j in range(B)]).reshape(-1, 2).cuda()
    return dict(desc0=desc0.contiguous(), desc1=d1[:B * n1_max].view(B, n1_max, 64), d1buf=d1, k1buf=k1,
                kpts0=grid_kpts(n_max).expand(B, -1, -1).contiguous().cuda(),
                kpts1=k1[:B * n1_max].view(B, n1_max, 2), scales0=scales0.cuda().contiguous(),
                idx0=torch.stack([i for i, _ in idx]).cuda(), idx1=torch.stack([j for _, j in idx]).cuda(), n_max=n_max,
                n1_max=n1_max)


def run_refine(xf, c, counts, fine_conf, pairs=None):
    lib = xf._lib
    P, n_max = c["idx0"].shape
    cnt = torch.tensor(counts, dtype=torch.int32, device="cuda")
    out = torch.full((P, n_max, 4), SENT, device="cuda")
    n_ref = torch.full((P,), NSENT, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    if pairs is None:
        ws = torch.empty(lib.xfeat_refine_workspace_bytes(P, n_max), dtype=torch.uint8, device="cuda")
        rc = lib.xfeat_refine(xf._ctx, c["desc0"].data_ptr(), c["desc1"].data_ptr(), c["kpts0"].data_ptr(), c["kpts1"].data_ptr(),
                              c["scales0"].data_ptr(), c["idx0"].data_ptr(), c["idx1"].data_ptr(), cnt.data_ptr(), P, n_max,
                              c["n1_max"], float(fine_conf), out.data_ptr(), n_ref.data_ptr(), ws.data_ptr(), ws.numel(), st)
    else:
        tp = torch.tensor(pairs, dtype=torch.int32, device="cuda")
        ws = torch.empty(lib.xfeat_refine_pairs_workspace_bytes(P, n_max), dtype=torch.uint8, device="cuda")
        rc = lib.xfeat_refine_pairs(xf._ctx, c["desc0"].data_ptr(), c["kpts0"].data_ptr(), c["scales0"].data_ptr(), n_max,
                                    tp.data_ptr(), c["idx0"].data_ptr(), c["idx1"].data_ptr(), cnt.data_ptr(), P, float(fine_conf),
                                    out.data_ptr(), n_ref.data_ptr(), ws.data_ptr(), ws.numel(), st)
    _lib.check(rc, "refine")
    torch.cuda.synchronize()
    return out.cpu(), n_ref.cpu()


def reference(sd, c, counts, fine_conf, pairs=None):
    tp = None if pairs is None else torch.tensor(pairs)
    out = rr.refine_ref(sd, c["desc0"], c["desc1"], c["kpts0"], c["kpts1"], c["scales0"], c["idx0"], c["idx1"],
                        torch.tensor(counts), fine_conf, pairs=tp)
    return [{k: (v.cpu() if torch.is_tensor(v) else v) for k, v in o.items()} for o in out]


def check(name, c, ref, got, n_ref, counts, fine_conf, pairs=None, gain=None):
    """All assertions of one run; returns (rows kept, rows in the band, worst coordinate error / bound).  gain[p] scales pair p's
    logit and offset tolerances: inputs scaled by g scale the activations, and with them the fp32 accumulation error, by ~g."""
    P, n_max = c["idx0"].shape
    idx0 = c["idx0"].cpu()
    sc0 = c["scales0"].cpu()
    kept = unsure_n = 0
    worst = 0.0
    for p in range(P):
        tag = f"{name} pair {p}"
        if counts[p] < 0:
            assert int(n_ref[p]) == counts[p], f"{tag}: n_refined {int(n_ref[p])}, the count's status is {counts[p]}"
            assert bool((got[p] == SENT).all()), f"{tag}: an overflowed pair wrote rows"
            continue
        r = ref[p]
        n, k = r["n"], int(n_ref[p])
        assert 0 <= k <= n, f"{tag}: n_refined {k} outside [0, {n}]"
        assert bool((got[p, k:] == SENT).all()), f"{tag}: rows past n_refined = {k} were written"
        rows_out = got[p, :k]
        i = pairs[p][0] if pairs is not None else p
        inv = torch.full((n_max,), -1, dtype=torch.long)
        inv[idx0[p, :n]] = torch.arange(n)
        slot = slot_of(rows_out[:, :2])
        assert bool(((slot >= 0) & (slot < n_max)).all()), f"{tag}: a refined row names no slot"
        rows = inv[slot]
        assert bool((rows >= 0).all()), f"{tag}: a refined row is not one of the live coarse matches"
        assert bool((rows[1:] > rows[:-1]).all()), f"{tag}: refined rows out of coarse-row order"
        gp = 1.0 if gain is None else float(gain[p])
        band = (r["conf"] - fine_conf).abs() <= rr.conf_band(r["conf"], sr.FINE_MATCHER_TOL * gp)
        wrong = ~r["keep"][rows] & ~band[rows]
        assert not bool(wrong.any()), f"{tag}: {int(wrong.sum())} rows below the threshold kept (first {rows[wrong][:5].tolist()})"
        missing = r["keep"] & ~band
        missing[rows] = False
        assert not bool(missing.any()), f"{tag}: {int(missing.sum())} confident rows dropped (first {torch.nonzero(missing)[:5, 0].tolist()})"
        assert torch.equal(rows_out[:, 2:], r["xy1"][rows]), f"{tag}: (x1, y1) differ from kpts1[j, idx1]"
        s = sc0[i, idx0[p, rows]].double()[:, None]
        want = r["xy0"][rows]
        tol = sr.SUBPIX_TOL * gp * s + 2 * U32 * (want.abs() + 4 * s)
        err = (rows_out[:, :2].double() - want).abs()
        if k:
            worst = max(worst, float((err / tol).max()))
        assert bool((err <= tol).all()), f"{tag}: (x0, y0) off by {float(err.max()):.3e} px"
        kept += k
        unsure_n += int(band.sum())
    return kept, unsure_n, worst


def run_and_check(xf, sd, name, c, counts, fine_conf, impl, pairs=None, ref=None, gain=None):
    if ref is None:
        ref = reference(sd, c, counts, fine_conf, pairs)
    with conv_impl(xf, impl):
        got, n_ref = run_refine(xf, c, counts, fine_conf, pairs)
    kept, unsure, worst = check(f"{name} impl {impl} thr {fine_conf:.4g}", c, ref, got, n_ref, counts, fine_conf, pairs, gain)
    WORST[impl] = max(WORST.get(impl, 0.0), worst)
    live = sum(o["n"] for o in ref)
    print(f"{name} impl {impl} thr {fine_conf:.4g}: {live} live rows, {kept} refined, {unsure} in the band, worst coordinate "
          f"error / bound {worst:.3f} (worst so far under impl {impl}: {WORST[impl]:.3f})")
    return n_ref


UNEQUAL = [("n_max>n1_max", 4, 700, 300, [700, 650, 0, 333]),
           ("n_max<n1_max", 4, 300, 700, [300, 1, 250, 299]),
           ("n1_max=1", 3, 200, 1, [200, 150, 37])]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", UNEQUAL, ids=lambda c: c[0])
def test_unequal_set_sizes(xf, oracle_state, pool, case, impl):
    name, B, n_max, n1_max, counts = case
    c = make_case(pool, B, n_max, n1_max, seed=n_max * 7 + n1_max)
    run_and_check(xf, oracle_state, name, c, counts, 0.25, impl)


@pytest.fixture(scope="module")
def dualscale(xf, assets_vga):
    """Real dual-scale tables of a VGA set and a 1280 x 960 set (top_k 10000: 9728 and 10000 rows)."""
    ref, tgt = assets_vga
    vga = torch.cat([orc.parse_input(ref), orc.parse_input(tgt), orc.parse_input(ref)], 0)
    big = F.interpolate(torch.cat([orc.parse_input(tgt), orc.parse_input(ref), orc.parse_input(tgt)], 0), size=(960, 1280),
                        mode="bilinear", align_corners=False)
    out = []
    for x in (vga, big):
        mk, sc, ft = xf.extract_dualscale(x.cuda(), 10000)
        torch.cuda.synchronize()
        out.append((ft.contiguous(), sc.contiguous()))
    assert out[0][0].shape[1] != out[1][0].shape[1]
    return out


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("order", ["vga_vs_1280", "1280_vs_vga"])
def test_dualscale_row_counts(xf, oracle_state, dualscale, order, impl):
    (f0, s0), (f1, _) = dualscale if order == "vga_vs_1280" else dualscale[::-1]
    n_max, n1_max = f0.shape[1], f1.shape[1]
    c = make_case(None, 3, n_max, n1_max, seed=5, desc0=f0, desc1=f1, scales0=s0.cpu())
    counts = [n_max, n_max // 3, 2000]
    run_and_check(xf, oracle_state, order, c, counts, 0.25, impl)


@pytest.mark.parametrize("impl", IMPLS)
def test_counts(xf, oracle_state, pool, impl):
    """0, 1, n_max, n_max + 5 (clamped) and XF_N_OVERFLOW next to ordinary pairs."""
    n_max, n1_max = 300, 257
    counts = [0, 1, n_max, n_max + 5, _lib.N_OVERFLOW, 150, _lib.N_OVERFLOW, 299]
    c = make_case(pool, len(counts), n_max, n1_max, seed=31)
    n_ref = run_and_check(xf, oracle_state, "counts", c, counts, 0.25, impl)
    assert int(n_ref[0]) == 0 and int(n_ref[4]) == int(n_ref[6]) == _lib.N_OVERFLOW


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("counts", [[0, 1, 0], [60, 0, 67], [64, 64, 0], [43, 43, 43]], ids=["rows1", "rows127", "rows128", "rows129"])
def test_tile_edges(xf, oracle_state, pool, counts, impl):
    """Total live rows 1, 127, 128, 129 around the MLP's 128-row tile; fine_conf -1 keeps every row."""
    c = make_case(pool, 3, 100, 90, seed=sum(counts))
    run_and_check(xf, oracle_state, f"rows{sum(counts)}", c, counts, 0.25, impl)
    n_ref = run_and_check(xf, oracle_state, f"rows{sum(counts)}", c, counts, -1.0, impl)
    assert n_ref.tolist() == counts


@pytest.mark.parametrize("impl", IMPLS)
def test_chunk_edges(xf, oracle_state, pool, impl):
    """Per-pair counts 1023, 1024, 1025 and 2049 at n_max = 2049, across the compaction's 1024-row chunks."""
    counts = [1023, 1024, 1025, 2049]
    c = make_case(pool, 4, 2049, 1800, seed=77)
    run_and_check(xf, oracle_state, "chunks", c, counts, 0.25, impl)
    n_ref = run_and_check(xf, oracle_state, "chunks", c, counts, 0.0, impl)
    assert n_ref.tolist() == counts


@pytest.mark.parametrize("impl", IMPLS)
def test_confidence_cut(xf, oracle_state, pool, impl):
    """fine_conf <= 0 keeps every live row in order (conf >= 1/64); fine_conf = 1 keeps none, although pair 2 (descriptors x 64)
    has rows whose fp32 confidence is exactly 1 (strict >); thresholds at quantiles of the float64 confidences."""
    counts = [600, 517, 400]
    gain = torch.tensor([1.0, 1.0, 64.0])
    c = make_case(pool, 3, 600, 500, seed=13, gain=gain)
    ref = reference(oracle_state, c, counts, 0.25)
    conf = torch.cat([o["conf"] for o in ref])
    sure1 = int((1 - conf < U32 / 4).sum())
    assert sure1 > 0, "no row has a confidence of 1 in fp32: the fine_conf = 1 case would not test the strict >"
    qs = [float(q) for q in torch.quantile(torch.cat([o["conf"] for o in ref[:2]]), torch.tensor([0.1, 0.5, 0.9], dtype=torch.float64))]
    print(f"confidence quantiles {[f'{q:.4f}' for q in qs]}, {sure1} rows at conf 1")
    for thr in [-1.0, 0.0] + qs + [1.0]:
        r = [dict(o, keep=o["conf"] > thr, rows=torch.nonzero(o["conf"] > thr)[:, 0]) for o in ref]
        n_ref = run_and_check(xf, oracle_state, "cut", c, counts, thr, impl, ref=r, gain=gain)
        if thr <= 0:
            assert n_ref.tolist() == counts
        if thr == 1.0:
            assert n_ref.tolist() == [0, 0, 0]


@pytest.mark.parametrize("impl", IMPLS)
def test_pairs_vs_float64(xf, oracle_state, pool, impl):
    """xfeat_refine_pairs on a 5-image table against float64 directly: repeated pairs, (i, i), reversed pairs, the last slot, more
    pairs than images, and both star scales (1 / 0.6 and 1 / 1.3) in each image's rows."""
    n_img, n_max = 5, 900
    g = torch.Generator().manual_seed(41)
    table = torch.stack([draw(pool[i % 2], n_max, g) for i in range(n_img)]).contiguous()
    split = [180, 250, 300, 120, 600]
    scales = torch.stack([torch.cat([torch.full((k,), 1 / 0.6), torch.full((n_max - k,), 1 / 1.3)]) for k in split]).float()
    pairs = [(0, 1), (1, 0), (0, 1), (2, 2), (4, 3), (3, 4), (4, 4), (1, 4), (0, 3), (4, 0)]
    idx = [coarse_matches(table[i], table[j], n_max, n_max, g) for i, j in pairs]
    # one keypoint table serves both sides: the grid cell names the slot, a fraction j * 2^-6 the image
    kp = torch.stack([grid_kpts(n_max) + j * 2.0 ** -6 for j in range(n_img)])
    c = dict(desc0=table, desc1=table, kpts0=kp.cuda().contiguous(), kpts1=kp.cuda().contiguous(), scales0=scales.cuda(),
             idx0=torch.stack([i for i, _ in idx]).cuda(), idx1=torch.stack([j for _, j in idx]).cuda(), n_max=n_max, n1_max=n_max)
    counts = [n_max, 700, 333, n_max, 512, 1, 0, n_max + 5, 640, 129]
    run_and_check(xf, oracle_state, "pairs", c, counts, 0.25, impl, pairs=pairs)
