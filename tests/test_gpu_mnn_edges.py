"""The MNN matchers against the float64 restatement of mnn_ref.py, through the C ABI, at the edges where they could go wrong:
every implementation (0-4) of xfeat_mnn_match_bounded and the presplit, pair-table and per-pair-scale entry points.

Every output is pre-filled with a sentinel; slots past each pair's count must keep it.  Random inputs are judged by
mnn_ref.admissible under the implementation's bound; dyadic inputs, where S is exact in every implementation, must give the
float64 lists bit for bit.  Each case prints its worst error-to-bound ratio (mnn_ref.admissible).
"""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from accelerated_features_b200 import _lib  # noqa: E402
from tests import mnn_ref as mr  # noqa: E402

SENT_I = -7
SENT_N = -999
SENT_K = -12345.5
PAD = 1e30            # finite, so that an fmaxf over a padding row would see it (a NaN would be skipped)
IMPLS = [0, 1, 2, 3, 4]
SPLIT_IMPLS = [1, 2, 3]
SIZES = [1, 2, 127, 128, 129, 255, 256, 257, 511, 512, 513, 4095, 4096, 4097]
WORST = {}


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat(device=0)


@pytest.fixture(scope="module")
def lib(xf):
    return xf._lib


@pytest.fixture(scope="module")
def real_desc(xf, assets_vga):
    """The asset pair's 4096 unit-norm descriptors per image."""
    ref, tgt = assets_vga
    out = xf.detectAndCompute(torch.from_numpy(np.stack([ref, tgt])).permute(0, 3, 1, 2).float() / 255, top_k=4096)
    return out[0]["descriptors"].contiguous(), out[1]["descriptors"].contiguous()


@contextlib.contextmanager
def mnn_impl(lib, impl):
    old = lib.xfeat_get_mnn_impl()
    lib.xfeat_set_mnn_impl(impl)
    try:
        yield
    finally:
        lib.xfeat_set_mnn_impl(old)


def note(impl, r):
    WORST[impl] = max(WORST.get(impl, 0.0), r)


def report(name):
    print(f"{name}: worst error/bound " + ", ".join(f"impl {k} {v:.3g}" for k, v in sorted(WORST.items())))


def dptr(t):
    return None if t is None else t.data_ptr()


def outputs(B, cap):
    return (torch.full((B, cap), SENT_I, dtype=torch.int64, device="cuda"),
            torch.full((B, cap), SENT_I, dtype=torch.int64, device="cuda"),
            torch.full((B,), SENT_N, dtype=torch.int32, device="cuda"))


def unpack(i0, i1, cnt):
    """[(idx0, idx1) or None for a negative count] per pair, after checking that slots past the count keep the sentinel."""
    torch.cuda.synchronize()
    i0, i1, cnt = i0.cpu(), i1.cpu(), cnt.cpu()
    res = []
    for b, c in enumerate(cnt.tolist()):
        assert c != SENT_N, f"pair {b}: count not written"
        k = max(c, 0)
        assert bool((i0[b, k:] == SENT_I).all()) and bool((i1[b, k:] == SENT_I).all()), f"pair {b}: write past its count {c}"
        res.append(None if c < 0 else (i0[b, :c], i1[b, :c]))
    return res, cnt


def bounded(lib, f1, n1, n1_max, stride1, f2, n2, n2_max, stride2, B, thr, abs_bound=0.0):
    """xfeat_mnn_match_bounded on flat fp32 device buffers; counts are host lists or None."""
    n1d = None if n1 is None else torch.tensor(n1, dtype=torch.int32, device="cuda")
    n2d = None if n2 is None else torch.tensor(n2, dtype=torch.int32, device="cuda")
    i0, i1, cnt = outputs(B, n1_max)
    ws = torch.empty(lib.xfeat_mnn_workspace_bytes(B, n1_max, n2_max), dtype=torch.uint8, device="cuda")
    _lib.check(lib.xfeat_mnn_match_bounded(f1.data_ptr(), dptr(n1d), n1_max, stride1, f2.data_ptr(), dptr(n2d), n2_max, stride2, B,
                                           float(thr), float(abs_bound), i0.data_ptr(), i1.data_ptr(), cnt.data_ptr(),
                                           ws.data_ptr(), ws.numel(), None), "xfeat_mnn_match_bounded")
    return unpack(i0, i1, cnt)


def presplit(lib, s1, n1, n1_max, s2, n2, n2_max, n_pad, B, sl, thr):
    n1d = None if n1 is None else torch.tensor(n1, dtype=torch.int32, device="cuda")
    n2d = None if n2 is None else torch.tensor(n2, dtype=torch.int32, device="cuda")
    i0, i1, cnt = outputs(B, n1_max)
    ws = torch.empty(lib.xfeat_mnn_presplit_workspace_bytes(B, n1_max, n2_max), dtype=torch.uint8, device="cuda")
    _lib.check(lib.xfeat_mnn_match_presplit(s1.data_ptr(), dptr(n1d), n1_max, s2.data_ptr(), dptr(n2d), n2_max, n_pad, B, sl,
                                            float(thr), i0.data_ptr(), i1.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(),
                                            None), "xfeat_mnn_match_presplit")
    return unpack(i0, i1, cnt)


def pairs_split(lib, table, n, n_max, pairs, sl, thr):
    nd = torch.tensor(n, dtype=torch.int32, device="cuda")
    tp = torch.tensor(pairs, dtype=torch.int32, device="cuda").reshape(-1, 2).contiguous()
    P = tp.shape[0]
    i0, i1, cnt = outputs(P, n_max)
    ws = torch.empty(lib.xfeat_mnn_pairs_workspace_bytes(P, n_max), dtype=torch.uint8, device="cuda")
    _lib.check(lib.xfeat_mnn_match_pairs(table.data_ptr(), nd.data_ptr(), table.shape[0], n_max, table.shape[1], tp.data_ptr(), P,
                                         sl, float(thr), i0.data_ptr(), i1.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(),
                                         None), "xfeat_mnn_match_pairs")
    return unpack(i0, i1, cnt), (tp, i0, i1, cnt)


def pairs_f32(lib, table, n, pairs):
    nd = torch.tensor(n, dtype=torch.int32, device="cuda")
    tp = torch.tensor(pairs, dtype=torch.int32, device="cuda").reshape(-1, 2).contiguous()
    P, n_max = tp.shape[0], table.shape[1]
    i0, i1, cnt = outputs(P, n_max)
    ws = torch.empty(lib.xfeat_mnn_pairs_f32_workspace_bytes(P, n_max), dtype=torch.uint8, device="cuda")
    _lib.check(lib.xfeat_mnn_match_pairs_f32(table.data_ptr(), nd.data_ptr(), table.shape[0], n_max, tp.data_ptr(), P,
                                             i0.data_ptr(), i1.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(), None),
               "xfeat_mnn_match_pairs_f32")
    return unpack(i0, i1, cnt), (tp, i0, i1, cnt)


def padded(sets, n_max, stride):
    """Flat buffer: set b's rows at b * stride, everything else (rows past the set, the stride gap) PAD."""
    buf = torch.full((len(sets) * stride + 64,), PAD, dtype=torch.float32, device="cuda")
    for b, s in enumerate(sets):
        buf[b * stride:b * stride + s.shape[0] * 64] = s.reshape(-1).to("cuda", torch.float32)
    return buf


def judge(impl, f1, f2, got, sl, thr, exact=False):
    st = mr.Stats(f1.cuda(), f2.cuda(), mr.bound(impl, sl))
    r = mr.admissible(got[0], got[1], st, thr, Bt=mr.thr_bound(impl, sl), exact=exact)
    note(impl, r)
    return r


def family(kind, n, g):
    if kind == "unit":
        return F.normalize(torch.randn(n, 64, generator=g), dim=-1)
    if kind == "x3":
        return torch.randn(n, 64, generator=g) * 3
    if kind == "x13":
        return torch.randn(n, 64, generator=g) * 13
    raise ValueError(kind)


def near_pair(n1, n2, g):
    """Set 2 holds perturbed copies of set 1's rows: every row's runner-up is within ~1e-4."""
    base = F.normalize(torch.randn(max(n1, n2), 64, generator=g), dim=-1)
    near = F.normalize(base + 1e-4 * torch.randn(base.shape, generator=g), dim=-1)
    return torch.cat([base, near])[torch.randperm(2 * len(base), generator=g)][:n1], near[:n2]


# ------------------------------------------------------------------------------------------------------------------ 1. shapes
@pytest.mark.parametrize("impl", IMPLS)
def test_shapes(lib, real_desc, impl):
    """n1 != n2 and n1_max != n2_max around every tile (128), slab (256) and padding (512) edge, four descriptor families, the
    measured scale and abs_bound = 1 on unit-norm sets.  Rows past each count are PAD."""
    g = torch.Generator().manual_seed(100 + impl)
    kinds = ["unit", "x3", "near", "x13", "real"]          # the asset descriptors land on n = 129 and 512
    with mnn_impl(lib, impl):
        for k, n1 in enumerate(SIZES):
            n2 = SIZES[(k + 5) % len(SIZES)]
            kind = kinds[k % len(kinds)]
            if kind == "near":
                f1, f2 = near_pair(n1, n2, g)
            elif kind == "real":
                f1, f2 = real_desc[0][:n1].cpu(), real_desc[1][:n2].cpu()
            else:
                f1, f2 = family(kind, n1, g), family(kind, n2, g)
            n1_max, n2_max = n1 + 3, n2 + 9
            b1, b2 = padded([f1], n1_max, n1_max * 64), padded([f2], n2_max, n2_max * 64)
            for ab in ((0.0, 1.0) if kind in ("unit", "near", "real") else (0.0,)):
                sl = mr.scale_log2_for(ab if ab else max(float(f1.abs().max()), float(f2.abs().max())))
                for thr in (-1, 0.5 if kind != "x13" else 40.0):
                    (got,), cnt = bounded(lib, b1, [n1], n1_max, n1_max * 64, b2, [n2], n2_max, n2_max * 64, 1, thr, ab)
                    judge(impl, f1, f2, got, sl, thr)
    report(f"shapes impl {impl}")


def test_shapes_32768(lib):
    g = torch.Generator(device="cuda").manual_seed(7)
    n1, n2 = 32768, 32761
    f1 = F.normalize(torch.randn(n1, 64, generator=g, device="cuda"), dim=-1)
    f2 = F.normalize(torch.randn(n2, 64, generator=g, device="cuda"), dim=-1)
    (got,), _ = bounded(lib, f1.reshape(-1).contiguous(), None, n1, n1 * 64, f2.reshape(-1).contiguous(), None, n2, n2 * 64, 1, -1)
    sl = mr.scale_log2_for(max(float(f1.abs().max()), float(f2.abs().max())))
    r = judge(lib.xfeat_get_mnn_impl(), f1, f2, got, sl, -1)
    print(f"32768 x 32761, default implementation: {len(got[0])} matches, worst error/bound {r:.3g}")


# ------------------------------------------------------------------------------------------------------- 2. strides, padding
@pytest.mark.parametrize("impl", IMPLS)
def test_strides_and_padding(lib, impl):
    """Per-pair strides beyond n_max * 64, and the gap plus the rows past each count filled with 1e30: neither the max-reduction
    nor the split may read them."""
    g = torch.Generator().manual_seed(200)
    n1_max, n2_max = 300, 260
    s1, s2 = (n1_max + 7) * 64, (n2_max + 5) * 64
    c1, c2 = [300, 17, 129], [260, 255, 1]
    A = [family("x3", c, g) for c in c1]
    Bs = [family("x3", c, g) for c in c2]
    sl = mr.scale_log2_for(max(max(float(a.abs().max()) for a in A), max(float(b.abs().max()) for b in Bs)))
    with mnn_impl(lib, impl):
        for thr in (-1, 10.0):
            res, _ = bounded(lib, padded(A, n1_max, s1), c1, n1_max, s1, padded(Bs, n2_max, s2), c2, n2_max, s2, 3, thr)
            for b in range(3):
                judge(impl, A[b], Bs[b], res[b], sl, thr)
    report(f"strides impl {impl}")


# ------------------------------------------------------------------------------------------------------------ 3. exact cases
def dyadic_sets():
    """Values k / 8 (|k| <= 4) and -2048.25 / 2^14: every product and sum is exact in fp32 and in the split (s = 2^14).
    Row 0 of set 1 is +0, row 200 is -0, row 0 of set 2 is all -2048.25 / 2^14 (hi -2048, lo -0.25): column 0 sees +-0 on rows 0
    and 200, below zero everywhere else, so the +-0 tie rule must give it row 0, and rows 0 / 200 see +-0 in every column.
    Duplicates: rows 5 = 133 = 261 = 517 of set 1 (tile, slab and row-block edges), columns 5 = 133 = 300 = 520 of set 2."""
    g = torch.Generator().manual_seed(300)
    n1, n2 = 700, 600
    f1 = torch.randint(-4, 5, (n1, 64), generator=g).float() / 8
    neg = f1.sum(1) <= 0
    f1[neg] = -f1[neg]
    f1[f1.sum(1) == 0, 0] = 0.5
    f2 = torch.randint(-4, 5, (n2, 64), generator=g).float() / 8
    for r in (133, 261, 517):
        f1[r] = f1[5]
    f2[:150] = f1[:150]
    for c in (300, 520):
        f2[c] = f2[5]
    f2[0] = -2048.25 / 16384
    f1[0] = 0.0
    f1[200] = -0.0
    return f1, f2


@pytest.mark.parametrize("impl", IMPLS)
def test_exact_bounded(lib, impl):
    f1, f2 = dyadic_sets()
    n1, n2 = f1.shape[0], f2.shape[0]
    w0, w1 = mr.reference(f1, f2, -1)
    assert w0[0] == 0 and w1[0] == 0 and 200 not in w0.tolist()
    i7, v = top_match(f1, f2)
    below = float(np.nextafter(np.float32(v), np.float32(-np.inf)))
    with mnn_impl(lib, impl):
        for ab in (0.0, 1.0):
            for thr in (-1, v, below):
                (got,), _ = bounded(lib, f1.reshape(-1).cuda(), None, n1, n1 * 64, f2.reshape(-1).cuda(), None, n2, n2 * 64, 1, thr,
                                    ab)
                judge(impl, f1, f2, got, 14, thr, exact=True)
                if thr == v:
                    assert i7 not in got[0].tolist()          # equal to min_cossim: rejected (strict >)
                if thr == below:
                    assert i7 in got[0].tolist()


def top_match(f1, f2):
    """(row, value) of the float64 mutual pair with the largest value."""
    w0, w1 = mr.reference(f1, f2, -1)
    vals = (f1[w0].double() * f2[w1].double()).sum(1)
    k = int(vals.argmax())
    assert float(vals[k]) > 0
    return int(w0[k]), float(vals[k])


def split_rows(f, n_pad, sl_build=13):
    """Host-built operand rows [hi | lo] of f * 2^sl_build, zero past len(f), as a (n_pad, 128) fp16 CUDA tensor."""
    hi, lo = mr.split(f, sl_build)
    out = torch.zeros(n_pad, 128, dtype=torch.float16)
    out[:len(f), :64], out[:len(f), 64:] = hi, lo
    return out.cuda()


@pytest.mark.parametrize("impl", SPLIT_IMPLS)
@pytest.mark.parametrize("sl", [0, 13, 20])
def test_exact_presplit_and_pairs(lib, impl, sl):
    """The same rows through xfeat_mnn_match_presplit and xfeat_mnn_match_pairs, declared at scale 2^sl: the matcher sees
    f * 2^(13 - sl), and min_cossim equal to a matched value of that must reject it, one fp32 ulp below must accept it."""
    f1, f2 = dyadic_sets()
    n1, n2 = f1.shape[0], f2.shape[0]
    e1, e2 = f1 * 2.0 ** (13 - sl), f2 * 2.0 ** (13 - sl)
    i7, v = top_match(e1, e2)
    below = float(np.nextafter(np.float32(v), np.float32(-np.inf)))
    r1, r2 = split_rows(f1, 1024), split_rows(f2, 1024)
    table = torch.stack([r1, r2])
    with mnn_impl(lib, impl):
        for thr in (-1, v, below):
            (got,), _ = presplit(lib, r1, [n1], n1, r2, [n2], n2, 1024, 1, sl, thr)
            judge(impl, e1, e2, got, sl, thr, exact=True)
            ((gp,), _), _ = pairs_split(lib, table, [n1, n2], max(n1, n2), [0, 1], sl, thr)
            assert torch.equal(gp[0], got[0]) and torch.equal(gp[1], got[1])
            assert (i7 in got[0].tolist()) == (thr != v)


# --------------------------------------------------------------------------------------------------------- 4. threshold band
@pytest.mark.parametrize("impl", IMPLS)
def test_threshold_band(lib, impl):
    """Thresholds at matched values +- small multiples of B: outside the band the decision is float64's."""
    g = torch.Generator().manual_seed(400)
    f1, f2 = near_pair(1000, 900, g)
    f1, f2 = f1.contiguous(), f2.contiguous()
    sl = mr.scale_log2_for(max(float(f1.abs().max()), float(f2.abs().max())))
    st = mr.Stats(f1.cuda(), f2.cuda(), mr.bound(impl, sl))
    w0, w1 = st.mutual()
    sure = (~st.row_amb[w0] & ~st.col_amb[w1]).nonzero()[:, 0]
    picks = sure[torch.linspace(0, len(sure) - 1, 4).long()]
    bt = mr.thr_bound(impl, sl)
    with mnn_impl(lib, impl):
        for p in picks.tolist():
            i, j = int(w0[p]), int(w1[p])
            sv = float(f1[i].double() @ f2[j].double())
            b = float(bt(f1[i:i + 1].cuda(), f2[j:j + 1].cuda())[0, 0])
            for m in (-3.0, -1.5, -0.5, 0.5, 1.5, 3.0):
                thr = sv + m * b
                (got,), _ = bounded(lib, f1.reshape(-1).cuda(), None, 1000, 0, f2.reshape(-1).cuda(), None, 900, 0, 1, thr)
                r = mr.admissible(got[0], got[1], st, thr, Bt=bt)
                note(impl, r)
                if abs(m) > 1:
                    assert (i in got[0].tolist()) == (m < 0), f"pair ({i}, {j}) at S {sv:.9g}, threshold S + {m} B"
    report(f"threshold band impl {impl}")


# ----------------------------------------------------------------------------------------------- 5. power-of-two invariance
@pytest.mark.parametrize("impl", IMPLS)
def test_power_of_two_invariance(lib, impl):
    g = torch.Generator().manual_seed(500)
    f1, f2 = F.normalize(torch.randn(3, 700, 64, generator=g), dim=-1), F.normalize(torch.randn(3, 650, 64, generator=g), dim=-1)
    c1, c2 = [700, 513, 129], [650, 257, 640]
    with mnn_impl(lib, impl):
        base = None
        for k in (0, -24, -10, 10, 24):
            a, b = (f1 * 2.0 ** k).reshape(-1).cuda(), (f2 * 2.0 ** k).reshape(-1).cuda()
            res, cnt = bounded(lib, a, c1, 700, 700 * 64, b, c2, 650, 650 * 64, 3, 0.3 * 4.0 ** k)
            if base is None:
                base = (res, cnt)
                for p in range(3):
                    sl = mr.scale_log2_for(max(mr.valid_absmax(f1, c1), mr.valid_absmax(f2, c2)))
                    judge(impl, f1[p, :c1[p]], f2[p, :c2[p]], res[p], sl, 0.3)
                continue
            assert torch.equal(cnt, base[1]), f"2^{k}: counts {cnt.tolist()} != {base[1].tolist()}"
            for p in range(3):
                assert torch.equal(res[p][0], base[0][p][0]) and torch.equal(res[p][1], base[0][p][1]), f"2^{k}, pair {p}"


# --------------------------------------------------------------------------------------------------- 6. mixed magnitudes
@pytest.mark.parametrize("impl", SPLIT_IMPLS)
def test_mixed_magnitudes(lib, impl):
    """Pairs at 2^12, 1, 2^-12 and 2^-20 in one batch: each admissible under the batch-wide scale of xfeat_mnn_match_bounded;
    xfeat_mnn_match_pairs_f32 on the same images equals single-pair calls and is admissible under each pair's own scale.  The
    images are near-duplicate sets, so that a change in the last bits of S moves some arg-maxes; under the batch-wide scale the
    2^-20 pair's operands are fp16 subnormals with a few bits each."""
    g = torch.Generator().manual_seed(600)
    n = 500
    mags = [2.0 ** 12, 1.0, 2.0 ** -12, 2.0 ** -20]
    imgs = []
    for m in mags:
        a, b = near_pair(n, n, g)
        imgs += [a * m, b * m]
    cnts = [500, 480, 333, 500, 129, 257, 500, 500]
    P = len(mags)
    A, Bs = [imgs[2 * p][:cnts[2 * p]] for p in range(P)], [imgs[2 * p + 1][:cnts[2 * p + 1]] for p in range(P)]
    batch_sl = mr.scale_log2_for(max(float(x.abs().max()) for x in A + Bs))
    table = torch.stack(imgs).cuda()
    with mnn_impl(lib, impl):
        res, _ = bounded(lib, padded(A, n, n * 64), cnts[0::2], n, n * 64, padded(Bs, n, n * 64), cnts[1::2], n, n * 64, P, -1)
        for p in range(P):
            judge(impl, A[p], Bs[p], res[p], batch_sl, -1)
        (pres, _), _ = pairs_f32(lib, table, cnts, list(range(2 * P)))
        for p in range(P):
            (single,), _ = bounded(lib, table[2 * p].reshape(-1), [cnts[2 * p]], n, n * 64, table[2 * p + 1].reshape(-1),
                                   [cnts[2 * p + 1]], n, n * 64, 1, -1)
            assert torch.equal(pres[p][0], single[0]) and torch.equal(pres[p][1], single[1]), f"pair {p}"
            own = mr.scale_log2_for(max(float(A[p].abs().max()), float(Bs[p].abs().max())))
            judge(impl, A[p], Bs[p], pres[p], own, -1)
    report(f"mixed magnitudes impl {impl}")


# ------------------------------------------------------------------------------------------------------------------ 7. counts
COUNT_CASES = {"none": None, "zero1": ([0, 1, 1, 1], None), "zero2": (None, [1, 0, 1, 1]), "zero12": ([1, 1, 0, 1], [1, 1, 0, 1]),
               "neg1": ([1, -1, 1, 1], None), "neg2": (None, [1, 1, -1, 1]), "above": ([5, 1, 1, 1], [1, 1, 1, 7])}


def count_lists(case, base1, base2, n_max):
    """Counts for a COUNT_CASES entry: 1 keeps the base count, 0 / -1 replace it, 5 / 7 put it above n_max."""
    if COUNT_CASES[case] is None:
        return None, None
    m1, m2 = COUNT_CASES[case]

    def app(m, base):
        if m is None:
            return list(base)
        return [b if k == 1 else (n_max + 40 if k in (5, 7) else k) for k, b in zip(m, base)]
    return app(m1, base1), app(m2, base2)


def clamp(c, n_max):
    return [min(x, n_max) for x in c]


def check_counts(res, cnt, ref_res, c1, c2):
    for p in range(len(res)):
        if c1[p] < 0 or c2[p] < 0:
            assert int(cnt[p]) == -1 and res[p] is None, f"pair {p}: an overflowed count must give -1"
            continue
        if c1[p] == 0 or c2[p] == 0:
            assert int(cnt[p]) == 0
            continue
        assert torch.equal(res[p][0], ref_res[p][0]) and torch.equal(res[p][1], ref_res[p][1]), f"pair {p} changed"


@pytest.mark.parametrize("impl", IMPLS)
def test_counts(lib, impl):
    """None, 0 on either or both sides, -1 on either side (that pair reports -1, the others are unchanged) and counts above
    n_max (clamped), through _bounded, and for the split implementations through _presplit, _pairs and _pairs_f32."""
    g = torch.Generator().manual_seed(700)
    n_max = 300
    A = [family("unit", n_max, g) for _ in range(4)]
    Bs = [family("unit", n_max, g) for _ in range(4)]
    base1, base2 = [300, 211, 129, 300], [300, 300, 77, 256]
    a, b = padded(A, n_max, n_max * 64), padded(Bs, n_max, n_max * 64)
    sl = mr.scale_log2_for(1.0)
    with mnn_impl(lib, impl):
        ref_res, _ = bounded(lib, a, base1, n_max, n_max * 64, b, base2, n_max, n_max * 64, 4, -1, 1.0)
        for p in range(4):
            judge(impl, A[p][:base1[p]], Bs[p][:base2[p]], ref_res[p], sl, -1)
        full, _ = bounded(lib, a, None, n_max, n_max * 64, b, None, n_max, n_max * 64, 4, -1, 1.0)
        for case in COUNT_CASES:
            c1, c2 = count_lists(case, base1, base2, n_max)
            if case == "none":
                res, cnt = bounded(lib, a, None, n_max, n_max * 64, b, None, n_max, n_max * 64, 4, -1, 1.0)
                for p in range(4):
                    judge(impl, A[p], Bs[p], res[p], sl, -1)
                continue
            res, cnt = bounded(lib, a, c1, n_max, n_max * 64, b, c2, n_max, n_max * 64, 4, -1, 1.0)
            want = [full[p] if (c1[p] >= n_max and c2[p] >= n_max) else ref_res[p] for p in range(4)]
            check_counts(res, cnt, want, c1, c2)
            if impl not in SPLIT_IMPLS:
                continue
            r1 = torch.stack([split_rows(x, 512) for x in A])
            r2 = torch.stack([split_rows(x, 512) for x in Bs])
            pres, pcnt = presplit(lib, r1, c1, n_max, r2, c2, n_max, 512, 4, 13, -1)
            assert torch.equal(pcnt, cnt)
            check_counts(pres, pcnt, res, clamp(c1, n_max), clamp(c2, n_max))
            table = torch.cat([r1, r2])
            (tres, tcnt), _ = pairs_split(lib, table, list(c1) + list(c2), n_max, [[p, 4 + p] for p in range(4)], 13, -1)
            assert torch.equal(tcnt, cnt)
            check_counts(tres, tcnt, res, clamp(c1, n_max), clamp(c2, n_max))
            ftab = torch.stack(A + Bs).cuda()
            (fres, fcnt), _ = pairs_f32(lib, ftab, list(c1) + list(c2), [[p, 4 + p] for p in range(4)])
            assert torch.equal(fcnt, cnt)
            for p in range(4):
                if fres[p] is not None and int(fcnt[p]) > 0:
                    own = mr.scale_log2_for(max(float(A[p][:min(c1[p], n_max)].abs().max()),
                                                float(Bs[p][:min(c2[p], n_max)].abs().max())))
                    judge(impl, A[p][:min(c1[p], n_max)], Bs[p][:min(c2[p], n_max)], fres[p], own, -1)
    report(f"counts impl {impl}")


# ----------------------------------------------------------------------------------------------------- 8. persistent schedule
@pytest.mark.parametrize("impl", IMPLS)
def test_persistent_batches(lib, impl):
    """Batches of SMs - 1, SMs, SMs + 1 and 2 SMs + 1 pairs with ragged counts, so that the persistent CTAs get unequal work."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(800)
    n_max = 300
    for B in (sms - 1, sms, sms + 1, 2 * sms + 1):
        f1 = F.normalize(torch.randn(B, n_max, 64, generator=g), dim=-1)
        f2 = F.normalize(torch.randn(B, n_max, 64, generator=g), dim=-1)
        c1 = [(37 * b) % n_max + 1 for b in range(B)]
        c2 = [n_max - (53 * b) % 280 for b in range(B)]
        with mnn_impl(lib, impl):
            res, _ = bounded(lib, f1.reshape(-1).cuda(), c1, n_max, n_max * 64, f2.reshape(-1).cuda(), c2, n_max, n_max * 64, B,
                             -1, 1.0)
        for p in range(B):
            judge(impl, f1[p, :c1[p]], f2[p, :c2[p]], res[p], 13, -1)
    report(f"persistent impl {impl}")


@pytest.mark.parametrize("impl", SPLIT_IMPLS)
def test_pair_tables(lib, impl):
    """Pair tables with repeated images, self-pairs (the identity on distinct rows) and images of different counts, through
    xfeat_mnn_match_pairs and xfeat_mnn_match_pairs_f32, and the matched keypoints through xfeat_gather_matches_pairs and
    xfeat_gather_matches, exactly."""
    g = torch.Generator().manual_seed(900)
    n_max, n_img = 400, 5
    imgs = [F.normalize(torch.randn(n_max, 64, generator=g), dim=-1) for _ in range(n_img)]
    cnts = [400, 129, 257, 1, 383]
    pairs = [[0, 0], [1, 1], [0, 2], [2, 0], [3, 1], [0, 2], [4, 4], [4, 2], [2, 4]]
    kp = torch.stack([torch.stack([torch.arange(n_max).float() + 0.25, torch.full((n_max,), i + 0.5)], 1) for i in range(n_img)])
    kp = kp.cuda().contiguous()
    table = torch.stack([split_rows(x[:c], 512) for x, c in zip(imgs, cnts)])
    ftab = torch.stack([torch.where(torch.arange(n_max)[:, None] < c, x, torch.full_like(x, PAD)) for x, c in zip(imgs, cnts)])
    with mnn_impl(lib, impl):
        (res, cnt), (tp, i0, i1, cd) = pairs_split(lib, table, cnts, n_max, pairs, 13, -1)
        (fres, fcnt), _ = pairs_f32(lib, ftab.cuda(), cnts, pairs)
    for p, (i, j) in enumerate(pairs):
        a, b = imgs[i][:cnts[i]], imgs[j][:cnts[j]]
        judge(impl, a, b, res[p], 13, -1)
        judge(impl, a, b, fres[p], mr.scale_log2_for(max(float(a.abs().max()), float(b.abs().max()))), -1)
        if i == j:
            assert torch.equal(res[p][0], torch.arange(cnts[i])) and torch.equal(res[p][1], torch.arange(cnts[i]))
            assert torch.equal(fres[p][0], res[p][0]) and torch.equal(fres[p][1], res[p][1])
    assert torch.equal(res[2][0], res[5][0]) and torch.equal(res[2][1], res[5][1])      # a repeated pair
    # keypoints of the pair table
    P = len(pairs)
    o0 = torch.full((P, n_max, 2), SENT_K, device="cuda")
    o1 = torch.full((P, n_max, 2), SENT_K, device="cuda")
    _lib.check(lib.xfeat_gather_matches_pairs(kp.data_ptr(), n_max, tp.data_ptr(), i0.data_ptr(), i1.data_ptr(), cd.data_ptr(), P,
                                              o0.data_ptr(), o1.data_ptr(), None), "xfeat_gather_matches_pairs")
    # ... and the per-pair form on the same matches, keypoints gathered per pair
    k0 = kp[tp[:, 0].long()].contiguous()
    k1 = kp[tp[:, 1].long()].contiguous()
    q0 = torch.full((P, n_max, 2), SENT_K, device="cuda")
    q1 = torch.full((P, n_max, 2), SENT_K, device="cuda")
    _lib.check(lib.xfeat_gather_matches(k0.data_ptr(), k1.data_ptr(), n_max, n_max, i0.data_ptr(), i1.data_ptr(), cd.data_ptr(), P,
                                        q0.data_ptr(), q1.data_ptr(), None), "xfeat_gather_matches")
    torch.cuda.synchronize()
    o0, o1, q0, q1, kpc = o0.cpu(), o1.cpu(), q0.cpu(), q1.cpu(), kp.cpu()
    for p, (i, j) in enumerate(pairs):
        c = len(res[p][0])
        for o, q, img, idx in ((o0, q0, i, res[p][0]), (o1, q1, j, res[p][1])):
            assert torch.equal(o[p, :c], kpc[img][idx]) and torch.equal(q[p, :c], kpc[img][idx])
            assert bool((o[p, c:] == SENT_K).all()) and bool((q[p, c:] == SENT_K).all())


# ----------------------------------------------------------------------------------------------- 9. implementation 4's filter
def test_filter_border(lib):
    """Rows on both sides of implementation 4's tau, in both directions (mnn_ref.filter_border_sets).  The host emulation shows
    that the filtered and the re-scored branch are both reached, and that one row per direction has a wrong hi-only arg-max
    whose gap is above 1.0x the Cauchy-Schwarz term; implementation 4 must equal implementation 1 bit for bit and give those
    rows their exact partner."""
    f1, f2, rows = mr.filter_border_sets()
    n1, n2 = f1.shape[0], f2.shape[0]
    for d, (a, b) in enumerate(((f1, f2), (f2, f1))):
        gap, tau, arg = mr.filter_rows(a, b, mr.BORDER_SCALE_LOG2, a.shape[0], b.shape[0])
        _, tau1, _ = mr.filter_rows(a, b, mr.BORDER_SCALE_LOG2, a.shape[0], b.shape[0], k=1.0)
        filt = gap > tau
        assert bool(filt.any()) and bool((~filt).any()), f"direction {d}: one branch of the filter is not reached"
        r0, e0, h0 = rows[d][0]
        assert tau1[r0] < gap[r0] <= tau[r0] and int(arg[r0]) == h0 != e0
    out = {}
    for impl in (1, 4):
        with mnn_impl(lib, impl):
            for ab in (1.0, 0.0):
                (got,), cnt = bounded(lib, f1.reshape(-1).cuda(), None, n1, 0, f2.reshape(-1).cuda(), None, n2, 0, 1, -1, ab)
                sl = mr.scale_log2_for(ab if ab else max(float(f1.abs().max()), float(f2.abs().max())))
                judge(impl, f1, f2, got, sl, -1)
                out[impl, ab] = got
        for ab in (1.0, 0.0):
            part = dict(zip(out[impl, ab][0].tolist(), out[impl, ab][1].tolist()))
            r0, e0, _ = rows[0][0]
            assert part.get(r0) == e0, f"impl {impl}: row {r0} matched {part.get(r0)}, exact partner {e0}"
            r0, e0, _ = rows[1][0]
            inv = {v: k for k, v in part.items()}
            assert inv.get(r0) == e0, f"impl {impl}: column {r0} matched {inv.get(r0)}, exact partner {e0}"
    for ab in (1.0, 0.0):
        assert torch.equal(out[1, ab][0], out[4, ab][0]) and torch.equal(out[1, ab][1], out[4, ab][1])
    report("filter border")
