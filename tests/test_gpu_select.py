"""Keypoint selection (csrc/sparse.cu, csrc/dense.cu) against the exact host reference of tests/select_ref.py.

xfeat_detect_sparse_split and xfeat_detect_dense are called through the C-ABI with synthetic heat, reliability and feature
maps built on the host from seeded generators, every output pre-filled with a sentinel.  Selection is a chain of integer
decisions, so everything but the descriptors must match exactly: n_cand, n_valid, the keypoints and their order, the bits of
the scores, the zero slots past n_valid and the keypoint rescale.  The descriptors are held to a float64 bound derived below,
and the split operand rows to the exact fp16 split of the descriptors.

The inputs are built to reach the edges of every selection path: exact score ties at the top-k cut (so the radix select has to
decide on the pixel word of the key), more than NM_LIST = 1024 NMS maxima in one march CTA (direct emission), maxima at the
threshold and at the border, partial strips, the sorted sampler's Hm = 512 limit and the B = 32 / top_k = 8192 dispatch edges,
the cub paths, and constant, quantised and signed-zero reliability maps for the dense top-k.  A child process repeats a subset
with the diagnostic switches XFEAT_NMS_TILED, XFEAT_TOPK_CUB and XFEAT_SAMPLE_GENERIC set and must produce the same bits.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import select_ref as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
SENT = -7777.0          # output sentinel (float and int)
SENT_H = -777.0         # split-operand sentinel (fp16)
SWITCHES = ("XFEAT_NMS_TILED", "XFEAT_TOPK_CUB", "XFEAT_SAMPLE_GENERIC")

# Descriptor bound against float64, per element c of the unit descriptor n of one keypoint:
#   |n32_c - n64_c| <= EPS * (T_c + |n_c| * ||T||) / ||o|| + 8u |n_c|,
# o = the un-normalised bicubic sample, T_c = sum over the 16 taps of |f_c| / ||f|| (descriptors_f64).  The kernels' error in o_c:
#   den = 1 / max(||f||, 1e-12): 64 squares summed 8 per lane then over 3 shuffles (<= 11u), sqrt (+5.5u + u), 1/x (+u): 8u;
#   v * den: u;  the cubic weights (|w| <= 1) from the fp32 tx in fp32: <= 8u absolute each, 16u for the product cx * cy;
#   the two 4-term fma chains: <= 8u of the sum of |terms| <= T_c.  Total <= 33u of T_c; EPS = 40u.
# The normalisation: ss from 4 fma and 4 shuffle sums (8u), sqrt and 1/x (6u), the product (u), so n32 = o32 (1 + <= 8u) /
# ||o32||, and | ||o32|| - ||o|| | <= ||o32 - o|| <= EPS ||T||.  The bound is checked per element; WORST records the largest
# error and ratio seen.  Measured on an H100 over all the cases here: 4.5e-7 at most, 0.14 of the bound.
EPS = 40 * U
DESC_CAP = 2e-6         # and no element may be further than this from float64 (the previous check allowed 2e-5)
WORST = {"err": 0.0, "ratio": 0.0}


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# input builders (host, seeded)
def peaks(rng, H, W, n, levels=None):
    """n isolated maxima (3 px apart) at grid points where the float32 bilinear factor of a constant 1.0 reliability map is
    exactly 1.0, values k/16 assigned cyclically over `levels` levels: every level holds several keys with exactly the same
    score, so ties straddle any cut."""
    heat = np.zeros((H, W), np.float32)
    gy, gx = (a.reshape(-1) for a in np.meshgrid(np.arange(1, H - 2, 3), np.arange(1, W - 2, 3), indexing="ij"))
    unit = ref.scores_f32(np.ones((H, W), np.float32), np.ones((H // 8, W // 8), np.float32), gx, gy) == 1.0
    gx, gy = gx[unit], gy[unit]
    assert len(gx) >= n
    pick = rng.permutation(len(gx))[:n]
    if levels is None:
        levels = max(1, min(15, n // 4))
    vals = (1 + np.arange(n) % levels).astype(np.float32) / np.float32(16)
    heat[gy[pick], gx[pick]] = vals[rng.permutation(n)]
    return heat


def quantised(rng, H, W):
    """i.i.d. heat quantised to k/16: plateaus and ties everywhere, ~7 % of the pixels are maxima."""
    return (rng.integers(0, 16, (H, W)).astype(np.float32) / np.float32(16))


def noise(rng, H, W, scale=0.3):
    return rng.random((H, W), dtype=np.float32) * np.float32(scale)


def feats_for(rng, B, H, W):
    return rng.standard_normal((B, H // 8, W // 8, 64), dtype=np.float32)


def case_ties(top_k):
    """Case 1: counts top_k - 1, top_k, top_k + 1 of isolated quantised maxima, and quantised noise with far more."""
    def build():
        H = W = 320 if top_k <= 513 else 640
        rng = np.random.default_rng(1000 + top_k)
        heat = np.stack([peaks(rng, H, W, max(0, n)) for n in (top_k - 1, top_k, top_k + 1)] + [quantised(rng, H, W)])
        rel = np.ones((4, H // 8, W // 8), np.float32)
        return dict(heat=heat, rel=rel, feats=feats_for(rng, 4, H, W), top_k=top_k, thr=0.05, ties=True)
    return build


def case_overflow_list(kind):
    """Case 2: more than NM_LIST maxima in one 128 x 64 march CTA (x in [128, 256), y in [64, 128)), below the image
    capacity, so the directly emitted survivors must be in the output (top_k >= their count)."""
    def build():
        H = W = 512
        rng = np.random.default_rng(2000 + ("1024", "1025", "full_cta", "straddle").index(kind))
        h0 = np.zeros((H, W), np.float32)
        if kind in ("1024", "1025"):
            h0[74:106, 148:180] = 0.5                 # 32 x 32 = 1024 equal maxima
            if kind == "1025":
                h0[74, 180] = 0.5
        elif kind == "full_cta":
            h0[64:128, 128:256] = 0.5                 # 8192 maxima in one CTA
        else:
            h0[32:96, 64:192] = 0.5                   # 8192 maxima across four CTAs, 2048 in each
        heat = np.stack([h0, quantised(rng, H, W)])
        rel = np.stack([np.ones((H // 8, W // 8), np.float32), rng.random((H // 8, W // 8), dtype=np.float32)])
        expect = {"1024": 1024, "1025": 1025}.get(kind, 8192)
        return dict(heat=heat, rel=rel, feats=feats_for(rng, 2, H, W), top_k=8192, thr=0.05, n_cand0=expect)
    return build


def case_threshold(kind):
    """Case 3, B = 32 (sorted sampler, whose bicubic4<true> takes the border path warp-wide): maxima exactly at and one ulp
    above the threshold, negative heat, and maxima on the first and last three rows and columns mixed with interior ones."""
    def build():
        B, H, W = 32, 128, 160
        rng = np.random.default_rng(3000 + ("ulp", "negative", "negative_thr", "border").index(kind))
        heat = np.empty((B, H, W), np.float32)
        thr = {"ulp": 0.25, "negative": 0.0, "negative_thr": -0.5, "border": 0.05}[kind]
        for b in range(B):
            if kind == "ulp":
                h = noise(rng, H, W, 0.2)
                t = np.float32(thr)
                for i, (y, x) in enumerate(zip(rng.integers(3, H - 3, 60), rng.integers(3, W - 3, 60))):
                    h[y - 2:y + 3, x - 2:x + 3] = np.minimum(h[y - 2:y + 3, x - 2:x + 3], np.float32(0.2))
                    h[y, x] = t if i % 2 == 0 else np.nextafter(t, np.float32(1))
            elif kind.startswith("negative"):
                h = -noise(rng, H, W, 1.0) + (np.float32(0.3) if b % 2 else np.float32(0.0))
            else:
                h = noise(rng, H, W, 0.04)
                band = quantised(rng, H, W)
                m = np.zeros((H, W), bool)
                m[:3] = m[-3:] = True
                m[:, :3] = m[:, -3:] = True
                h[m] = band[m]
                h[40:90:3, 40:120:3] = band[40:90:3, 40:120:3]
            heat[b] = h
        rel = rng.random((B, H // 8, W // 8), dtype=np.float32) + np.float32(0.05)
        return dict(heat=heat, rel=rel, feats=feats_for(rng, B, H, W), top_k=1024, thr=thr)
    return build


def case_geometry(H, W, B, top_k):
    """Case 4: partial strips (W % 128 != 0), H % 64 != 0, tiny images, the sorted sampler at Hm = 512 (one strip per
    feature row) and at Hm = 256 (two strips), and Hm = 516, which takes the generic sampler."""
    def build():
        rng = np.random.default_rng(4000 + H + W + B)
        heat = np.stack([noise(rng, H, W) for _ in range(B)])
        rel = rng.random((B, H // 8, W // 8), dtype=np.float32)
        return dict(heat=heat, rel=rel, feats=feats_for(rng, B, H, W), top_k=top_k, thr=0.05, rw=1.25, rh=0.75)
    return build


def case_batch(B, top_k, H=128, W=192, sub=None):
    """Case 5: batch and dispatch edges.  Image 0 is empty, image 1 overflows the H*W/4 capacity (XF_N_OVERFLOW, its
    neighbours unaffected), the rest are quantised noise; `sub` re-runs the batch in sub-batches and requires the same bits."""
    def build():
        rng = np.random.default_rng(5000 + B + top_k)
        heat = np.stack([quantised(rng, H, W) for _ in range(B)])
        if B > 2:
            heat[0] = 0.0
            heat[1] = 0.5
        rel = rng.random((B, H // 8, W // 8), dtype=np.float32) + np.float32(0.05)
        return dict(heat=heat, rel=rel, feats=feats_for(rng, B, H, W), top_k=top_k, thr=0.05, sub=sub)
    return build


def case_capacity():
    """Case 5: top_k larger than the capacity of a small image; a plateau of exactly the capacity (1024 maxima at 64 x 64,
    accepted) and one of capacity + 1 (overflow)."""
    def build():
        rng = np.random.default_rng(5999)
        H = W = 64
        heat = np.stack([quantised(rng, H, W), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32)])
        heat[1, 10:42, 10:42] = 0.5
        heat[2, 10:42, 10:42] = 0.5
        heat[2, 10, 42] = 0.5
        rel = np.full((3, H // 8, W // 8), 0.75, np.float32)
        return dict(heat=heat, rel=rel, feats=feats_for(rng, 3, H, W), top_k=2000, thr=0.05, n_valid=[None, 1024, -1])
    return build


SPARSE_CASES = {
    **{f"ties_k{k}": case_ties(k) for k in (1, 2, 511, 512, 513, 4096, 8191, 8192)},
    **{f"nms_list_{k}": case_overflow_list(k) for k in ("1024", "1025", "full_cta", "straddle")},
    **{f"thr_{k}": case_threshold(k) for k in ("ulp", "negative", "negative_thr", "border")},
    "geom_96x160": case_geometry(96, 160, 3, 512),
    "geom_64x416": case_geometry(64, 416, 2, 1000),
    "geom_32x256": case_geometry(32, 256, 2, 300),
    "geom_480x320": case_geometry(480, 320, 2, 2048),
    "geom_32x32": case_geometry(32, 32, 2, 64),
    "geom_4096x256_sorted_hm512": case_geometry(4096, 256, 32, 4096),
    "geom_4128x256_generic_hm516": case_geometry(4128, 256, 32, 4096),
    "geom_2048x2048_sorted_2strips": case_geometry(2048, 2048, 32, 4096),
    "batch_b1": case_batch(1, 1000),
    "batch_b31": case_batch(31, 1000),
    "batch_b32": case_batch(32, 1000, sub=[31, 1]),
    "batch_b33": case_batch(33, 1000, sub=[16, 17]),
    "batch_b32_k8192": case_batch(32, 8192, H=512, W=512, sub=[16, 16]),
    "batch_b2_k8193_cub": case_batch(2, 8193, H=512, W=512),
    "batch_b33_k20000_cub": case_batch(33, 20000, H=640, W=640),
    "capacity_topk_above_cap": case_capacity(),
}


# ---------------------------------------------------------------------------------------------------------------------
def run_sparse(xf, heat, rel, feats, top_k, thr, rw=1.0, rh=1.0, split_rows=None):
    """One xfeat_detect_sparse_split call on host arrays; every output starts as a sentinel.  Returns numpy arrays."""
    from accelerated_features_b200 import _lib
    B, H, W = heat.shape
    if split_rows is None:
        split_rows = -(-top_k // 512) * 512 + 512    # one block of padding rows past top_k
    d_heat, d_rel, d_feats = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (heat, rel, feats))
    kpts = torch.full((B, top_k, 2), SENT, device="cuda")
    scores = torch.full((B, top_k), SENT, device="cuda")
    desc = torch.full((B, top_k, 64), SENT, device="cuda")
    nv = torch.full((B,), int(SENT), dtype=torch.int32, device="cuda")
    nc = torch.full((B,), int(SENT), dtype=torch.int32, device="cuda")
    ki = torch.full((B, top_k, 2), int(SENT), dtype=torch.int32, device="cuda")
    split = torch.full((B, split_rows, 128), SENT_H, dtype=torch.float16, device="cuda")
    ws = torch.empty(xf._lib.xfeat_sparse_workspace_bytes(B, H, W, top_k), dtype=torch.uint8, device="cuda")
    _lib.check(xf._lib.xfeat_detect_sparse_split(
        xf._ctx, d_feats.data_ptr(), d_heat.data_ptr(), d_rel.data_ptr(), B, H, W, top_k, float(thr), float(rw), float(rh),
        kpts.data_ptr(), scores.data_ptr(), desc.data_ptr(), nv.data_ptr(), nc.data_ptr(), ki.data_ptr(), split.data_ptr(),
        split_rows, ws.data_ptr(), ws.numel(), _stream()), "detect_sparse_split")
    torch.cuda.synchronize()
    return dict(kpts=kpts.cpu().numpy(), scores=scores.cpu().numpy(), desc=desc.cpu().numpy(), n_valid=nv.cpu().numpy(),
                n_cand=nc.cpu().numpy(), kpts_int=ki.cpu().numpy(), split=split.cpu().numpy())


def run_case(xf, c, heat=None):
    heat = c["heat"] if heat is None else heat
    return run_sparse(xf, heat, c["rel"], c["feats"], c["top_k"], c["thr"], c.get("rw", 1.0), c.get("rh", 1.0))


def bits(a):
    return np.ascontiguousarray(a).view(np.int32 if a.dtype.itemsize == 4 else np.int16)


def check_descriptors(feats, x, y, H, W, got):
    want, T, norm = ref.descriptors_f64(feats, x, y, H, W)
    err = np.abs(got.astype(np.float64) - want)
    bound = EPS * (T + np.abs(want) * np.linalg.norm(T, axis=1, keepdims=True)) / norm[:, None] + 8 * U * np.abs(want)
    bound = bound * 1.01 + 1e-12   # second-order terms of the first-order derivation
    assert (err <= bound).all(), f"descriptor outside its float64 bound: {int((err > bound).sum())} elements"
    if len(err):
        WORST["err"] = max(WORST["err"], float(err.max()))
        WORST["ratio"] = max(WORST["ratio"], float((err / bound).max()))
        assert err.max() <= DESC_CAP, err.max()


def check_sparse(c, out):
    """Every output of every image against select_ref."""
    heat, rel, feats, top_k, thr = c["heat"], c["rel"], c["feats"], c["top_k"], c["thr"]
    rw, rh = np.float32(c.get("rw", 1.0)), np.float32(c.get("rh", 1.0))
    B, H, W = heat.shape
    split_rows = out["split"].shape[1]
    for b in range(B):
        sel = ref.sparse_select(heat[b], rel[b], thr, top_k)
        nv = int(out["n_valid"][b])
        assert int(out["n_cand"][b]) == sel["n_cand"], (b, int(out["n_cand"][b]), sel["n_cand"])
        assert nv == sel["n_valid"], (b, nv, sel["n_valid"])
        n = max(nv, 0)
        if c.get("ties") and n >= 2:     # the case really exercises ties, at the cut whenever the select runs
            cut = sel["score"][-1]
            if sel["n_keep"] > top_k:
                assert (sel["all_scores"] == cut).sum() > (sel["score"] == cut).sum(), "no tie straddles the cut"
            else:
                assert len(np.unique(sel["score"])) < n
        assert np.array_equal(out["kpts_int"][b, :n, 0], sel["x"]) and np.array_equal(out["kpts_int"][b, :n, 1], sel["y"]), b
        assert np.array_equal(bits(out["scores"][b, :n]), bits(sel["score"])), b
        want_kp = np.stack([sel["x"].astype(np.float32) * rw, sel["y"].astype(np.float32) * rh], -1)
        assert np.array_equal(bits(out["kpts"][b, :n]), bits(want_kp.reshape(-1, 2))), b
        for k in ("kpts", "scores", "desc", "kpts_int"):        # slots past n_valid (all of an overflowed image) are zero
            assert not out[k][b, n:].any(), (b, k)
        assert not out["split"][b, n:].any(), b                 # operand rows past n_valid, up to split_rows
        d = out["desc"][b, :n]
        check_descriptors(feats[b], sel["x"], sel["y"], H, W, d)
        hi, lo = ref.split_f16(d)
        assert np.array_equal(bits(out["split"][b, :n, :64]), bits(hi)) and np.array_equal(bits(out["split"][b, :n, 64:]), bits(lo)), b
    assert split_rows > top_k


@pytest.mark.parametrize("name", list(SPARSE_CASES))
def test_sparse_selection(xf, name):
    c = SPARSE_CASES[name]()
    out = run_case(xf, c)
    check_sparse(c, out)
    if "n_cand0" in c:
        assert int(out["n_cand"][0]) == c["n_cand0"] and int(out["n_valid"][0]) == c["n_cand0"]
    for b, w in enumerate(c.get("n_valid", [])):
        assert w is None or int(out["n_valid"][b]) == w, (b, int(out["n_valid"][b]), w)
    if c.get("sub"):   # the same images in sub-batches (other sampler / other batch position): the same bits
        lo = 0
        for nb in c["sub"]:
            part = run_sparse(xf, c["heat"][lo:lo + nb], c["rel"][lo:lo + nb], c["feats"][lo:lo + nb], c["top_k"], c["thr"],
                              split_rows=out["split"].shape[1])
            for k, v in part.items():
                assert np.array_equal(bits(v), bits(out[k][lo:lo + nb])), (k, lo, nb)
            lo += nb
        assert lo == c["heat"].shape[0]
    print(f"[{name}] n_valid {out['n_valid'][:4].tolist()}... worst descriptor error so far {WORST['err']:.2e} "
          f"({WORST['ratio']:.3f} of the bound)")


# ---------------------------------------------------------------------------------------------------------------------
# dense selection (xfeat_detect_dense)
def rel_maps(rng, Hm, Wm, kinds):
    out = []
    for kind in kinds:
        if kind == "constant":
            r = np.full((Hm, Wm), 0.625, np.float32)
        elif kind == "three_level":
            r = (rng.integers(0, 3, (Hm, Wm)).astype(np.float32) * np.float32(0.25))
        elif kind == "random":
            r = rng.random((Hm, Wm), dtype=np.float32)
        else:   # signed zeros and negative values: -0 must tie with +0
            r = rng.choice(np.array([0.0, -0.0, -0.5, 0.25, -1e-30], np.float32), (Hm, Wm))
        out.append(r)
    return np.stack(out)


KINDS = ("constant", "three_level", "random", "signed_zero")


def dense_case(H, W, k, B=4):
    rng = np.random.default_rng(6000 + H + k + B)
    kinds = [KINDS[i % 4] for i in range(B)]
    rel = rel_maps(rng, H // 8, W // 8, kinds)
    return dict(rel=rel, feats=feats_for(rng, B, H, W), H=H, W=W, top_k=k, rw=1.25, rh=0.8, div_scale=0.6, scale_value=1.25)


def run_dense(xf, c, offset=3, extra=5):
    from accelerated_features_b200 import _lib
    rel, feats, H, W, top_k = c["rel"], c["feats"], c["H"], c["W"], c["top_k"]
    B, cells = rel.shape[0], (H // 8) * (W // 8)
    k = min(top_k, cells)
    rows = offset + k + extra
    d_rel, d_feats = torch.from_numpy(rel).cuda(), torch.from_numpy(feats).cuda()
    kpts = torch.full((B, rows, 2), SENT, device="cuda")
    desc = torch.full((B, rows, 64), SENT, device="cuda")
    sc = torch.full((B, rows), SENT, device="cuda")
    ti = torch.full((B, k), int(SENT), dtype=torch.int32, device="cuda")
    ws = torch.empty(xf._lib.xfeat_dense_workspace_bytes(B, H, W, top_k), dtype=torch.uint8, device="cuda")
    _lib.check(xf._lib.xfeat_detect_dense(xf._ctx, d_feats.data_ptr(), d_rel.data_ptr(), B, H, W, top_k, c["rw"], c["rh"],
                                          c["div_scale"], c["scale_value"], rows, offset, kpts.data_ptr(), desc.data_ptr(),
                                          sc.data_ptr(), ti.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "detect_dense")
    torch.cuda.synchronize()
    return dict(kpts=kpts.cpu().numpy(), desc=desc.cpu().numpy(), scales=sc.cpu().numpy(), topk_idx=ti.cpu().numpy())


def check_dense(c, out, offset=3):
    rel, feats, H, W = c["rel"], c["feats"], c["H"], c["W"]
    B, Wm = rel.shape[0], W // 8
    k = out["topk_idx"].shape[1]
    for b in range(B):
        want = ref.dense_select(rel[b], k)
        assert np.array_equal(out["topk_idx"][b], want), b
        rows = slice(offset, offset + k)
        assert np.array_equal(bits(out["kpts"][b, rows]), bits(ref.dense_kpts_f32(want, Wm, c["rw"], c["rh"], c["div_scale"]))), b
        assert np.array_equal(bits(out["desc"][b, rows]), bits(feats[b].reshape(-1, 64)[want])), b
        assert (out["scales"][b, rows] == np.float32(c["scale_value"])).all()
        for key in ("kpts", "desc", "scales"):      # rows outside [offset, offset + k) are untouched
            assert (out[key][b, :offset] == SENT).all() and (out[key][b, offset + k:] == SENT).all(), (b, key)


DENSE_CASES = {f"{H}x{W}_k{k}": (H, W, k, 4) for H, W in ((1248, 1664), (480, 640)) for k in (1, 7, 8191, 8192, 8193, 10 ** 8)}
DENSE_CASES["1248x1664_k8192_b33"] = (1248, 1664, 8192, 33)
DENSE_CASES["480x640_k2000_b33"] = (480, 640, 2000, 33)


@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_dense_selection(xf, name):
    c = dense_case(*DENSE_CASES[name])
    check_dense(c, run_dense(xf, c))


# ---------------------------------------------------------------------------------------------------------------------
# the diagnostic switches: a child process with all three set must reproduce the outputs bit for bit
SWITCH_SPARSE = ["ties_k512", "ties_k8192", "nms_list_1025", "nms_list_full_cta", "nms_list_straddle", "batch_b33",
                 "batch_b33_k20000_cub", "thr_border"]
SWITCH_DENSE = ["1248x1664_k8192", "1248x1664_k8193", "480x640_k7"]


def run_switch_set(xf):
    outs = {}
    for name in SWITCH_SPARSE:
        outs["s_" + name] = run_case(xf, SPARSE_CASES[name]())
    for name in SWITCH_DENSE:
        outs["d_" + name] = run_dense(xf, dense_case(*DENSE_CASES[name]))
    return outs


def child_main(outdir):
    """Entry point of the child process: run the switch set and save every output array."""
    from accelerated_features_b200 import XFeat
    outs = run_switch_set(XFeat())
    for name, o in outs.items():
        np.savez(os.path.join(outdir, name + ".npz"), **o)


def test_diagnostic_switches_give_the_same_bits(xf, tmp_path):
    env = dict(os.environ, **{s: "1" for s in SWITCHES})
    r = subprocess.run([sys.executable, "-c", f"from tests.test_gpu_select import child_main; child_main({str(tmp_path)!r})"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    for s in SWITCHES:
        assert s not in os.environ          # this process runs the default paths
    mine = run_switch_set(xf)
    for name, o in mine.items():
        with np.load(tmp_path / (name + ".npz")) as z:
            assert set(z.files) == set(o)
            for k, v in o.items():
                assert np.array_equal(bits(z[k]), bits(v)), (name, k)


# ---------------------------------------------------------------------------------------------------------------------
# misaligned pointers are refused before any launch
@pytest.mark.parametrize("which,shift", [("heat", 4), ("feats", 4), ("feats", 8), ("desc", 4), ("desc", 8), ("split", 2),
                                         ("split", 8)])
def test_sparse_misaligned_pointer_is_an_error(xf, which, shift):
    from accelerated_features_b200 import _lib
    B, H, W, k = 1, 64, 64, 64
    bufs = dict(heat=torch.zeros(B * H * W + 16, device="cuda"), feats=torch.zeros(B * (H // 8) * (W // 8) * 64 + 16, device="cuda"),
                desc=torch.zeros(B * k * 64 + 16, device="cuda"), split=torch.zeros(B * 512 * 128 + 16, dtype=torch.float16, device="cuda"))
    ptr = {n: t.data_ptr() for n, t in bufs.items()}
    ptr[which] += shift
    rel = torch.zeros(B * (H // 8) * (W // 8), device="cuda")
    kpts = torch.zeros(B * k * 2, device="cuda"); sc = torch.zeros(B * k, device="cuda")
    nv = torch.zeros(B, dtype=torch.int32, device="cuda")
    ws = torch.empty(xf._lib.xfeat_sparse_workspace_bytes(B, H, W, k), dtype=torch.uint8, device="cuda")
    rc = xf._lib.xfeat_detect_sparse_split(xf._ctx, ptr["feats"], ptr["heat"], rel.data_ptr(), B, H, W, k, 0.05, 1.0, 1.0,
                                           kpts.data_ptr(), sc.data_ptr(), ptr["desc"], nv.data_ptr(), None, None, ptr["split"],
                                           512, ws.data_ptr(), ws.numel(), _stream())
    torch.cuda.synchronize()
    assert rc == 1, rc                                                    # XF_E_INVALID
    assert "aligned" in xf._lib.xfeat_last_error().decode()
    assert not (bufs["desc"].any() or bufs["split"].any() or kpts.any() or nv.any()), "a refused call wrote its outputs"


@pytest.mark.parametrize("which,shift", [("feats", 4), ("desc", 4)])
def test_dense_misaligned_pointer_is_an_error(xf, which, shift):
    from accelerated_features_b200 import _lib
    B, H, W, k = 1, 64, 64, 16
    bufs = dict(feats=torch.zeros(B * (H // 8) * (W // 8) * 64 + 16, device="cuda"), desc=torch.zeros(B * k * 64 + 16, device="cuda"))
    ptr = {n: t.data_ptr() for n, t in bufs.items()}
    ptr[which] += shift
    rel = torch.zeros(B * (H // 8) * (W // 8), device="cuda")
    kpts = torch.zeros(B * k * 2, device="cuda")
    ws = torch.empty(xf._lib.xfeat_dense_workspace_bytes(B, H, W, k), dtype=torch.uint8, device="cuda")
    rc = xf._lib.xfeat_detect_dense(xf._ctx, ptr["feats"], rel.data_ptr(), B, H, W, k, 1.0, 1.0, 1.0, 1.0, k, 0, kpts.data_ptr(),
                                    ptr["desc"], None, None, ws.data_ptr(), ws.numel(), _stream())
    torch.cuda.synchronize()
    assert rc == 1, rc                                                    # XF_E_INVALID
    assert "aligned" in xf._lib.xfeat_last_error().decode()
    assert not (bufs["desc"].any() or kpts.any()), "a refused call wrote its outputs"
