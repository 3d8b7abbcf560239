"""Host references of the keypoint selection in csrc/sparse.cu and csrc/dense.cu (numpy only; imports neither torch nor the
product).

Selection is a chain of integer decisions -- which pixel survives the 5x5 NMS, which key passes the top-k cut, in what order --
so the references here are exact wherever the kernels are meant to be exact:
  * `nms_mask`: 5x5 max with -inf padding, x == max and x > thr.  Max is exact, so this is the kernels' decision bit for bit.
  * `scores_f32`: the score nearest(heat) * bilinear(reliability) performed with the operations of `nms_score_key` in its order.
    The kernels use `_rn` intrinsics and `rintf` throughout, so per-operation numpy float32 arithmetic (round to nearest even)
    reproduces them bit for bit.  `scores_f64` is the same formula in float64.
  * `sparse_select` / `dense_select`: the order (score desc, raster index asc) of the emulated float32 scores.
  * `descriptors_f64`: bicubic sampling (A = -0.75, zero padding, ATen grid_sampler_2d) of the channel-normalised feature map
    at the same float32 source coordinate, then L2 normalisation, in float64.
  * `magic_div`: the 2^40-reciprocal division of sample_desc_sorted_kernel.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
NMS_R = 2
BICUBIC_A = -0.75
MAGIC_SHIFT = 40


def f2ord(v: np.ndarray) -> np.ndarray:
    """common.cuh f2ord: float32 -> order-preserving uint32 (larger float, larger uint)."""
    u = np.asarray(v, np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def nms_mask(heat: np.ndarray, thr: float) -> np.ndarray:
    """(..., H, W) float32 -> bool mask of the 5x5 maxima above thr (MaxPool2d(5, 1, 2) pads with -inf).  Separable: the max
    of a window is the max of its row maxima, and max is exact."""
    heat = np.asarray(heat, np.float32)
    H, W = heat.shape[-2:]
    pad = np.full(heat.shape[:-2] + (H + 2 * NMS_R, W + 2 * NMS_R), -np.inf, np.float32)
    pad[..., NMS_R:NMS_R + H, NMS_R:NMS_R + W] = heat
    row = pad[..., :, 0:W].copy()
    for d in range(1, 2 * NMS_R + 1):
        np.maximum(row, pad[..., :, d:d + W], out=row)
    m = row[..., 0:H, :].copy()
    for d in range(1, 2 * NMS_R + 1):
        np.maximum(m, row[..., d:d + H, :], out=m)
    return (heat == m) & (heat > F32(thr))


def src_coord_f32(p: np.ndarray, size_pos: int, size_map: int) -> np.ndarray:
    """common.cuh sparse_src_coord: ((2 * (p / (size_pos - 1)) - 1 + 1) * size_map - 1) / 2, one float32 rounding per op."""
    p = np.asarray(p).astype(np.float32)
    g = F32(2.0) * (p / F32(size_pos - 1)) - F32(1.0)
    return ((g + F32(1.0)) * F32(size_map) - F32(1.0)) / F32(2.0)


def _score(heat, rel, xs, ys, dt):
    """nearest(heat) * bilinear(rel) at integer pixels (xs, ys), every operation rounded to dtype `dt`; (0, 0) -> -1."""
    H, W = heat.shape
    Hm, Wm = rel.shape
    xs = np.asarray(xs, np.int64)
    ys = np.asarray(ys, np.int64)
    heat = heat.astype(dt)
    rel = rel.astype(dt)
    one, two = dt(1.0), dt(2.0)

    def src(p, size_pos, size_map):
        g = two * (p.astype(dt) / dt(size_pos - 1)) - one
        return ((g + one) * dt(size_map) - one) / two

    # nearest tap: round half to even (rintf / nearbyint); the last row / column falls out of range and reads 0
    xn = np.rint(src(xs, W, W)).astype(np.int64)
    yn = np.rint(src(ys, H, H)).astype(np.int64)
    inn = (xn >= 0) & (xn < W) & (yn >= 0) & (yn < H)
    kv = np.where(inn, heat[np.clip(yn, 0, H - 1), np.clip(xn, 0, W - 1)], dt(0.0))
    ix, iy = src(xs, W, Wm), src(ys, H, Hm)
    fx, fy = np.floor(ix), np.floor(iy)
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    wx1, wx0 = ix - fx, (fx + one) - ix
    wy1, wy0 = iy - fy, (fy + one) - iy
    bil = np.zeros(len(xs), dt)
    for yy, xx, w in ((y0, x0, wx0 * wy0), (y0, x0 + 1, wx1 * wy0), (y0 + 1, x0, wx0 * wy1), (y0 + 1, x0 + 1, wx1 * wy1)):
        ok = (xx >= 0) & (xx < Wm) & (yy >= 0) & (yy < Hm)    # zeros padding: a tap outside adds nothing (not even -0)
        r = rel[np.clip(yy, 0, Hm - 1), np.clip(xx, 0, Wm - 1)]
        bil = np.where(ok, bil + r * w, bil)
    s = kv * bil
    return np.where((xs == 0) & (ys == 0), dt(-1.0), s).astype(dt)


def scores_f32(heat: np.ndarray, rel: np.ndarray, xs, ys) -> np.ndarray:
    """Float32 emulation of nms_score_key for one image: heat (H, W), rel (H/8, W/8)."""
    return _score(np.asarray(heat, np.float32), np.asarray(rel, np.float32), xs, ys, np.float32)


def scores_f64(heat: np.ndarray, rel: np.ndarray, xs, ys) -> np.ndarray:
    """The score formula of scores_f32 evaluated in float64."""
    return _score(np.asarray(heat, np.float32), np.asarray(rel, np.float32), xs, ys, np.float64)


def sparse_select(heat: np.ndarray, rel: np.ndarray, thr: float, top_k: int, mask: np.ndarray = None) -> dict:
    """The selection of xfeat_detect_sparse for one image: NMS candidates, emulated float32 scores, `score > 0`, the
    H*W/4 capacity, and the top-k in the order (score desc, y * W + x asc).  `mask` may pass a precomputed nms_mask."""
    H, W = heat.shape
    if mask is None:
        mask = nms_mask(heat, thr)
    ys, xs = np.nonzero(mask)
    s = scores_f32(heat, rel, xs, ys)
    keep = s > 0
    xs, ys, s = xs[keep], ys[keep], s[keep]
    n_keep, cap = len(s), H * W // 4
    out = dict(n_cand=len(keep), n_keep=n_keep, cap=cap)
    if n_keep > cap:                                   # XF_N_OVERFLOW: nothing of the image is trusted
        out.update(n_valid=-1, x=xs[:0], y=ys[:0], score=s[:0], all_scores=s)
        return out
    lin = ys.astype(np.int64) * W + xs
    order = np.lexsort((lin, -s.astype(np.float64)))[:top_k]
    out.update(n_valid=len(order), x=xs[order], y=ys[order], score=s[order], all_scores=s)
    return out


def dense_select(rel: np.ndarray, k: int) -> np.ndarray:
    """Cell indices of the k most reliable cells, (value desc, cell asc); +0 and -0 are equal.  rel (Hm, Wm) float32."""
    v = np.asarray(rel, np.float32).reshape(-1) + F32(0.0)
    return np.lexsort((np.arange(len(v)), -v.astype(np.float64)))[:k]


def dense_kpts_f32(cells: np.ndarray, Wm: int, rw: float, rh: float, div_scale: float) -> np.ndarray:
    """dense_gather_kernel's keypoint: fp32(fp32(8 x) * rw) / div_scale, and the same for y."""
    x, y = cells % Wm, cells // Wm
    kx = (x * 8).astype(np.float32) * F32(rw) / F32(div_scale)
    ky = (y * 8).astype(np.float32) * F32(rh) / F32(div_scale)
    return np.stack([kx, ky], -1).astype(np.float32)


def _cubic1(t):   # |t| <= 1
    return ((BICUBIC_A + 2) * t - (BICUBIC_A + 3)) * t * t + 1


def _cubic2(t):   # 1 < |t| < 2
    return ((BICUBIC_A * t - 5 * BICUBIC_A) * t + 8 * BICUBIC_A) * t - 4 * BICUBIC_A


def bicubic_taps(xs, ys, H: int, W: int, Hm: int, Wm: int):
    """Per keypoint: tap cell rows (n, 4), columns (n, 4) and float64 weights cy (n, 4), cx (n, 4), at the float32 source
    coordinate of the kernels (ATen grid_sampler_2d bicubic, A = -0.75)."""
    ix = src_coord_f32(xs, W, Wm).astype(np.float64)
    iy = src_coord_f32(ys, H, Hm).astype(np.float64)
    fx, fy = np.floor(ix), np.floor(iy)
    tx, ty = ix - fx, iy - fy
    cx = np.stack([_cubic2(tx + 1), _cubic1(tx), _cubic1(1 - tx), _cubic2(2 - tx)], -1)
    cy = np.stack([_cubic2(ty + 1), _cubic1(ty), _cubic1(1 - ty), _cubic2(2 - ty)], -1)
    cols = fx.astype(np.int64)[:, None] - 1 + np.arange(4)
    rows = fy.astype(np.int64)[:, None] - 1 + np.arange(4)
    return rows, cols, cy, cx


def descriptors_f64(feats: np.ndarray, xs, ys, H: int, W: int):
    """Float64 descriptors of the keypoints (xs, ys) of one image: feats (Hm, Wm, 64) un-normalised.  Returns
    (unit descriptors (n, 64), T (n, 64), norm (n,)), where T[c] = sum over the 16 taps of |f_c| / ||f|| -- the size of the
    terms the kernel sums, which its rounding error scales with -- and norm the length before the final normalisation."""
    Hm, Wm, C = feats.shape
    f = feats.astype(np.float64)
    den = 1.0 / np.maximum(np.sqrt((f * f).sum(-1)), 1e-12)
    rows, cols, cy, cx = bicubic_taps(np.asarray(xs), np.asarray(ys), H, W, Hm, Wm)
    n = len(rows)
    acc = np.zeros((n, C))
    tsum = np.zeros((n, C))
    for i in range(4):
        for j in range(4):
            r, c = rows[:, i], cols[:, j]
            ok = (r >= 0) & (r < Hm) & (c >= 0) & (c < Wm)
            v = f[np.clip(r, 0, Hm - 1), np.clip(c, 0, Wm - 1)] * den[np.clip(r, 0, Hm - 1), np.clip(c, 0, Wm - 1)][:, None]
            v[~ok] = 0.0
            acc += (cy[:, i] * cx[:, j])[:, None] * v
            tsum += np.abs(v)
    norm = np.sqrt((acc * acc).sum(-1))
    return acc / np.maximum(norm, 1e-12)[:, None], tsum, norm


def split_f16(desc: np.ndarray):
    """store_desc_split: x * 2^13 = hi + lo, hi = fp16_rn(x * 2^13), lo = fp16_rn(x * 2^13 - hi) (the difference is exact
    in float32)."""
    x = np.asarray(desc, np.float32) * F32(8192.0)
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def magic(d: int) -> int:
    """The 2^40 reciprocal of d used by sample_desc_sorted_kernel: floor(2^40 / d) + 1."""
    return (1 << MAGIC_SHIFT) // d + 1


def magic_div(n: np.ndarray, d: int) -> np.ndarray:
    """(n * magic(d)) >> 40 in 64-bit unsigned arithmetic, as the kernel computes it.  Exact (== n // d) when n * d < 2^40:
    magic(d) * d = 2^40 + e with 0 < e <= d, so n * magic / 2^40 = n / d + n * e / (d * 2^40), and the excess stays below 1/d
    -- too little to reach the next integer -- while n * e < 2^40."""
    n = np.asarray(n, np.uint64)
    return (n * np.uint64(magic(d))) >> np.uint64(MAGIC_SHIFT)


def sorted_sampler_strips(Hm: int) -> int:
    """Column strips per feature row of sample_desc_sorted_kernel: max(1, min(8, 512 // Hm))."""
    return max(1, min(8, 512 // Hm))
