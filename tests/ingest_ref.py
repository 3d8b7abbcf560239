"""Host reference of image ingest in csrc/prep.cu (numpy only; imports neither torch nor the product).

Ingest is bilinear resampling (ATen upsample_bilinear2d, align_corners=False), a channel mean and InstanceNorm2d(1).  The
kernels do every float32 operation with an `_rn` intrinsic, and numpy float32 arithmetic is correctly rounded too, so the
emulation here reproduces them bit for bit:
  * `lin_taps`: common.cuh lin_tap, src = (dst + 0.5) * scale - 0.5 (no FMA) clamped at 0, i0 = int(src) clamped to in - 1,
    i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1.  ATen's CPU kernel contracts the source index into an FMA, so where
    the two source indices round apart, l1 differs by one ulp of src and the output by that times the neighbours' difference.
  * `bilinear`: per plane l0h * (l0w * v00 + l1w * v01) + l1h * (l0w * v10 + l1w * v11).  An axis whose size does not
    change is sampled at scale 1 (src == dst, l1 == 0): ATen copies along it, whatever scale it was given (`effective_scales`).
  * `gray`: uint8 taps as float(u8) / 255 when `div255` is set, the channel sum in channel order, then / C unless C == 1.
  * `instnorm_params` / `instnorm_f32`: InstanceNorm from given fp64 (sum, sum of squares), as instnorm_params in prep.cu.
`bilinear_f64`, `gray_f64` and `instnorm_f64` are the same operations in float64, for error bounds.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32
IN_EPS = 1e-5


def size_scale(n_in: int, n_out: int) -> np.float32:
    """ATen area_pixel_compute_scale for F.interpolate(size=...): float(in) / out."""
    return F32(n_in) / F32(n_out)


def factor_scale(s: float) -> np.float32:
    """ATen area_pixel_compute_scale for F.interpolate(scale_factor=s): float(1 / s)."""
    return F32(1.0 / s)


def effective_scales(Hi: int, Wi: int, Ho: int, Wo: int, scale_h, scale_w):
    """ATen copies along an axis whose size does not change, whatever its scale (compute_source_index_and_lambda); the kernels
    sample that axis at scale 1, which copies."""
    return F32(1) if Ho == Hi else F32(scale_h), F32(1) if Wo == Wi else F32(scale_w)


def lin_taps(n_out: int, n_in: int, scale, fma: bool = False):
    """common.cuh lin_tap for dst = 0 .. n_out-1 -> (i0, i1, l0, l1).  `fma`: the source index as one fused multiply-add
    instead, fl32((dst + 0.5) * scale - 0.5), as ATen's CPU build computes it (the float64 expression is exact)."""
    dst = np.arange(n_out, dtype=F32)
    if fma:
        src = ((dst + F32(0.5)).astype(np.float64) * float(F32(scale)) - 0.5).astype(F32)
    else:
        src = (dst + F32(0.5)) * F32(scale) - F32(0.5)
    src = np.where(src < 0, F32(0), src)
    i0 = np.minimum(src.astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = src - i0.astype(F32)
    l0 = F32(1) - l1
    return i0, i1, l0, l1


def values(img: np.ndarray, div255: bool) -> np.ndarray:
    """Pixel values as the kernels load them: float(u8) or the float32 value, then / 255 when `div255`."""
    v = np.asarray(img).astype(F32)
    return v / F32(255) if div255 else v


def bilinear(v: np.ndarray, Ho: int, Wo: int, scale_h, scale_w, fma: bool = False) -> np.ndarray:
    """(..., Hi, Wi) float32 -> (..., Ho, Wo) float32 in the kernels' operation order (`fma`: see lin_taps)."""
    v = np.asarray(v, F32)
    Hi, Wi = v.shape[-2:]
    sh, sw = effective_scales(Hi, Wi, Ho, Wo, scale_h, scale_w)
    i0h, i1h, l0h, l1h = lin_taps(Ho, Hi, sh, fma)
    i0w, i1w, l0w, l1w = lin_taps(Wo, Wi, sw, fma)
    r0, r1 = v[..., i0h, :], v[..., i1h, :]
    top = l0w * r0[..., i0w] + l1w * r0[..., i1w]
    bot = l0w * r1[..., i0w] + l1w * r1[..., i1w]
    return l0h[:, None] * top + l1h[:, None] * bot


def resize(img: np.ndarray, Ho: int, Wo: int, scale_h, scale_w, div255: bool = False, fma: bool = False) -> np.ndarray:
    """xfeat_resize_bilinear: (B, C, Hi, Wi) uint8 or float32 -> (B, C, Ho, Wo) float32."""
    return np.stack([bilinear(values(img[b], div255), Ho, Wo, scale_h, scale_w, fma) for b in range(img.shape[0])])


def gray(img: np.ndarray, H: int, W: int, scale_h=None, scale_w=None, div255: bool = False) -> np.ndarray:
    """The gray image of xfeat_preprocess(_scaled) before normalisation: (B, C, Hi, Wi) -> (B, H, W) float32.
    Scales default to in / out (xfeat_preprocess)."""
    B, C, Hi, Wi = img.shape
    sh = size_scale(Hi, H) if scale_h is None else scale_h
    sw = size_scale(Wi, W) if scale_w is None else scale_w
    out = np.empty((B, H, W), F32)
    for b in range(B):
        acc = np.zeros((H, W), F32)
        for c in range(C):
            acc = acc + bilinear(values(img[b, c], div255), H, W, sh, sw)
        out[b] = acc if C == 1 else acc / F32(C)
    return out


def stats_f64(g: np.ndarray) -> np.ndarray:
    """(B, H, W) -> (B, 2) float64 (sum, sum of squares) of the float32 gray values."""
    g = np.asarray(g, np.float64).reshape(g.shape[0], -1)
    return np.stack([g.sum(1), (g * g).sum(1)], 1)


def instnorm_params(s: float, ss: float, n: int):
    """prep.cu instnorm_params: every double operation rounded on its own, then mean and 1 / sqrt(var + eps) to float32."""
    mean = float(s) / float(n)
    var = float(ss) / float(n) - mean * mean
    var = max(var, 0.0)
    return F32(mean), F32(1.0 / math.sqrt(var + IN_EPS))


def instnorm_f32(g: np.ndarray, stats: np.ndarray) -> np.ndarray:
    """xn = fl32(fl32(g - meanf) * invstd) per image, with (meanf, invstd) from the given fp64 sums."""
    g = np.asarray(g, F32)
    out = np.empty_like(g)
    n = g.shape[1] * g.shape[2]
    for b in range(g.shape[0]):
        meanf, invstd = instnorm_params(stats[b, 0], stats[b, 1], n)
        out[b] = (g[b] - meanf) * invstd
    return out


# ---------------------------------------------------------------------------------------------------------------------
# float64 path
def bilinear_f64(v: np.ndarray, Ho: int, Wo: int, scale_h, scale_w) -> np.ndarray:
    """`bilinear` in float64: the kernels' taps (i0, i1, l1 = src - i0 from the float32 source index), l0 = 1 - l1 and the
    interpolation in float64."""
    v = np.asarray(v, np.float64)
    Hi, Wi = v.shape[-2:]
    sh, sw = effective_scales(Hi, Wi, Ho, Wo, scale_h, scale_w)

    def taps(n_out, n_in, scale):
        i0, i1, _, l1 = lin_taps(n_out, n_in, scale)
        l1 = l1.astype(np.float64)
        return i0, i1, 1.0 - l1, l1

    i0h, i1h, l0h, l1h = taps(Ho, Hi, sh)
    i0w, i1w, l0w, l1w = taps(Wo, Wi, sw)
    r0, r1 = v[..., i0h, :], v[..., i1h, :]
    top = l0w * r0[..., i0w] + l1w * r0[..., i1w]
    bot = l0w * r1[..., i0w] + l1w * r1[..., i1w]
    return l0h[:, None] * top + l1h[:, None] * bot


def gray_f64(img: np.ndarray, H: int, W: int, scale_h=None, scale_w=None, div255: bool = False) -> np.ndarray:
    B, C, Hi, Wi = img.shape
    sh = size_scale(Hi, H) if scale_h is None else scale_h
    sw = size_scale(Wi, W) if scale_w is None else scale_w
    v = np.asarray(img, np.float64)
    if div255:
        v = v / 255.0
    return bilinear_f64(v, H, W, sh, sw).mean(1)


def instnorm_f64(g: np.ndarray) -> np.ndarray:
    """InstanceNorm2d(1) in float64 with a two-pass (biased) variance."""
    g = np.asarray(g, np.float64)
    mean = g.mean((1, 2), keepdims=True)
    var = ((g - mean) ** 2).mean((1, 2), keepdims=True)
    return (g - mean) / np.sqrt(var + IN_EPS)


def instnorm_f32_bound(g: np.ndarray, stats: np.ndarray) -> np.ndarray:
    """Per-pixel bound on |instnorm_f32(g, stats) - instnorm_f64(g)| when `stats` are the fp64 sums of g up to summation error.
    Rounding the mean to float32 moves every value by |mean - meanf| * invstd.  g - meanf, invstd and the product are each
    rounded once to float32 (2^-24 relative each).  The one-pass variance sum_sq / n - mean^2 loses (sum_sq / n) / var times the
    relative error of sum_sq, taken here as 2^-44 (2^9 double roundings: the atomics of a two-kernel form add up to a few
    thousand block sums one after another, with errors of both signs); invstd gets half of that."""
    g64 = np.asarray(g, np.float64)
    n = g.shape[1] * g.shape[2]
    ref = instnorm_f64(g)
    out = np.empty_like(g64)
    for b in range(g.shape[0]):
        mean = g64[b].mean()
        var = ((g64[b] - mean) ** 2).mean()
        meanf, _ = instnorm_params(stats[b, 0], stats[b, 1], n)
        invstd = 1.0 / math.sqrt(var + IN_EPS)
        rel = 3 * 2.0 ** -24 + 0.5 * 2.0 ** -44 * (stats[b, 1] / n) / (var + IN_EPS)
        out[b] = abs(mean - float(meanf)) * invstd * (1 + rel) + np.abs(ref[b]) * rel * 1.01
    return out
