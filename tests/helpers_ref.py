"""Float64 / exact references of the stand-alone helper kernels (csrc/helpers.cu), with error bounds derived from each kernel's
operation order.  u = 2^-24 is the fp32 unit roundoff; CUDA's expf is within 2 ulp (CUDA C Programming Guide, Table 13).

- heatmap_ref: get_kpts_heatmap (xfeat.py:242-247) in float64.  heatmap_bound: the kernel rounds z = x * temp (|z| u, which
  enters the exponent as an absolute error), subtracts the cell maximum (|z - m| u), calls expf (2 ulp), sums 65 terms in order
  (64 u relative) and divides once (u).
- nms_ref: oracle.nms_numpy per image (MaxPool2d with -inf padding; NaN propagates through the max as in ATen).
- source_coord: oracle.source_coord, whose numpy float32 operations are each correctly rounded, so it is the kernel's hl_src for
  fractional positions too.
- sample_ref: grid_sample(align_corners=False, zeros padding) at that fp32 coordinate: nearest exactly (round half to even, as
  ATen's nearbyint and the kernel's rintf), bilinear and bicubic (A = -0.75) in float64, each with a bound on the kernel's fp32
  evaluation.
- subpix_ref: subpix_softmax2d (xfeat.py:292-304) in float64, with subpix_bound.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import xfeat_oracle as orc

U = 2.0 ** -24
EXPF_ULP = 2
TINY = 2.0 ** -120       # absolute slack for results that underflow in fp32
A_CUBIC = -0.75


def heatmap_ref(logits: torch.Tensor, temp: float) -> torch.Tensor:
    """(B, 65, Hc, Wc) fp32 -> (B, 1, 8 Hc, 8 Wc) float64: softmax(x * temp) over 65, dustbin dropped, depth-to-space."""
    return orc.kpts_heatmap(logits.double(), temp)


def heatmap_bound(logits: torch.Tensor, temp: float) -> torch.Tensor:
    """Per-element bound on |kernel - heatmap_ref|, laid out as the heat-map."""
    z = logits.double() * temp
    m = z.max(1, keepdim=True)[0]
    e_exp = U * (z.abs() + m.abs() + (z - m).abs()) + EXPF_ULP * U          # relative error of each exp term
    e_exp = torch.where(torch.isfinite(z), e_exp, torch.zeros_like(e_exp))   # exp(-inf) = 0 exactly
    rel = e_exp + e_exp.max(1, keepdim=True)[0] + 64 * U + U                 # its own term, the sum, the division
    p = torch.softmax(z, 1)
    b = p * rel * (1 + 1e-6) + TINY
    return _d2s(b[:, :64])


def _d2s(p: torch.Tensor) -> torch.Tensor:
    B, _, H, W = p.shape
    return p.permute(0, 2, 3, 1).reshape(B, H, W, 8, 8).permute(0, 1, 3, 2, 4).reshape(B, 1, H * 8, W * 8)


def nms_ref(heat: np.ndarray, threshold: float, kernel_size: int):
    """heat (B, H, W) float32 -> list of (n_b, 2) int64 (x, y) in raster order."""
    return [orc.nms_numpy(h, threshold, kernel_size // 2) for h in heat]


def source_coord(p: np.ndarray, size_pos: int, size_map: int) -> np.ndarray:
    return orc.source_coord(np.asarray(p, np.float32), size_pos, size_map)


def _taps(x: np.ndarray, b: np.ndarray, yy: np.ndarray, xx: np.ndarray) -> np.ndarray:
    """x (B, C, Hm, Wm) float64; b, yy, xx (M,) -> (M, C), zero outside the map."""
    _, _, Hm, Wm = x.shape
    ok = (yy >= 0) & (yy < Hm) & (xx >= 0) & (xx < Wm)
    v = x[b, :, np.clip(yy, 0, Hm - 1), np.clip(xx, 0, Wm - 1)]
    return np.where(ok[:, None], v, 0.0)


def _cubic1(t):
    return ((A_CUBIC + 2) * t - (A_CUBIC + 3)) * t * t + 1


def _cubic2(t):
    return ((A_CUBIC * t - 5 * A_CUBIC) * t + 8 * A_CUBIC) * t - 4 * A_CUBIC


def sample_ref(x: np.ndarray, pos: np.ndarray, H: int, W: int, mode: str):
    """x (B, C, Hm, Wm) float32, pos (B, N, 2) float32 -> (value (B, N, C) float64, bound (B, N, C) float64).  Nearest is exact
    (bound 0).  Bilinear: exact fp32 weights, four rounded products and four rounded sums -> 6 u sum |v w|.  Bicubic: each
    coefficient within 8 u of its float64 value (a cubic with |coefficients| <= 4 on [0, 2]), one product of two and a 16-term
    fma chain -> 32 u sum |v|."""
    B, C, Hm, Wm = x.shape
    N = pos.shape[1]
    xd = x.astype(np.float64)
    ix = source_coord(pos[..., 0], W, Wm).astype(np.float64).reshape(-1)
    iy = source_coord(pos[..., 1], H, Hm).astype(np.float64).reshape(-1)
    b = np.repeat(np.arange(B), N)
    if mode == "nearest":
        v = _taps(xd, b, np.rint(iy).astype(np.int64), np.rint(ix).astype(np.int64))
        return v.reshape(B, N, C), np.zeros((B, N, C))
    fx, fy = np.floor(ix), np.floor(iy)
    tx, ty = ix - fx, iy - fy
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    out = np.zeros((B * N, C))
    mag = np.zeros((B * N, C))
    if mode == "bilinear":
        for dy, wy in ((0, 1 - ty), (1, ty)):
            for dx, wx in ((0, 1 - tx), (1, tx)):
                t = _taps(xd, b, y0 + dy, x0 + dx) * (wx * wy)[:, None]
                out += t
                mag += np.abs(t)
        return out.reshape(B, N, C), (6 * U * mag + TINY).reshape(B, N, C)
    cx = [_cubic2(tx + 1), _cubic1(tx), _cubic1(1 - tx), _cubic2(2 - tx)]
    cy = [_cubic2(ty + 1), _cubic1(ty), _cubic1(1 - ty), _cubic2(2 - ty)]
    for i in range(4):
        for j in range(4):
            t = _taps(xd, b, y0 - 1 + i, x0 - 1 + j)
            out += t * (cx[j] * cy[i])[:, None]
            mag += np.abs(t)
    return out.reshape(B, N, C), (32 * U * mag + TINY).reshape(B, N, C)


def subpix_ref(maps: torch.Tensor, temp: float) -> torch.Tensor:
    """(n, 64) fp32 -> (n, 2) float64: E[(x - 4, y - 4)] under softmax(temp * map), x the fast axis."""
    p = torch.softmax(temp * maps.double(), -1)
    ar = torch.arange(64, device=maps.device)
    return torch.stack([p @ (ar % 8 - 4).double(), p @ (ar // 8 - 4).double()], -1)


def subpix_bound(maps: torch.Tensor, temp: float) -> torch.Tensor:
    """Per-map bound (n,) on |kernel - subpix_ref| in pixels.  Each weight exp(z_k - m) carries a relative error
    d_k <= u (|z_k| + |m| + |z_k - m|) + 2 u; an expectation of values in [-4, 3] moves by at most 2 * 8 max_k d_k.  The
    lane-pair products and the 6-level shuffle sums of sx, sy and s, and the final division, add < 16 u relative to s (x 4 px)."""
    z = maps.double() * temp
    m = z.max(1, keepdim=True)[0]
    d = (U * (z.abs() + m.abs() + (z - m).abs()) + EXPF_ULP * U).max(1)[0]
    return 16 * d + 64 * U + TINY
