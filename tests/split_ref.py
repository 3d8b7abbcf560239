"""Float64 references of the folded layers, and an exact emulation of the library's split-fp16 tensor-core arithmetic.

Every tensor-core kernel of the library (conv_tc.cu, conv_tc_halo.cu, head_chain_tc.cu, mlp_tc.cu) computes
    y = (hi.whi + hi.wlo + lo.whi) * 2^-k + b
with x = hi + lo (fp16, round to nearest, the activation unscaled) and w * 2^k = whi + wlo (fp16), where 2^k = 2^(13 - e) puts
max |w| of the layer in [2^12, 2^13) (conv_tc_prepare / mlp_tc_prepare).  `emulate` reproduces that with the three partial
products summed in float64, so its distance to the float64 reference is the representation error of the split alone; leaving
one term out shows what a kernel that lost that term would produce.  Functions run on the device of their input.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from accelerated_features_b200 import weights as _weights

BN_EPS = 1e-5

# Tolerances of the tensor-core kernel families against float64.  test_split_error_model.py proves on real weights and
# inputs that each is >= 5x the split's own error and <= 1/5 of the error with any one split term dropped.  The rest of each
# budget is for the fp32 accumulation inside the MMAs, which the emulation does not model (the fine matcher's K = 512 layers
# measure ~1.8e-4 on an H100 against an emulated 1e-5).
CONV_TC_TOL = 1e-5        # conv_tc / halo / 128-channel kernels: max |err| / max |reference| of one layer
KPT_LOGITS_TOL = 5e-4     # keypoint head chain: max |err| of the 65 logits
HEAT_TOL = 5e-5           # keypoint head chain: max |err| of the heat-map after soft-max + depth-to-space
RELIABILITY_TOL = 5e-6    # reliability head chain: max |err| after the sigmoid
FINE_MATCHER_TOL = 6e-4   # fine-matcher MLP: max |err| of the 64 logits
SUBPIX_TOL = 5e-4         # fine-matcher MLP + subpix_softmax2d: max |err| of the offsets, pixels at scale 1

TERMS = ("hi.whi", "hi.wlo", "lo.whi")
STRIDE2 = {1, 3, 7, 10, 13}          # block1.1, block1.3, block3.0, block4.0, block5.0 (csrc/layers.h)
L_SKIP1 = 4
FINE_MATCHER = (27, 28, 29, 30, 31)
KEYPOINT_HEAD = (23, 24, 25, 26)
HEATMAP_HEAD = (20, 21, 22)


def min_tiles_per_cta(rows: int, sms: int) -> int:
    """Lower bound of the tiles every CTA of a persistent launch processes: a tile covers at most 128 output pixels (rows),
    and the grid has at most `sms` CTAs, whatever tile shape pick_tile / pick_halo_tile choose."""
    return -(-rows // 128) // sms


def layer_geometry(layer: int):
    """(ks, stride, pad, relu) of a layer of the packed table."""
    conv, bn = _weights.LAYERS[layer]
    ks = 1 if (layer in (L_SKIP1, 9, 16) or layer >= 19) else 3
    stride = 2 if layer in STRIDE2 else 1
    return ks, stride, ks // 2, bn is not None


def fold64(sd, layer: int):
    """Conv/linear weight (cout, cin, ks, ks) and bias (cout) with the eval BatchNorm folded, in float64."""
    conv, bn = _weights.LAYERS[layer]
    w = sd[conv + ".weight"].double()
    if w.ndim == 2:
        w = w[:, :, None, None]
    b = sd[conv + ".bias"].double() if (conv + ".bias") in sd else torch.zeros(w.shape[0], dtype=torch.float64)
    if bn is not None:
        inv = 1.0 / torch.sqrt(sd[bn + ".running_var"].double() + BN_EPS)
        w = w * inv[:, None, None, None]
        b = (b - sd[bn + ".running_mean"].double()) * inv
    return w, b


def split_weights(sd, layer: int):
    """(whi, wlo, 2^-k, bias) as the library prepares them: BN folded and rounded to fp32 (weights.fold_layer, the blob the
    library is created from), scaled by 2^k, split to fp16.  whi / wlo are float64 tensors (cout, cin, ks, ks)."""
    conv, bn = _weights.LAYERS[layer]
    w32, b32 = _weights.fold_layer(sd, conv, bn)
    mx = float(np.abs(w32).max())
    e = math.frexp(mx)[1] if mx > 0 else 13
    s = np.float32(2.0 ** (13 - e))
    ks, _, _, _ = layer_geometry(layer)
    cout = w32.shape[1]
    v = torch.from_numpy(w32 * s).reshape(ks, ks, -1, cout).permute(3, 2, 0, 1).contiguous()   # [ky,kx,cin,cout] -> OIHW
    whi = v.half()
    wlo = (v - whi.float()).half()
    return whi.double(), wlo.double(), 2.0 ** (e - 13), torch.from_numpy(b32).double()


def split_act(x: torch.Tensor):
    """x = hi + lo as the kernels split fp32 activations (split_nhwc_kernel, store_split_row): hi = fp16_rn(x),
    lo = fp16_rn(x - hi).  Returns float64 tensors holding the fp16 values."""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.double(), lo.double()


def _apply(layer: int, x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    ks, stride, pad, _ = layer_geometry(layer)
    if x.ndim == 2:
        return F.linear(x, w[:, :, 0, 0])
    return F.conv2d(x, w, None, stride=stride, padding=pad)


def _skip64(sd, skip_xn: torch.Tensor) -> torch.Tensor:
    """skip1 (model.py:40-41): AvgPool2d(4) then 1x1 conv 1 -> 24 with bias, in float64.  skip_xn (B, H, W)."""
    w, b = fold64(sd, L_SKIP1)
    w, b = w.to(skip_xn.device), b.to(skip_xn.device)
    return F.conv2d(F.avg_pool2d(skip_xn.double()[:, None], 4, 4), w, b)


def reference(sd, layer: int, x: torch.Tensor, skip_xn: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Float64 layer: x (B,Cin,H,W) or (n,Cin) -> conv/linear + folded BN + ReLU [+ skip1, added after the ReLU]."""
    w, b = fold64(sd, layer)
    w, b = w.to(x.device), b.to(x.device)
    y = _apply(layer, x.double(), w)
    y = y + (b[:, None, None] if y.ndim == 4 else b)
    if layer_geometry(layer)[3]:
        y = torch.relu(y)
    if skip_xn is not None:
        y = y + _skip64(sd, skip_xn)
    return y


def emulate(sd, layer: int, x: torch.Tensor, terms: Iterable[str] = TERMS, skip_xn: Optional[torch.Tensor] = None):
    """The library's split arithmetic on x (fp32 values), the selected subset of TERMS summed in float64."""
    terms = tuple(terms)
    assert set(terms) <= set(TERMS), terms
    whi, wlo, inv, b = split_weights(sd, layer)
    whi, wlo, b = whi.to(x.device), wlo.to(x.device), b.to(x.device)
    hi, lo = split_act(x)
    ops = {"hi.whi": (hi, whi), "hi.wlo": (hi, wlo), "lo.whi": (lo, whi)}
    acc = sum(_apply(layer, *ops[t]) for t in terms) if terms else 0.0
    y = acc * inv + (b[:, None, None] if x.ndim == 4 else b)
    if layer_geometry(layer)[3]:
        y = torch.relu(y)
    if skip_xn is not None:
        y = y + _skip64(sd, skip_xn)
    return y


def reference_chain(sd, layers: Sequence[int], x: torch.Tensor) -> torch.Tensor:
    for l in layers:
        x = reference(sd, l, x)
    return x


def emulate_chain(sd, layers: Sequence[int], x: torch.Tensor, terms: Iterable[str] = TERMS) -> torch.Tensor:
    """Layers in sequence as the fused kernels run them: each output is rounded to fp32 and re-split for the next layer."""
    terms = tuple(terms)
    for l in layers:
        x = emulate(sd, l, x, terms).float()
    return x.double()


def coarse_pairs(f0: torch.Tensor, f1: torch.Tensor) -> torch.Tensor:
    """Fine-matcher input rows as refine_matches builds them (xfeat.py:306-325): [f0[i] | f1[j]] for the mutual nearest
    neighbours (raw dot product) between two dense feature maps (64, h, w).  (n, 128) float32."""
    a, b = f0.reshape(64, -1).t().float(), f1.reshape(64, -1).t().float()
    s = a @ b.t()
    m12, m21 = s.argmax(1), s.argmax(0)
    i0 = torch.nonzero(m21[m12] == torch.arange(len(a), device=a.device))[:, 0]
    return torch.cat([a[i0], b[m12[i0]]], 1)


def dropped_variants():
    """(name, terms) for the full three-term product and for each single term left out."""
    return [("3-term", TERMS)] + [(f"no {t}", tuple(u for u in TERMS if u != t)) for t in TERMS]


def error_model(run, err) -> Dict[str, float]:
    """{variant name: err(run(terms))} over dropped_variants(); `run(terms)` produces the emulated output."""
    return {name: float(err(run(terms))) for name, terms in dropped_variants()}


def check_bound(name: str, bound: float, model: Dict[str, float]):
    """A tolerance must clear the split's own error by 5x and catch each single dropped term by 5x."""
    three = model["3-term"]
    dropped = min(v for k, v in model.items() if k != "3-term")
    assert bound >= 5 * three, f"{name}: bound {bound:.3e} < 5 x three-term error {three:.3e}"
    assert bound <= dropped / 5, f"{name}: bound {bound:.3e} > 1/5 of the smallest dropped-term error {dropped:.3e}"


def fmt_model(model: Dict[str, float]) -> str:
    return ", ".join(f"{k} {v:.2e}" for k, v in model.items())
