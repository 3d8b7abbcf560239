"""Pack an XFeat state_dict into the flat fp32 blob libxfeat_sm90.so expects (csrc/layers.h).

Every conv / linear is stored as W[tap][cin][cout] (cout fastest) followed by bias[cout], with the eval-mode
BatchNorm(affine=False, eps=1e-5) that follows it folded in (model.py:12-25, 97-111):
    W' = W / sqrt(var + eps)        b' = (b - mean) / sqrt(var + eps)
"""
from __future__ import annotations

import os
from typing import Dict, Mapping

import numpy as np

BN_EPS = 1e-5
DEFAULT_WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "weights", "xfeat_state.npz")

# (conv/linear prefix, batch-norm prefix or None) in csrc/layers.h order
_BASIC = lambda p: (p + ".layer.0", p + ".layer.1")  # noqa: E731
LAYERS = [
    _BASIC("block1.0"), _BASIC("block1.1"), _BASIC("block1.2"), _BASIC("block1.3"), ("skip1.1", None),
    _BASIC("block2.0"), _BASIC("block2.1"),
    _BASIC("block3.0"), _BASIC("block3.1"), _BASIC("block3.2"),
    _BASIC("block4.0"), _BASIC("block4.1"), _BASIC("block4.2"),
    _BASIC("block5.0"), _BASIC("block5.1"), _BASIC("block5.2"), _BASIC("block5.3"),
    _BASIC("block_fusion.0"), _BASIC("block_fusion.1"), ("block_fusion.2", None),
    _BASIC("heatmap_head.0"), _BASIC("heatmap_head.1"), ("heatmap_head.2", None),
    _BASIC("keypoint_head.0"), _BASIC("keypoint_head.1"), _BASIC("keypoint_head.2"), ("keypoint_head.3", None),
    ("fine_matcher.0", "fine_matcher.1"), ("fine_matcher.3", "fine_matcher.4"), ("fine_matcher.6", "fine_matcher.7"),
    ("fine_matcher.9", "fine_matcher.10"), ("fine_matcher.12", None),
]


def _np(v) -> np.ndarray:
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v)


def load_state_dict(weights) -> Dict[str, np.ndarray]:
    """Accepts a path (.npz, or .pt/.pth via torch.load), or a mapping name -> tensor/ndarray."""
    if isinstance(weights, (str, os.PathLike)):
        path = os.fspath(weights)
        if path.endswith(".npz"):
            with np.load(path) as z:
                return {k: z[k] for k in z.files}
        import torch
        sd = torch.load(path, map_location="cpu")
        return {k: _np(v) for k, v in sd.items()}
    if isinstance(weights, Mapping):
        return {k: _np(v) for k, v in weights.items()}
    raise TypeError(f"unsupported weights argument: {type(weights)!r}")


def random_state_dict(seed: int = 0) -> Dict[str, np.ndarray]:
    """Random-init weights of the XFeat architecture (for `weights=None` and synthetic benchmarks)."""
    rs = np.random.RandomState(seed)
    spec = [(1, 4, 3), (4, 8, 3), (8, 8, 3), (8, 24, 3), (1, 24, 1), (24, 24, 3), (24, 24, 3), (24, 64, 3), (64, 64, 3),
            (64, 64, 1), (64, 64, 3), (64, 64, 3), (64, 64, 3), (64, 128, 3), (128, 128, 3), (128, 128, 3), (128, 64, 1),
            (64, 64, 3), (64, 64, 3), (64, 64, 1), (64, 64, 1), (64, 64, 1), (64, 1, 1), (64, 64, 1), (64, 64, 1),
            (64, 64, 1), (64, 65, 1)]
    sd: Dict[str, np.ndarray] = {}
    for (conv, bn), (cin, cout, ks) in zip(LAYERS[:27], spec):
        bound = 1.0 / np.sqrt(cin * ks * ks)
        sd[conv + ".weight"] = rs.uniform(-bound, bound, (cout, cin, ks, ks)).astype(np.float32)
        if bn is None:
            sd[conv + ".bias"] = rs.uniform(-bound, bound, (cout,)).astype(np.float32)
        else:
            sd[bn + ".running_mean"] = (0.1 * rs.standard_normal(cout)).astype(np.float32)
            sd[bn + ".running_var"] = rs.uniform(0.5, 1.5, cout).astype(np.float32)
    for (lin, bn), (cin, cout) in zip(LAYERS[27:], [(128, 512), (512, 512), (512, 512), (512, 512), (512, 64)]):
        bound = 1.0 / np.sqrt(cin)
        sd[lin + ".weight"] = rs.uniform(-bound, bound, (cout, cin)).astype(np.float32)
        sd[lin + ".bias"] = rs.uniform(-bound, bound, (cout,)).astype(np.float32)
        if bn is not None:
            sd[bn + ".running_mean"] = (0.1 * rs.standard_normal(cout)).astype(np.float32)
            sd[bn + ".running_var"] = rs.uniform(0.5, 1.5, cout).astype(np.float32)
    return sd


def fold_layer(sd: Mapping[str, np.ndarray], conv: str, bn):
    """Returns (W[tap][cin][cout] float32, bias[cout] float32) with BN folded (computed in float64)."""
    w = _np(sd[conv + ".weight"]).astype(np.float64)
    if w.ndim == 2:  # nn.Linear (cout, cin)
        w = w[:, :, None, None]
    cout = w.shape[0]
    b = _np(sd[conv + ".bias"]).astype(np.float64) if (conv + ".bias") in sd else np.zeros(cout)
    if bn is not None:
        inv = 1.0 / np.sqrt(_np(sd[bn + ".running_var"]).astype(np.float64) + BN_EPS)
        w = w * inv[:, None, None, None]
        b = (b - _np(sd[bn + ".running_mean"]).astype(np.float64)) * inv
    wk = np.transpose(w, (2, 3, 1, 0)).reshape(-1, cout)  # (ky,kx,cin,cout) -> [tap*cin][cout]
    return np.ascontiguousarray(wk, dtype=np.float32), b.astype(np.float32)


def pack_weights(sd: Mapping[str, np.ndarray]) -> np.ndarray:
    chunks = []
    pad4 = lambda n: (-n) % 4  # noqa: E731
    for conv, bn in LAYERS:
        w, b = fold_layer(sd, conv, bn)
        for arr in (w.reshape(-1), b):
            chunks.append(arr)
            if pad4(arr.size):
                chunks.append(np.zeros(pad4(arr.size), np.float32))
    return np.ascontiguousarray(np.concatenate(chunks), dtype=np.float32)
