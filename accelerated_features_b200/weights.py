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


def _pad4(chunks, arr):
    chunks.append(np.asarray(arr, np.float32).reshape(-1))
    if chunks[-1].size % 4:
        chunks.append(np.zeros((-chunks[-1].size) % 4, np.float32))


# ---------------------------------------------------------------------------------------------------------------------
# LighterGlue (modules/lighterglue.py): the `matcher.*` part of weights/xfeat-lighterglue.pt
# ---------------------------------------------------------------------------------------------------------------------
# The matcher's weights are not shipped with the package: they are the published weights/xfeat-lighterglue.pt of the reference
# (the reference itself downloads them when its checkout lacks the file, lighterglue.py:35-38).  Put that file here, or pass its
# path to XFeat(lighterglue_weights=...).
LG_DEFAULT_WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "weights", "xfeat-lighterglue.pt")
LG_LAYERS = 6
LG_DIM = 96


def save_lighterglue_state(pt_path: str, out_path: str) -> Dict[str, np.ndarray]:
    """Re-save the published `matcher.*` state as .npz with lighterglue.py:40-46's renaming (`self_attn.{i}` ->
    `transformers.{i}.self_attn`, same for cross_attn, `matcher.` prefix dropped)."""
    sd = load_lighterglue_state(pt_path)
    np.savez(out_path, **{k: np.ascontiguousarray(v, dtype=np.float32) for k, v in sd.items()})
    return sd


def load_lighterglue_state(weights=LG_DEFAULT_WEIGHTS) -> Dict[str, np.ndarray]:
    """The matcher state from the published .pt (extractor + matcher; the `matcher.*` part is kept, renamed), a re-saved .npz,
    or a mapping with the renamed keys."""
    if isinstance(weights, (str, os.PathLike)) and not os.path.exists(weights):
        raise FileNotFoundError(
            f"LighterGlue weights not found at {os.fspath(weights)}: place the published weights/xfeat-lighterglue.pt of "
            "verlab/accelerated_features there, or pass its path as XFeat(lighterglue_weights=...)")
    sd = load_state_dict(weights)
    if any(k.startswith("matcher.") for k in sd):
        out = {}
        for k, v in sd.items():
            if not k.startswith("matcher."):
                continue
            for i in range(LG_LAYERS):
                k = k.replace(f"self_attn.{i}", f"transformers.{i}.self_attn").replace(f"cross_attn.{i}",
                                                                                     f"transformers.{i}.cross_attn")
            out[k[len("matcher."):]] = v
        sd = out
    return sd


def pack_lighterglue(sd: Mapping[str, np.ndarray]) -> np.ndarray:
    """Flat fp32 blob of xfeat_lg_create (csrc/lighterglue.cu, `LgWeights`).  Every linear is stored as W[in][out] (out fastest)
    followed by its bias, each array padded to 4 floats.  Only row permutations, no arithmetic: Wqkv is de-interleaved from
    (q, k, v) = output rows (3i, 3i+1, 3i+2) into [q | k | v], and each cross block's to_qk and to_v are stored as one
    96 -> 192 linear [qk | v]."""
    g = lambda k: _np(sd[k]).astype(np.float32)  # noqa: E731
    lin = lambda w: np.ascontiguousarray(w.T)     # noqa: E731  (out,in) -> [in][out]
    chunks = []
    _pad4(chunks, lin(g("input_proj.weight")))
    _pad4(chunks, g("input_proj.bias"))
    _pad4(chunks, lin(g("posenc.Wr.weight")))                                   # [2][48]
    for i in range(LG_LAYERS):
        p = f"transformers.{i}."
        w, b = g(p + "self_attn.Wqkv.weight"), g(p + "self_attn.Wqkv.bias")
        perm = np.concatenate([np.arange(LG_DIM) * 3 + c for c in range(3)])
        _pad4(chunks, lin(w[perm]))
        _pad4(chunks, b[perm])
        _pad4(chunks, lin(g(p + "self_attn.out_proj.weight")))
        _pad4(chunks, g(p + "self_attn.out_proj.bias"))
        for blk in ("self_attn", "cross_attn"):
            if blk == "cross_attn":
                _pad4(chunks, lin(np.concatenate([g(p + "cross_attn.to_qk.weight"), g(p + "cross_attn.to_v.weight")])))
                _pad4(chunks, np.concatenate([g(p + "cross_attn.to_qk.bias"), g(p + "cross_attn.to_v.bias")]))
                _pad4(chunks, lin(g(p + "cross_attn.to_out.weight")))
                _pad4(chunks, g(p + "cross_attn.to_out.bias"))
            q = p + blk + ".ffn."
            for name in ("0.weight", "0.bias", "1.weight", "1.bias", "3.weight", "3.bias"):
                a = g(q + name)
                _pad4(chunks, lin(a) if a.ndim == 2 else a)
    for i in range(LG_LAYERS):
        p = f"log_assignment.{i}."
        _pad4(chunks, lin(g(p + "final_proj.weight")))
        _pad4(chunks, g(p + "final_proj.bias"))
        _pad4(chunks, g(p + "matchability.weight"))
        _pad4(chunks, g(p + "matchability.bias"))
    return np.ascontiguousarray(np.concatenate(chunks), dtype=np.float32)


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
