"""CPU restatement of LighterGlue inference (modules/lighterglue.py:12-27 configuration of LightGlue; xfeat.py:131-162), written
from the model's definition, in numpy at float32 or float64.

    k'   = (k - size/2) / (max(W, H)/2)                                   size = (W, H) per image
    x    = input_proj(desc)                                               64 -> 96
    p    = Wr k' (48);  cos(p), sin(p) each repeated twice -> 96          rotary encoding of the self blocks
    6 x  [ self block on each image ; cross block on the pair ]
         self:  q, k, v = Wqkv(x) interleaved (rows 3i, 3i+1, 3i+2); q, k rotated; m = out_proj(softmax(q k^T/sqrt(96)) v)
         cross: a = to_qk(x), v = to_v(x); m0 = to_out(softmax_rows(a0 a1^T/sqrt(96)) v1), m1 likewise with the transpose
         both:  x += ffn([x | m]),  ffn = Linear(192,192) . LayerNorm(192) . GELU(erf) . Linear(192,96)
    pruning after layers 0..4 for an image with more than `prune_min_points` points: keep sigmoid(matchability_l(x)) > 0.05
    assignment (layer 5): md = final_proj(x)/96^0.25, S = md0 md1^T,
         scores = logsoftmax_rows(S) + logsoftmax_cols(S) + logsigmoid(z0)_i + logsigmoid(z1)_j
         mutual row/column arg-max (first index on ties), mscore = exp(row max), valid = mutual & mscore > min_conf

`keep_sets` replays externally chosen pruning decisions (one boolean mask per pruned layer and image, over that image's points at
that layer) instead of the matchability test.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
from scipy.special import erf

N_LAYERS = 6
DIM = 96
KEEP_THRESHOLD = np.float32(1 - 0.95)       # width_confidence 0.95: keep sigmoid(z) > 1 - 0.95


def load_state(path: Optional[str] = None) -> Dict[str, np.ndarray]:
    """The matcher state staged by oracle/build_lighterglue.py (default) or any file weights.load_lighterglue_state reads."""
    if path is None:
        from oracle import build_lighterglue
        path = build_lighterglue.path()
    import sys
    import os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from accelerated_features_b200 import weights
    return {k: np.asarray(v, np.float32) for k, v in weights.load_lighterglue_state(path).items()}


def normalize_keypoints(k: np.ndarray, size, dt) -> np.ndarray:
    size = np.asarray(size, dt)
    return ((k.astype(dt) - size / 2) / (size.max() / 2)).astype(dt)


class _Model:
    def __init__(self, sd, dt):
        self.dt = dt
        self.sd = {k: v.astype(dt) for k, v in sd.items()}

    def lin(self, name, x):
        y = x @ self.sd[name + ".weight"].T
        b = self.sd.get(name + ".bias")
        return y if b is None else y + b

    def ffn(self, p, x):
        h = self.lin(p + ".0", x)
        mu = h.mean(-1, keepdims=True)
        var = ((h - mu) ** 2).mean(-1, keepdims=True)
        h = (h - mu) / np.sqrt(var + self.dt(1e-5)) * self.sd[p + ".1.weight"] + self.sd[p + ".1.bias"]
        h = (h * 0.5 * (1.0 + erf(h / np.sqrt(2.0)))).astype(self.dt)
        return self.lin(p + ".3", h)

    def attend(self, q, k, v):
        if len(k) == 0:
            return np.zeros((len(q), DIM), self.dt)
        s = (q @ k.T) / self.dt(np.sqrt(DIM))
        s = np.exp(s - s.max(1, keepdims=True))
        return ((s / s.sum(1, keepdims=True)) @ v).astype(self.dt)

    def self_block(self, i, x, enc):
        p = f"transformers.{i}.self_attn"
        qkv = self.lin(p + ".Wqkv", x)
        q, k, v = qkv[:, 0::3], qkv[:, 1::3], qkv[:, 2::3]
        cos, sin = enc

        def rot(t):
            r = np.empty_like(t)
            r[:, 0::2], r[:, 1::2] = -t[:, 1::2], t[:, 0::2]
            return t * cos + r * sin
        m = self.lin(p + ".out_proj", self.attend(rot(q), rot(k), v))
        return x + self.ffn(p + ".ffn", np.concatenate([x, m], 1))

    def cross_block(self, i, x0, x1):
        p = f"transformers.{i}.cross_attn"
        a0, a1 = self.lin(p + ".to_qk", x0), self.lin(p + ".to_qk", x1)
        v0, v1 = self.lin(p + ".to_v", x0), self.lin(p + ".to_v", x1)
        m0 = self.lin(p + ".to_out", self.attend(a0, a1, v1))
        m1 = self.lin(p + ".to_out", self.attend(a1, a0, v0))
        return (x0 + self.ffn(p + ".ffn", np.concatenate([x0, m0], 1)),
                x1 + self.ffn(p + ".ffn", np.concatenate([x1, m1], 1)))

    def matchability(self, i, x):
        return self.lin(f"log_assignment.{i}.matchability", x)[:, 0]


def _logsigmoid(z):
    return np.minimum(z, 0) - np.log1p(np.exp(-np.abs(z)))


def _logsoftmax(s, axis):
    m = s.max(axis, keepdims=True)
    return s - (m + np.log(np.exp(s - m).sum(axis, keepdims=True)))


def keep_rule(z: np.ndarray) -> np.ndarray:
    """Pruning keep mask from matchability logits: sigmoid(z) > 0.05, evaluated in float32 like the model."""
    z = np.asarray(z, np.float32)
    return (np.float32(1) / (np.float32(1) + np.exp(-z))) > KEEP_THRESHOLD


def match(sd, kpts0, desc0, size0, kpts1, desc1, size1, min_conf: float = 0.1, prune_min_points: Optional[int] = None,
          keep_sets: Optional[Sequence[Sequence[Optional[np.ndarray]]]] = None, dtype=np.float32,
          n_layers: int = N_LAYERS) -> Dict[str, object]:
    """One pair.  Returns idx0 (ascending), idx1, scores (float of `dtype`), and the diagnostics the parity tests use:
    'x' (the two final descriptor sets), 'ind' (surviving original indices per image), 'keep' (per pruned layer, per image: the
    keep mask or None), 'z' (matchability logits at each pruning step), 'row_max' / 'col_max' / 'row_gap' / 'col_gap' (assignment row
    and column maxima and top-2 gaps over the surviving points), 'mscore' (exp(row max)) and the mutual mask.  `n_layers` < 6 stops after
    that many layers and returns only 'x', 'ind', 'keep' and 'z'."""
    dt = np.dtype(dtype).type
    m = _Model(sd, dt)
    n0, n1 = len(kpts0), len(kpts1)
    out: Dict[str, object] = {"keep": [], "z": []}
    if n0 == 0 or n1 == 0:
        e = np.zeros(0, np.int64)
        out.update(idx0=e, idx1=e.copy(), scores=np.zeros(0, dt))
        return out
    xs = [m.lin("input_proj", np.asarray(d, dt)) for d in (desc0, desc1)]
    encs = []
    for k, s in ((kpts0, size0), (kpts1, size1)):
        p = normalize_keypoints(np.asarray(k), s, dt) @ m.sd["posenc.Wr.weight"].T
        p = np.repeat(p, 2, axis=1)
        encs.append((np.cos(p), np.sin(p)))
    inds = [np.arange(n0), np.arange(n1)]
    for i in range(n_layers):
        xs = [m.self_block(i, x, e) for x, e in zip(xs, encs)]
        xs = list(m.cross_block(i, xs[0], xs[1]))
        if i == N_LAYERS - 1:
            break
        keeps, zs = [], []
        for s in range(2):
            replay = None if keep_sets is None else keep_sets[i][s]
            pruned = replay is not None or (prune_min_points is not None and len(xs[s]) > prune_min_points)
            if not pruned:
                keeps.append(None)
                zs.append(None)
                continue
            z = m.matchability(i, xs[s])
            keep = np.asarray(replay, bool) if replay is not None else keep_rule(z)
            keeps.append(keep)
            zs.append(z)
            xs[s] = xs[s][keep]
            encs[s] = (encs[s][0][keep], encs[s][1][keep])
            inds[s] = inds[s][keep]
        out["keep"].append(keeps)
        out["z"].append(zs)
    out["x"], out["ind"] = xs, inds
    if n_layers < N_LAYERS:
        return out
    if len(xs[0]) == 0 or len(xs[1]) == 0:
        e = np.zeros(0, np.int64)
        out.update(idx0=e, idx1=e.copy(), scores=np.zeros(0, dt))
        return out
    md = [m.lin("log_assignment.5.final_proj", x) / dt(DIM ** 0.25) for x in xs]
    z0, z1 = m.matchability(5, xs[0]), m.matchability(5, xs[1])
    S = md[0] @ md[1].T
    sc = _logsoftmax(S, 1) + _logsoftmax(S, 0) + (_logsigmoid(z0)[:, None] + _logsigmoid(z1)[None, :])
    m0, m1 = sc.argmax(1), sc.argmax(0)                 # numpy: first index on ties
    mutual = m1[m0] == np.arange(len(m0))
    rmax = sc.max(1)
    mscore = np.exp(rmax)
    valid = mutual & (mscore > dt(min_conf))
    i0 = np.nonzero(valid)[0]

    def gap(a, axis):
        if a.shape[axis] < 2:
            return np.full(a.shape[1 - axis], np.inf)
        t = -np.partition(-a, 1, axis=axis)
        return (t.take(0, axis) - t.take(1, axis))
    out.update(idx0=inds[0][i0].astype(np.int64), idx1=inds[1][m0[i0]].astype(np.int64), scores=mscore[i0].astype(dt),
               row_max=rmax, row_arg=m0, col_max=sc.max(0), col_arg=m1, row_gap=gap(sc, 1), col_gap=gap(sc, 0), mscore=mscore,
               mutual=mutual)
    return out
