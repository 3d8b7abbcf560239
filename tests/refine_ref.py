"""Float64 restatement of XFeat.refine_matches (xfeat.py:306-325) for a whole batch, as xfeat_refine / xfeat_refine_pairs
compute it: pair p reads desc0 / kpts0 / scales0 of image i (stride n_max) and desc1 / kpts1 of image j (stride n1_max), with
(i, j) = pairs[p], or (p, p) without a pair table.  Its live rows are the first clamp(n_matches[p], 0, n_max) coarse matches.

Per live row: logits = the float64 fine matcher (split_ref.reference_chain), conf = max softmax(3 logits), offset = E[(x - 4, y - 4)]
under that softmax (x the fast axis), xy0 = kp0 + offset * scale0; the row is kept when conf > fine_conf, in coarse-row order.
The confidences of every live row are returned too, so that tests can tell which rows sit too close to a threshold to be decided.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from tests import split_ref as sr

# The kernel's confidence comes from logits within FINE_MATCHER_TOL of float64 (test_fine_matcher_depth).  conf = 1 / sum_k
# exp(3 (l_k - l_max)): an error e on every logit moves each exponent by at most 6 e, so conf moves by a factor within
# exp(+-6 e).  CONF_FP32 covers the fp32 soft-max itself (64 expf, a 64-term sum and one division: < 80 u relative).
CONF_FP32 = 80 * 2.0 ** -24


def conf_band(conf: torch.Tensor, logit_tol: float = sr.FINE_MATCHER_TOL) -> torch.Tensor:
    """Largest |conf_kernel - conf_float64| the logit tolerance allows, per row."""
    return conf * (math.expm1(6 * logit_tol) + CONF_FP32)


def refine_ref(sd, desc0, desc1, kpts0, kpts1, scales0, idx0, idx1, n_matches, fine_conf: float,
               pairs: Optional[torch.Tensor] = None) -> List[dict]:
    """desc0 (I0, n_max, 64), desc1 (I1, n1_max, 64), kpts0 (I0, n_max, 2), kpts1 (I1, n1_max, 2), scales0 (I0, n_max),
    idx0 / idx1 (P, n_max) int64, n_matches (P) int, pairs (P, 2) or None.  Tensors on one device (the fine matcher runs there).

    Returns one dict per pair: n (live rows), conf (n) float64, xy0 (n, 2) float64, xy1 (n, 2) float32 (kpts1 as read),
    keep (n) bool, rows (kept row indices, increasing)."""
    P, n_max = idx0.shape
    dev = desc0.device
    cnt = [max(0, min(int(c), n_max)) for c in n_matches.tolist()]
    pr = pairs.tolist() if pairs is not None else [(p, p) for p in range(P)]
    xs, meta = [], []
    for p in range(P):
        i, j = pr[p]
        a, b = idx0[p, :cnt[p]].to(dev), idx1[p, :cnt[p]].to(dev)
        xs.append(torch.cat([desc0[i, a], desc1[j, b]], 1).double())
        meta.append((kpts0[i, a].double(), scales0[i, a].double(), kpts1[j, b].float()))
    x = torch.cat(xs, 0) if xs else torch.zeros(0, 128, dtype=torch.float64, device=dev)
    logits = sr.reference_chain(sd, sr.FINE_MATCHER, x) if len(x) else torch.zeros(0, 64, dtype=torch.float64, device=dev)
    p64 = torch.softmax(3 * logits, -1)
    conf_all = p64.max(-1)[0]
    ar = torch.arange(64, device=dev)
    gx, gy = (ar % 8 - 4).double(), (ar // 8 - 4).double()
    off_all = torch.stack([(p64 * gx).sum(-1), (p64 * gy).sum(-1)], -1)
    out, r0 = [], 0
    for p in range(P):
        n = cnt[p]
        conf, off = conf_all[r0:r0 + n], off_all[r0:r0 + n]
        r0 += n
        k0, s0, k1 = meta[p]
        keep = conf > fine_conf
        out.append(dict(n=n, conf=conf, xy0=k0 + off * s0[:, None], xy1=k1, keep=keep,
                        rows=torch.nonzero(keep)[:, 0], logits=logits[r0 - n:r0]))
    return out

