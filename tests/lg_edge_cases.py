"""Edge-case inputs for the LighterGlue stage tests (test_lighterglue_edges_ref.py on the CPU, test_gpu_lighterglue_edges.py on the
H100), and the plain-numpy rules those tests hold the kernels to.  numpy only.

Every case is a subset of the 4096-point asset pair (tests/golden/lg_assets_4096.npz): image-0 points on side 0, image-1 points on
side 1, so the activations are those of real features.  The counts sit where the kernels' tiling can go wrong:

    (1, 1, 1), (1, 700, 700), (700, 1, 700), (2, 3, 64)      a single point or a handful against a 64-row tile
    (63, 65, 65), (64, 64, 64), (65, 63, 130)                one row either side of a tile boundary
    (700, 1900, 1937)                                        n_max = 17 mod 64: the linears' 64-row tiles straddle two images
    (1536, 1537, 1600)                                       either side of the default pruning threshold (1536)

and the image geometry varies with them: the asset size (800 x 600), portrait (600 x 800, x and y swapped, so max(W, H) = H), a
different size on each side, and keypoints on the exact image corners plus two outside the frame (the model normalises by the
image size without clipping).
"""
import os
from typing import List, NamedTuple, Tuple

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lg_assets_4096.npz")
ASSET_SIZE = (800, 600)


class Case(NamedTuple):
    name: str
    n0: int
    n1: int
    n_max: int
    geometry: str            # "asset" | "portrait" | "mixed" | "corners"


CASES = [
    Case("1x1", 1, 1, 1, "asset"),
    Case("1x700", 1, 700, 700, "portrait"),
    Case("700x1", 700, 1, 700, "mixed"),
    Case("2x3", 2, 3, 64, "corners"),
    Case("63x65", 63, 65, 65, "corners"),
    Case("64x64", 64, 64, 64, "portrait"),
    Case("65x63", 65, 63, 130, "mixed"),
    Case("700x1900", 700, 1900, 1937, "corners"),
    Case("1536x1537", 1536, 1537, 1600, "asset"),
]
CASE_IDS = [c.name for c in CASES]
BY_NAME = {c.name: c for c in CASES}
N_MAX_ALL = max(c.n_max for c in CASES)       # 1937: the whole table as one batch

# Per-case bounds where a shape needs more than the shared LAYER_TOL / SCORE_TOL (tests/test_lighterglue_oracle.py); keyed
# (case, 'layer1' | 'layer6' | 'score').  test_lighterglue_edges_ref.py proves each is >= 5x the float32 oracle's error.
# 1536 x 1537 after six layers: the float32 oracle is 9.1e-3 off float64 (2.7x the 1024-point pair's 3.4e-3), so 2e-2 is only
# 2.2x; 5e-2 is 5.5x.
CASE_TOL = {("1536x1537", "layer6"): 5e-2}

_assets = None


def assets():
    """The 4096-point asset pair; the stored int8 descriptors q decode to q / 128 (exact in fp32)."""
    global _assets
    if _assets is None:
        with np.load(GOLDEN) as z:
            _assets = {k: z[k] for k in z.files}
        for s in range(2):
            _assets[f"desc{s}"] = _assets.pop(f"desc{s}_q").astype(np.float32) / np.float32(128)
    return _assets


def _side(case: Case, s: int, n: int) -> Tuple[np.ndarray, np.ndarray, Tuple[float, float]]:
    g = assets()
    rs = np.random.RandomState(1000 * case.n0 + case.n1 + 7 * s)
    sel = np.sort(rs.choice(len(g[f"kpts{s}"]), n, replace=False))
    k = g[f"kpts{s}"][sel].copy()
    d = g[f"desc{s}"][sel].copy()
    W, H = ASSET_SIZE
    if case.geometry == "portrait":
        k = k[:, ::-1].copy()
        W, H = H, W
    elif case.geometry == "mixed" and s == 1:
        W, H = 1000, 750
    elif case.geometry == "corners":
        special = np.array([[0, 0], [W, H], [W, 0], [0, H], [-3.5, 20.0], [W + 11.0, H + 2.25]], np.float32)
        m = min(n, len(special))
        k[:m] = special[(np.arange(m) + s) % len(special)]
    return k.astype(np.float32), d, (float(W), float(H))


def case_args(case) -> tuple:
    """(kpts0, desc0, size0, kpts1, desc1, size1) in the oracle's argument order."""
    case = BY_NAME[case] if isinstance(case, str) else case
    k0, d0, s0 = _side(case, 0, case.n0)
    k1, d1, s1 = _side(case, 1, case.n1)
    return k0, d0, s0, k1, d1, s1


def pad(a: np.ndarray, n_max: int, fill=0.0) -> np.ndarray:
    """Rows of `a` followed by n_max - len(a) rows of `fill` (0 or NaN), float32 unless `a` is float64."""
    a = np.asarray(a)
    out = np.full((n_max,) + a.shape[1:], fill, np.float64 if a.dtype == np.float64 else np.float32)
    out[:len(a)] = a
    return out


def batch_arrays(pairs: List[tuple], n_max: int, fill=0.0) -> tuple:
    """Pairs in the oracle's argument order -> host arrays in match_lighterglue_batch order: kpts0 (B, n_max, 2), desc0
    (B, n_max, 64), n0 (B) int32, size0 (B, 2), then the same for side 1.  Rows past a count hold `fill`."""
    out = []
    for s in range(2):
        k = np.stack([pad(p[3 * s], n_max, fill).reshape(n_max, 2) for p in pairs])
        d = np.stack([pad(p[3 * s + 1], n_max, fill).reshape(n_max, 64) for p in pairs])
        n = np.array([len(p[3 * s]) for p in pairs], np.int32)
        sz = np.array([p[3 * s + 2] for p in pairs], np.float32)
        out += [k, d, n, sz]
    return tuple(out)


def finalize_rule(best, arg, ind, cnt, min_conf) -> List[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
    """The match filter in plain numpy.  best / arg / ind (2, B, n_max) or (2, n_max): side 0 the row maxima and arg-maxima of the
    log-assignment, side 1 the column arg-maxima, ind the original index of each surviving point; cnt (2, B) or (2,).  Row i of
    pair b is a match when it is mutual (arg[1][arg[0][i]] == i) and exp(best) > min_conf, both in best's precision; matches come
    in ascending i, mapped through ind.  Returns per pair (idx0 int64, idx1 int64, scores)."""
    best, arg, ind, cnt = (np.asarray(a) for a in (best, arg, ind, cnt))
    if cnt.ndim == 1:
        best, arg, ind, cnt = best[:, None], arg[:, None], ind[:, None], cnt[:, None]
    out = []
    for b in range(cnt.shape[1]):
        n0, n1 = int(cnt[0, b]), int(cnt[1, b])
        if n0 == 0 or n1 == 0:
            e = np.zeros(0, np.int64)
            out.append((e, e.copy(), np.zeros(0, best.dtype)))
            continue
        a0, a1 = arg[0, b, :n0], arg[1, b, :n1]
        sc = np.exp(best[0, b, :n0])
        ok = (a1[a0] == np.arange(n0)) & (sc > best.dtype.type(min_conf))
        i = np.nonzero(ok)[0]
        out.append((ind[0, b, i].astype(np.int64), ind[1, b, a0[i]].astype(np.int64), sc[i]))
    return out
