#!/usr/bin/env python
"""Generate tests/golden/ransac_pinned.npz: the exact outputs of the three RANSAC estimators on a seeded corpus.

Run on a GPU with the library built:

    python tools/make_golden_ransac.py [out.npz]

The float64 reference tests (tests/test_gpu_ransac_models.py) check tolerances and properties; a change in which samples are
drawn (a hash constant, a hypothesis id, the pair id) passes them all and still changes every user's masks.  This fixture pins
the outputs bit for bit (tests/test_gpu_ransac_pinned.py).  It stores the inputs of every call next to its outputs, so the
test replays the calls without regenerating anything.

Corpus, per model (homography "h", essential "e", fundamental "f"):
  * "mixed": one batch with garbage past each count -- counts 0, 3, 4, 7, 8 and N_OVERFLOW on real scene points, a noise-free
    scene, two scenes with 0.5 px noise, and the degenerate scenes of test_gpu_ransac_models.py (identical and collinear
    points; for E and F a plane and a pure rotation);
    run at iters 1, 255, 256, 257, 700, 1024 and 2049 (the rounding of blocks per pair, hypotheses per warp and rounds),
    each with two seeds, one above 2^31; F also with a permutation of the pair ids;
  * "big": one pair of 8192 correspondences at n_max 8192.
Plus the 7-point solver hook (xfeat_debug_seven_point) on random samples and the rank-deficient ones.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from accelerated_features_b200 import _lib  # noqa: E402
from tests import ransac_ref as ref  # noqa: E402
from tests import test_gpu_ransac_models as M  # noqa: E402
from tests.test_gpu_ransac_pinned import run  # noqa: E402

F32 = np.float32
ITERS = [1, 255, 256, 257, 700, 1024, 2049]
SEEDS = [7, 0x9E3779B1]                       # the second is above 2^31
THR = {"h": 3.0, "e": 1.5 / 600.0, "f": 1.0}
SHORT_COUNTS = [0, 3, 4, 7, 8, _lib.N_OVERFLOW]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "ransac_pinned.npz")


def e_degenerate(rng):
    ident = (np.full((100, 2), [0.1, -0.2], F32), np.full((100, 2), [0.15, -0.18], F32))
    R, t = ref.rodrigues([0.02, 0.1, 0.0]), np.array([0.4, 0.1, 0.05])
    xy = rng.uniform(-0.5, 0.5, (400, 2))
    X0 = np.concatenate([xy, np.ones((400, 1))], 1) * (4.0 / (1 - 0.3 * xy[:, 0]))[:, None]     # the plane Z = 4 + 0.3 X
    X1 = X0 @ R.T + t
    X1r = X0 @ ref.rodrigues([0.05, -0.1, 0.02]).T
    x0 = (X0[:, :2] / X0[:, 2:]).astype(F32)
    return [ident, (x0, (X1[:, :2] / X1[:, 2:]).astype(F32)), (x0, (X1r[:, :2] / X1r[:, 2:]).astype(F32))]


def scenes(kind, rng):
    """The (p0, p1) scenes of the mixed batch and of the big pair, and the mixed batch's n_max."""
    if kind == "h":
        W, H = 640, 480
        mk = lambda motion, n, w, noise: M.h_scene(rng, W, H, M.motion_h(motion, W, H), n, w, THR[kind], noise)[:2]  # noqa: E731
        clean, noisy = mk("perspective", 300, 0.6, 0.0), [mk("rot90", 380, 0.5, 0.5), mk("scale3", 200, 0.8, 0.5)]
        degen = [(a, c) for _, a, c in M.h_degenerate_scenes(rng)]
        big = mk("perspective", 8192, 0.5, 0.5)
    elif kind == "e":
        f, W, H = M.CAMS[0]
        mk = lambda motion, n, w, noise: M.e_scene(rng, f, W, H, *M.E_MOTIONS[motion], n, w, THR[kind], noise)[:2]  # noqa: E731
        clean, noisy = mk("sideways", 300, 0.6, 0.0), [mk("rot30", 380, 0.5, 0.5), mk("forward", 200, 0.8, 0.5)]
        degen = e_degenerate(rng)
        big = mk("sideways", 8192, 0.5, 0.5)
    else:
        mk = lambda pair, motion, n, w, noise: M.f_scene(rng, pair, motion, n, w, THR[kind], noise)[:2]  # noqa: E731
        clean = mk(M.SAME_PAIRS[1], "general", 300, 0.6, 0.0)
        noisy = [mk(M.MIXED_PAIRS[1], "sideways", 380, 0.5, 0.5), mk(M.SAME_PAIRS[2], "forward", 200, 0.8, 0.5)]
        degen = [(a, c) for _, a, c in M.f_degenerate_scenes(rng)]
        big = mk(M.SAME_PAIRS[1], "general", 8192, 0.5, 0.5)
    return [clean] * len(SHORT_COUNTS) + [clean] + noisy + degen, big, 400


def main(path):
    rng = np.random.default_rng(2024)
    arrays, n_calls = {}, 0

    def call(kind, name, iters, seed, ids=None):
        nonlocal n_calls
        p0, p1, cnt = arrays[f"{kind}_{name}.p0"], arrays[f"{kind}_{name}.p1"], arrays[f"{kind}_{name}.cnt"]
        model, mask, n = run(kind, p0, p1, cnt, THR[kind], iters, seed, ids)
        pre = f"call{n_calls:03d}."
        arrays.update({pre + "kind": np.array(kind), pre + "set": np.array(name), pre + "thr": np.float64(THR[kind]),
                       pre + "iters": np.int64(iters), pre + "seed": np.int64(seed), pre + "model": model,
                       pre + "mask": np.packbits(mask, axis=1), pre + "n_inliers": n})
        if ids is not None:
            arrays[pre + "pair_ids"] = np.asarray(ids, np.int32)
        n_calls += 1
        print(f"{kind} {name:5s} iters {iters:5d} seed {seed:#x}{'' if ids is None else ' ids':4s} n_inliers {n.tolist()}")

    for kind in ("h", "e", "f"):
        mixed, big, n_max = scenes(kind, rng)
        p0, p1, cnt = M.pack(rng, mixed, n_max)
        cnt[:len(SHORT_COUNTS)] = SHORT_COUNTS
        arrays.update({f"{kind}_mixed.p0": p0, f"{kind}_mixed.p1": p1, f"{kind}_mixed.cnt": cnt})
        arrays.update({f"{kind}_big.p0": big[0][None], f"{kind}_big.p1": big[1][None],
                       f"{kind}_big.cnt": np.array([len(big[0])], np.int32)})
        ids = rng.permutation(len(cnt)).astype(np.int32)
        for seed in SEEDS:
            for iters in ITERS:
                call(kind, "mixed", iters, seed)
                if kind == "f":
                    call(kind, "mixed", iters, seed, ids)
        call(kind, "big", 1024, SEEDS[0])

    # 7-point solver hook: random normalised samples, then seven identical points and points collinear in both images
    t = np.linspace(-1, 1, 7)
    samples = np.concatenate([rng.normal(0, 1, (300, 7, 4)).astype(F32),
                              np.tile(np.array([0.3, -0.2, 0.5, 0.1], F32), (1, 7, 1)),
                              np.stack([t, 0.5 * t + 0.1, 0.8 * t - 0.3, -0.2 * t + 0.4], 1)[None].astype(F32)])
    Fc, nc = M.run_seven_point(samples)
    arrays.update({"seven.samples": samples, "seven.F": Fc.reshape(len(samples), 3, 9), "seven.count": nc})

    arrays["n_calls"] = np.int64(n_calls)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez_compressed(path, **arrays)
    print(f"{path}: {os.path.getsize(path) / 1e6:.2f} MB, {n_calls} calls, {torch.cuda.get_device_name()}")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
