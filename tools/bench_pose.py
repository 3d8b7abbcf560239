#!/usr/bin/env python
"""Calibrated relative pose of a list of matched pairs: (a) one geometry.estimate_relative_pose_batch call (five-point RANSAC +
cheirality on the GPU, per-pair intrinsics), (b) the per-pair evalharness.estimate_pose_gpu (8-point essential RANSAC on the
GPU, host recover_pose), (c) the evalharness.estimate_pose_opencv loop spread over the host's threads.

Workload: 1 500 seeded synthetic calibrated pairs (tests/pose_ref.py calibrated_scene: random R, t, focal lengths 600-1200 px
per camera, 0.5 px noise, uniform outliers), n drawn from 256-4096 and inlier fractions from 0.3-0.8, at 1 px.  Each arm
reports AUC@5/10/20 of max(R, t) angular error against ground truth (evalharness.compute_maa) and its wall time, a host clock
around the whole arm ending in a device synchronise (inputs start on the host, as the harness hands them over).  (a) runs once
as warm-up, then `--reps` times.  The card's name, power limit and max SM clock are read in the same run, with the
`-Xptxas -v` registers and spills of the new kernels from the build logs.

    python tools/bench_pose.py [--pairs 1500] [--reps 3] [--out FILE]     # prints one JSON result line
"""
import argparse
import json
import os
import re
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from accelerated_features_b200 import evalharness as eh  # noqa: E402
from accelerated_features_b200.geometry import estimate_relative_pose_batch  # noqa: E402
from tests import pose_ref as P  # noqa: E402
from tools.bench_pairs import card  # noqa: E402


def pairs(n_pairs, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_pairs):
        Ks = [np.array([[f, 0, 512], [0, f * rng.uniform(0.98, 1.02), 384], [0, 0, 1.0]]) for f in rng.uniform(600, 1200, 2)]
        R, t = P.random_pose(rng)
        n = int(rng.integers(256, 4097))
        p0, p1, _ = P.calibrated_scene(rng, n, Ks[0], Ks[1], R, t, inlier_frac=rng.uniform(0.3, 0.8), noise_px=0.5)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, t
        out.append((p0.astype(np.float32), p1.astype(np.float32), Ks[0], Ks[1], T))
    return out


def auc(rets, data):
    errs = []
    for ret, (_, _, _, _, T) in zip(rets, data):
        if ret is None:
            errs.append({"t_err": np.inf, "R_err": np.inf})
            continue
        te, re_ = eh.relative_pose_error(T, ret[0], ret[1])
        errs.append({"t_err": te, "R_err": re_})
    m = eh.compute_maa(errs)
    return {k: round(v, 4) for k, v in m.items() if k.startswith("auc")}


def arm_batch(data, thr, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    B = len(data)
    n = np.array([len(d[0]) for d in data], np.int32)
    p0 = np.zeros((B, n.max(), 2), np.float32)
    p1 = np.zeros_like(p0)
    for b, d in enumerate(data):
        p0[b, :n[b]], p1[b, :n[b]] = d[0], d[1]
    K0 = np.array([P.intrinsics4(d[2]) for d in data], np.float32)
    K1 = np.array([P.intrinsics4(d[3]) for d in data], np.float32)
    E, R, t, mask, n_inl, _ = estimate_relative_pose_batch(torch.from_numpy(p0).cuda(), torch.from_numpy(p1).cuda(), K0, K1,
                                                           torch.from_numpy(n).cuda(), thr, iters)
    R, t, n_inl = R.cpu().numpy().astype(np.float64), t.cpu().numpy().astype(np.float64), n_inl.cpu().numpy()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dt, [(R[b], t[b], None) if n_inl[b] >= 5 else None for b in range(B)]


def arm_loop(fn, data, thr, threads=1):
    """fn over the pairs, in order (threads=1) or spread over a pool of host threads (cv2 releases the GIL)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    args = [(d[0].astype(np.float64), d[1].astype(np.float64), d[2], d[3], thr) for d in data]
    if threads == 1:
        rets = [fn(*x) for x in args]
    else:
        with ThreadPoolExecutor(threads) as ex:
            rets = list(ex.map(lambda x: fn(*x), args))
    torch.cuda.synchronize()
    return time.perf_counter() - t0, rets


def kernel_resources():
    log = os.path.join(ROOT, "accelerated_features_b200", "build", "ransac.o.log")
    out = {}
    if not os.path.exists(log):
        return out
    txt = open(log).read()
    for m in re.finditer(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill "
                         r"loads.*?Used (\d+) registers", txt, re.S):
        name = m.group(1)
        if "RsEssential5" in name or "pose_kernel" in name or "five_point" in name:
            short = re.sub(r"_ZN2xf\d+(\w+?)(I.*|E.*)", r"\1", name) + (" <RsEssential5>" if "RsEssential5" in name else "")
            out[short] = {"registers": int(m.group(5)), "stack_bytes": int(m.group(2)), "spill_stores": int(m.group(3)),
                          "spill_loads": int(m.group(4))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1500)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--thr", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pose: needs a CUDA device")
    data = pairs(a.pairs)
    res = {"card": card(), "pairs": a.pairs, "thr_px": a.thr, "kernels": kernel_resources()}
    print("card", json.dumps(res["card"]), flush=True)
    arm_batch(data, a.thr, 1024)                                 # warm-up
    times = []
    for _ in range(a.reps):
        dt, rets = arm_batch(data, a.thr, 1024)
        times.append(dt)
    res["a_estimate_relative_pose_batch"] = {"s": [round(x, 4) for x in times], "iters": 1024, **auc(rets, data)}
    print("a", json.dumps(res["a_estimate_relative_pose_batch"]), flush=True)
    eh.estimate_pose_gpu(data[0][0].astype(np.float64), data[0][1].astype(np.float64), data[0][2], data[0][3], a.thr)
    dt, rets = arm_loop(eh.estimate_pose_gpu, data, a.thr)
    res["b_estimate_pose_gpu_loop"] = {"s": round(dt, 3), "iters": 8192, **auc(rets, data)}
    print("b", json.dumps(res["b_estimate_pose_gpu_loop"]), flush=True)
    import cv2
    dt, rets = arm_loop(eh.estimate_pose_opencv, data, a.thr, threads=os.cpu_count())
    res["c_estimate_pose_opencv_loop"] = {"s": round(dt, 3), "host_threads": os.cpu_count(), **auc(rets, data)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
