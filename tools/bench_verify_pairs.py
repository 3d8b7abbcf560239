#!/usr/bin/env python
"""Fundamental-matrix verification of pair lists on the GPU (find_fundamental_batch, XFeat.match_xfeat_verified_pairs) against
the per-pair host loop users run today, cv2.findFundamentalMat(p0, p1, cv2.USAC_MAGSAC, thr, 0.999, 10000).

Workloads:
  a  1 500 seeded synthetic two-view correspondence sets (random 3-D points, random R, t and focal length, 0.5 px noise,
     uniform outliers), n drawn from 256-4096 and inlier fractions from 0.3-0.8, at thr 1.5 px.  GPU: one find_fundamental_batch
     call over the whole list on device tensors (CUDA events), at 2048 and 8192 samples per pair.  CPU: the cv2 loop (one pass).
     Also the agreement statistics of tests/test_gpu_fundamental.py per set: inlier agreement with cv2, inlier-count difference,
     true-inlier recall, false-inlier rate and the mean Sampson error of the true inliers under each F.
  b  exhaustive matching of 64 VGA images (2016 pairs, top_k 4096, the images of tools/bench_pairs.py workload b) at 3 px:
     match_xfeat_verified_pairs against match_xfeat_pairs followed by the cv2 loop.  The GPU arms alternate; the cv2 loop runs once.
Times of the GPU arms are CUDA events around the whole call (which ends with the results on the host).  The card's name and power
limit, the CPU model and cv2's thread count are read in the same run.

    python tools/bench_verify_pairs.py [--reps 5] [--out FILE]     # prints one JSON result line; --out also writes it to FILE
"""
import argparse
import json
import os
import platform
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from accelerated_features_b200 import XFeat  # noqa: E402
from accelerated_features_b200.geometry import find_fundamental_batch  # noqa: E402
from tools.bench_pairs import card, synth, timed  # noqa: E402

TOPK = 4096


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor()


def scene(rng, n, w):
    """As tests/test_gpu_fundamental.py synth_scene: a non-planar two-view scene in pixels."""
    R, _ = cv2.Rodrigues(rng.uniform(-0.3, 0.3, 3))
    t = rng.uniform(-1, 1, 3)
    t /= np.linalg.norm(t)
    f = rng.uniform(450, 900)
    K = np.array([[f, 0, 320], [0, f, 240], [0, 0, 1.0]])
    X0 = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 9, n)], 1)
    X1 = X0 @ R.T + t
    p0 = ((X0 / X0[:, 2:]) @ K.T)[:, :2] + rng.normal(0, 0.5, (n, 2))
    p1 = ((X1 / X1[:, 2:]) @ K.T)[:, :2] + rng.normal(0, 0.5, (n, 2))
    inl = rng.uniform(size=n) < w
    p1[~inl] = np.stack([rng.uniform(0, 640, (~inl).sum()), rng.uniform(0, 480, (~inl).sum())], 1)
    return p0.astype(np.float32), p1.astype(np.float32), inl


def sampson(F, p0, p1):
    F = np.asarray(F, np.float64)
    h0 = np.concatenate([p0.astype(np.float64), np.ones((len(p0), 1))], 1)
    h1 = np.concatenate([p1.astype(np.float64), np.ones((len(p1), 1))], 1)
    a, b = h0 @ F.T, h1 @ F
    return np.abs((h1 * a).sum(1)) / np.sqrt(a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2)


def cv2_loop(p0s, p1s, thr):
    out = []
    t = time.perf_counter()
    for a, c in zip(p0s, p1s):
        if len(a) < 8:
            out.append((None, np.zeros(len(a), bool)))
            continue
        F, m = cv2.findFundamentalMat(a, c, cv2.USAC_MAGSAC, thr, 0.999, 10000)
        out.append((None if F is None else F[:3], np.zeros(len(a), bool) if m is None else m.ravel() > 0))
    return time.perf_counter() - t, out


def stats(xs):
    xs = np.asarray(xs, np.float64)
    return {"min": float(xs.min()), "p5": float(np.percentile(xs, 5)), "median": float(np.median(xs)), "max": float(xs.max())}


def workload_a(reps, n_sets=1500, thr=1.5):
    rng = np.random.default_rng(0)
    ns = rng.integers(256, 4097, n_sets)
    ws = rng.uniform(0.3, 0.8, n_sets)
    sets = [scene(rng, int(n), float(w)) for n, w in zip(ns, ws)]
    p0 = np.zeros((n_sets, int(ns.max()), 2), np.float32)
    p1 = np.zeros_like(p0)
    for b, (a, c, _) in enumerate(sets):
        p0[b, :len(a)], p1[b, :len(c)] = a, c
    d0, d1, dc = torch.from_numpy(p0).cuda(), torch.from_numpy(p1).cuda(), torch.from_numpy(ns.astype(np.int32)).cuda()
    t_cv, cv = cv2_loop([s[0] for s in sets], [s[1] for s in sets], thr)
    res = {"sets": n_sets, "thr_px": thr, "matches_total": int(ns.sum()), "cv2_loop_s": t_cv, "cv2_threads": cv2.getNumThreads()}
    for iters in (2048, 8192):
        def call():
            F, m, n = find_fundamental_batch(d0, d1, dc, thr=thr, iters=iters, seed=0)
            return F.cpu().numpy(), m.cpu().numpy(), n.cpu().numpy()
        call()
        times = [timed(call)[0] for _ in range(reps)]
        F, m, n = call()
        agree, dcount, rec, false, e_gpu, e_cv = [], [], [], [], [], []
        for b, (a, c, inl) in enumerate(sets):
            k = len(a)
            g, mc = m[b, :k], cv[b][1]
            agree.append((g == mc).mean())
            dcount.append(abs(int(n[b]) - int(mc.sum())) / k)
            rec.append(g[inl].mean())
            false.append(g[~inl].mean() if (~inl).any() else 0.0)
            e_gpu.append(sampson(F[b], a[inl], c[inl]).mean())
            e_cv.append(sampson(cv[b][0], a[inl], c[inl]).mean() if cv[b][0] is not None else np.inf)
        e_gpu, e_cv = np.asarray(e_gpu), np.asarray(e_cv)
        res[f"gpu_iters{iters}"] = {
            "median_s": float(np.median(times)), "min_s": float(np.min(times)), "max_s": float(np.max(times)),
            "agreement_with_cv2": stats(agree), "sets_agreement_below_0.97": int((np.asarray(agree) < 0.97).sum()),
            "inlier_count_diff_frac": stats(dcount), "true_inlier_recall": stats(rec), "false_inlier_rate": stats(false),
            "sampson_true_inliers_gpu_minus_cv2_px": stats(e_gpu - e_cv),
            "sets_sampson_worse_than_cv2_by_0.1px": int((e_gpu > e_cv + 0.1).sum())}
        print("a", iters, json.dumps(res[f"gpu_iters{iters}"]), flush=True)
    print("a cv2", t_cv, flush=True)
    return res


def workload_b(xf, reps, thr=3.0):
    with np.load(os.path.join(ROOT, "tests", "golden", "inputs_assets_vga.npz")) as z:
        ref, tgt = z["ref"], z["tgt"]
    rng = np.random.default_rng(0)
    vga = [synth(ref if k % 2 == 0 else tgt, 480, 640, rng) for k in range(64)]
    pairs = np.array([(i, j) for i in range(64) for j in range(i + 1, 64)], np.int64)
    arms = {"verified_pairs": lambda: xf.match_xfeat_verified_pairs(vga, pairs, top_k=TOPK, ransac_thr=thr),
            "pairs_only": lambda: xf.match_xfeat_pairs(vga, pairs, top_k=TOPK)}
    outs = {k: f() for k, f in arms.items()}
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            times[k].append(timed(f)[0])
    ver, mat = outs["verified_pairs"], outs["pairs_only"]
    same = all(np.array_equal(v["mkpts0"], m[0]) and np.array_equal(v["mkpts1"], m[1]) for v, m in zip(ver, mat))
    t_cv, cv = cv2_loop([m[0] for m in mat], [m[1] for m in mat], thr)
    agree = [(v["inliers"] == c[1]).mean() for v, c in zip(ver, cv) if len(v["inliers"])]
    res = {k: {"median_s": float(np.median(v)), "min_s": float(np.min(v)), "max_s": float(np.max(v))} for k, v in times.items()}
    res.update({"pairs": len(pairs), "thr_px": thr, "matches_total": int(sum(len(m[0]) for m in mat)), "cv2_loop_s": t_cv,
                "pairs_then_cv2_s": res["pairs_only"]["median_s"] + t_cv, "matches_identical": same,
                "agreement_with_cv2": stats(agree), "inliers_total_gpu": int(sum(v["n_inliers"] for v in ver)),
                "inliers_total_cv2": int(sum(c[1].sum() for c in cv))})
    print("b", json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="ab")
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_verify_pairs needs a GPU")
    result = {"card": card(), "cpu": cpu_model(), "cpu_count": os.cpu_count(), "cv2": cv2.__version__,
              "cv2_threads": cv2.getNumThreads(), "reps": args.reps}
    t0 = time.time()
    if "a" in args.only:
        result["a_synthetic1500"] = workload_a(args.reps)
    if "b" in args.only:
        result["b_exhaustive64"] = workload_b(XFeat(), args.reps)
    result["wall_s"] = time.time() - t0
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
