#!/usr/bin/env python
"""Per-frame latency of reference tracking (realtime_demo.py's step: match the camera frame against a cached reference at
min_cossim 0.82, then a USAC_MAGSAC homography at 4 px with 700 iterations), on one GPU.

Routes, each timed on the host from numpy uint8 frames in to results on the host:
  a  XFeat.tracker: one CUDA graph replay per step, reference extracted once.
  b  match_xfeat_verified_batch(ref, frame, min_cossim=0.82, ransac_thr=4.0, iters=700): re-extracts the reference every step.
  c  the demo's eager sequence: detectAndCompute(frame), match(ref_desc, desc, 0.82) and find_homography_batch on the matched
     keypoints, the reference's descriptors cached once.
Workloads: one 640x480 camera at top_k 3000 (the demo's --max_kpts) and 4096, and four 640x480 cameras per step at 4096
(multi-camera: one tracker call of B = 4; route c runs the demo's step once per camera).  Frames are seeded perspective warps
of the VGA asset; each route runs --frames steps after --warmup, in rounds of 50 steps alternating the routes.
Also reported: the device time of the replay alone (CUDA events around the graph replay, without the host copies in and out),
and whether routes a and b return identical matches, inlier masks and H on every frame of the sequence.  The card's name,
power limit and maximum SM clock are read in the same run.

    python tools/bench_tracker.py [--frames 500] [--warmup 50] [--out FILE]   # prints one JSON result line
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from accelerated_features_b200 import XFeat  # noqa: E402
from accelerated_features_b200.geometry import find_homography_batch  # noqa: E402

MIN_COSSIM, THR, ITERS = 0.82, 4.0, 700


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi (name, power.limit, clocks.max.sm)": q[0] if q else None}


def make_frames(img, n, seed=0):
    import cv2
    rng = np.random.default_rng(seed)
    h, w = img.shape[:2]
    src = np.float32([[0, 0], [w, 0], [w, h], [0, h]])
    return [cv2.warpPerspective(img, cv2.getPerspectiveTransform(src, (src + rng.uniform(-60, 60, src.shape)).astype(np.float32)),
                                (w, h), flags=cv2.INTER_LINEAR) for _ in range(n)]


def demo_step(xf, ref_desc, ref_kpts, frames, top_k):
    """realtime_demo.py's per-frame sequence, one camera after the other."""
    out = []
    for f in frames:
        cur = xf.detectAndCompute(f, top_k=top_k)[0]
        i0, i1 = xf.match(ref_desc, cur["descriptors"], MIN_COSSIM)
        p0, p1 = ref_kpts[i0][None], cur["keypoints"][i1][None]
        H, mask, n_inl = find_homography_batch(p0, p1, None, THR, ITERS) if len(i0) else (None, None, None)
        out.append((p0[0].cpu().numpy(), p1[0].cpu().numpy(), None if H is None else H[0].cpu().numpy(),
                    None if mask is None else mask[0].cpu().numpy()))
    return out


def stats(ts):
    ms = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90)),
            "n": len(ms)}


def replay_device_ms(tr, reps=200):
    """CUDA events around the graph replay alone (the one graph the tracker captured for this workload)."""
    (r,) = [r for r in tr._routes.values() if r.graph is not None]
    times = []
    with torch.cuda.stream(tr._stream):
        for _ in range(reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r.graph.replay()
            e.record()
            e.synchronize()
            times.append(s.elapsed_time(e))
    return {"median_ms": float(np.median(times)), "p10_ms": float(np.percentile(times, 10)),
            "p90_ms": float(np.percentile(times, 90)), "n": reps}


def workload(xf, ref, seq, B, top_k, n_frames, warmup, rounds_of=50):
    tr = xf.tracker(ref, top_k=top_k)
    ref_out = xf.detectAndCompute(ref, top_k=top_k)[0]
    ref_desc, ref_kpts = ref_out["descriptors"], ref_out["keypoints"]
    steps = [np.stack([seq[(k * B + b) % len(seq)] for b in range(B)]) for k in range(len(seq))]
    refs = np.stack([ref] * B)
    routes = {
        "a_tracker": lambda x: tr(x),
        "b_verified_batch": lambda x: xf.match_xfeat_verified_batch(refs, x, top_k=top_k, min_cossim=MIN_COSSIM, ransac_thr=THR,
                                                                    iters=ITERS),
        "c_demo_eager": lambda x: demo_step(xf, ref_desc, ref_kpts, list(x), top_k),
    }
    for f in routes.values():
        for k in range(warmup):
            f(steps[k % len(steps)])
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    i = 0
    while i < n_frames:
        for name, f in routes.items():
            for k in range(i, min(i + rounds_of, n_frames)):
                x = steps[k % len(steps)]
                t0 = time.perf_counter()
                f(x)
                times[name].append(time.perf_counter() - t0)
        i += rounds_of
    res = {name: stats(ts) for name, ts in times.items()}
    # identical results of routes a and b over every step of the sequence
    same_matches, same_h = True, True
    for x in steps:
        ga, gb = tr(x), xf.match_xfeat_verified_batch(refs, x, top_k=top_k, min_cossim=MIN_COSSIM, ransac_thr=THR, iters=ITERS)
        for a, b in zip(ga, gb):
            same_matches &= np.array_equal(a["mkpts0"], b["mkpts0"]) and np.array_equal(a["mkpts1"], b["mkpts1"])
            same_h &= np.array_equal(a["inliers"], b["inliers"]) and (a["H"] is None or np.array_equal(a["H"], b["H"]))
    res["a_equals_b_matches"] = bool(same_matches)
    res["a_equals_b_inliers_and_H"] = bool(same_h)
    res["a_replay_device"] = replay_device_ms(tr)
    res["captures"] = tr.capture_count
    res["mean_matches_per_frame"] = float(np.mean([len(r["mkpts0"]) for x in steps[:8] for r in tr(x)]))
    res["speedup_a_over_b"] = res["b_verified_batch"]["median_ms"] / res["a_tracker"]["median_ms"]
    res["speedup_a_over_c"] = res["c_demo_eager"]["median_ms"] / res["a_tracker"]["median_ms"]
    print(f"B={B} top_k={top_k}", json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500, help="timed steps per route and workload (at least 500 for the record)")
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tracker needs a GPU")
    xf = XFeat()
    with np.load(os.path.join(ROOT, "tests", "golden", "inputs_assets_vga.npz")) as z:
        ref, tgt = z["ref"], z["tgt"]
    seq = [tgt] + make_frames(ref, 15)
    result = {"card": card(), "frames": args.frames, "warmup": args.warmup}
    t0 = time.time()
    result["vga_B1_top_k3000"] = workload(xf, ref, seq, 1, 3000, args.frames, args.warmup)
    result["vga_B1_top_k4096"] = workload(xf, ref, seq, 1, 4096, args.frames, args.warmup)
    result["vga_B4_top_k4096"] = workload(xf, ref, seq, 4, 4096, args.frames, args.warmup)
    result["wall_s"] = time.time() - t0
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
