#!/usr/bin/env python
"""Pair-list matching (XFeat.match_xfeat_pairs) against per-batch extraction (match_xfeat_stream), on one GPU.

Workloads (sparse, top_k 4096, uint8 numpy images on the host, as the evaluation harness passes them):
  a  MegaDepth-1500 replay: the benchmark's pair structure (tests/golden/megadepth1500_pairs.npz: 806 images in 20 shapes, 1500
     pairs) with seeded synthetic images -- the VGA assets resized to each size plus noise.  New: one match_xfeat_pairs call over
     all pairs, and one call per 64-pair chunk.  Old: the harness's former grouping by (shape0, shape1) into 64-pair batches
     through match_xfeat_stream, restated here.
  b  exhaustive matching of 64 VGA images (2016 pairs): one match_xfeat_pairs call against match_xfeat_stream over the same
     pairs in 64-pair batches.
  c  512 distinct VGA pairs, no image repeated: match_xfeat_pairs against match_xfeat_stream in 64-pair batches.
  d  the pair order of the matcher launch: xfeat_mnn_match_pairs alone on the extracted tables of (a) and (b), pairs sorted by
     (j, i) against a seeded shuffle.
Every time is CUDA events around the whole call (each call ends with its results on the host); A and B alternate.  The card's
name and power limit are read in the same run.

    python tools/bench_pairs.py [--reps 5] [--out FILE]     # prints one JSON result line; --out also writes it to FILE
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
from accelerated_features_b200.xfeat import PairPlan, pair_image_key  # noqa: E402

TOPK = 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3, out


def ab(name, arms, reps):
    """arms: {label: fn}; alternate them `reps` times after one warm-up each.  Returns {label: stats} and the last outputs."""
    outs = {k: f() for k, f in arms.items()}                 # warm-up (and the outputs compared below)
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            times[k].append(timed(f)[0])
    res = {k: {"median_s": float(np.median(v)), "min_s": float(np.min(v)), "max_s": float(np.max(v))} for k, v in times.items()}
    print(name, json.dumps(res), flush=True)
    return res, outs


def same(a, b):
    return all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b)) and len(a) == len(b)


def stream_grouped(xf, images, pairs, batch=64):
    """The harness's former sparse mode: pairs grouped by (shape0, shape1), 64-pair batches through match_xfeat_stream."""
    out = [None] * len(pairs)
    groups = {}
    for p, (i, j) in enumerate(pairs):
        groups.setdefault((images[i].shape, images[j].shape), []).append(p)
    for idxs in groups.values():
        chunks = [idxs[o:o + batch] for o in range(0, len(idxs), batch)]
        batches = ((np.stack([images[pairs[p][0]] for p in ch]), np.stack([images[pairs[p][1]] for p in ch])) for ch in chunks)
        for ch, res in zip(chunks, xf.match_xfeat_stream(batches, top_k=TOPK)):
            for p, r in zip(ch, res):
                out[p] = r
    return out


def pairs_chunked(xf, images, pairs, chunk):
    out = []
    for o in range(0, len(pairs), chunk):
        out += xf.match_xfeat_pairs(images, pairs[o:o + chunk], top_k=TOPK)
    return out


def order_effect(xf, images, pairs, reps):
    """xfeat_mnn_match_pairs alone: sorted (j, i) order against a seeded shuffle of the same pairs."""
    plan = PairPlan([pair_image_key(x) for x in images], pairs)
    tab = xf._extract_table(images, plan, TOPK, want_split=True, want_desc=False)
    sorted_tp = plan.table_pairs[plan.match_order()]
    shuffled = plan.table_pairs[np.random.default_rng(0).permutation(len(pairs))]
    arms = {}
    for label, tp in (("sorted_ji", sorted_tp), ("shuffled", shuffled)):
        t = torch.from_numpy(np.ascontiguousarray(tp)).cuda()
        arms[label] = (lambda t=t: xf._mnn_pairs_device(tab, t, TOPK, -1.0))
    res, outs = ab("order", arms, reps)
    torch.cuda.synchronize()
    return res


def synth(base, h, w, rng):
    import cv2
    im = cv2.resize(base, (w, h), interpolation=cv2.INTER_LINEAR).astype(np.int16)
    return np.clip(im + rng.integers(-10, 11, im.shape, dtype=np.int16), 0, 255).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", help="also write the JSON result to this file")
    ap.add_argument("--only", default="abcd")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pairs needs a GPU")
    xf = XFeat()
    with np.load(os.path.join(ROOT, "tests", "golden", "inputs_assets_vga.npz")) as z:
        ref, tgt = z["ref"], z["tgt"]
    rng = np.random.default_rng(0)
    result = {"card": card(), "top_k": TOPK, "reps": args.reps}
    t0 = time.time()

    if "a" in args.only or "d" in args.only:
        with np.load(os.path.join(ROOT, "tests", "golden", "megadepth1500_pairs.npz")) as z:
            sizes, md_pairs = z["sizes"], z["pairs"]
        md_images = [synth(ref if k % 2 == 0 else tgt, int(h), int(w), rng) for k, (h, w) in enumerate(sizes)]
        md_list = [tuple(p) for p in md_pairs.tolist()]
    if "a" in args.only:
        res, outs = ab("a_megadepth", {
            "pairs_one_call": lambda: xf.match_xfeat_pairs(md_images, md_pairs, top_k=TOPK),
            "pairs_64_chunks": lambda: pairs_chunked(xf, md_images, md_pairs, 64),
            "stream_grouped_64": lambda: stream_grouped(xf, md_images, md_list),
        }, args.reps)
        res["identical_outputs"] = same(outs["pairs_one_call"], outs["stream_grouped_64"]) and same(outs["pairs_64_chunks"],
                                                                                                     outs["stream_grouped_64"])
        res["matches_total"] = int(sum(len(r[0]) for r in outs["pairs_one_call"]))
        result["a_megadepth1500"] = res
        print("a identical:", res["identical_outputs"], flush=True)

    vga = [synth(ref if k % 2 == 0 else tgt, 480, 640, rng) for k in range(64)]
    ex_pairs = np.array([(i, j) for i in range(64) for j in range(i + 1, 64)], np.int64)
    if "b" in args.only:
        res, outs = ab("b_exhaustive", {
            "pairs_one_call": lambda: xf.match_xfeat_pairs(vga, ex_pairs, top_k=TOPK),
            "stream_64": lambda: stream_grouped(xf, vga, [tuple(p) for p in ex_pairs.tolist()]),
        }, args.reps)
        res["identical_outputs"] = same(outs["pairs_one_call"], outs["stream_64"])
        result["b_exhaustive64"] = res
    if "c" in args.only:
        uni = [synth(ref if k % 2 == 0 else tgt, 480, 640, rng) for k in range(1024)]
        u_pairs = np.arange(1024).reshape(512, 2)
        res, outs = ab("c_uniform", {
            "pairs_one_call": lambda: xf.match_xfeat_pairs(uni, u_pairs, top_k=TOPK),
            "stream_64": lambda: stream_grouped(xf, uni, [tuple(p) for p in u_pairs.tolist()]),
        }, args.reps)
        res["identical_outputs"] = same(outs["pairs_one_call"], outs["stream_64"])
        result["c_uniform512"] = res
        del uni
    if "d" in args.only:
        result["d_order"] = {"megadepth1500": order_effect(xf, md_images, md_pairs, 3 * args.reps),
                             "exhaustive64": order_effect(xf, vga, ex_pairs, 3 * args.reps)}
    result["wall_s"] = time.time() - t0
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
