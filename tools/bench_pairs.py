#!/usr/bin/env python
"""Pair-list matching (XFeat.match_xfeat_pairs, match_xfeat_star_pairs) against per-batch extraction (match_xfeat_stream,
match_xfeat_star), on one GPU.

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
Semi-dense (XFeat*), the same synthetic images:
  e  the MegaDepth-1500 replay at top_k 10 000 (the reference's XFeat* setting; all 20 sizes give 10 000 rows per image): one
     match_xfeat_star_pairs call against the harness's former star mode, restated here: (shape0, shape1) groups, 64-pair chunks
     through match_xfeat_star.
  f  exhaustive matching of 64 VGA images at top_k 4096: one match_xfeat_star_pairs call against the same pairs through
     match_xfeat_star in 64-pair batches.
  The batched old arm splits each batch's descriptors at one exponent for the whole batch, so both arms are also compared with
  per-pair match_xfeat_star calls on a seeded sample of pairs; every pair where an arm differs is listed.
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


def star_grouped(xf, images, pairs, top_k, batch=64):
    """The harness's former star mode: pairs grouped by (shape0, shape1), 64-pair chunks through match_xfeat_star."""
    out = [None] * len(pairs)
    groups = {}
    for p, (i, j) in enumerate(pairs):
        groups.setdefault((images[i].shape, images[j].shape), []).append(p)
    for idxs in groups.values():
        for ch in (idxs[o:o + batch] for o in range(0, len(idxs), batch)):
            res = xf.match_xfeat_star(np.stack([images[pairs[p][0]] for p in ch]), np.stack([images[pairs[p][1]] for p in ch]),
                                      top_k=top_k)
            if len(ch) == 1:
                out[ch[0]] = res                                  # B == 1: two numpy arrays
            else:
                for p, m in zip(ch, res):
                    m = m.cpu().numpy()
                    out[p] = (m[:, :2], m[:, 2:])
    return out


def star_workload(xf, name, images, pairs, top_k, reps, sample=48):
    pair_list = [tuple(p) for p in np.asarray(pairs).tolist()]
    res, outs = ab(name, {
        "star_pairs_one_call": lambda: xf.match_xfeat_star_pairs(images, pairs, top_k=top_k),
        "star_grouped_64": lambda: star_grouped(xf, images, pair_list, top_k),
    }, reps)
    sel = np.sort(np.random.default_rng(1).choice(len(pair_list), min(sample, len(pair_list)), replace=False)).tolist()
    diff = {"star_pairs_one_call": [], "star_grouped_64": []}
    for p in sel:
        i, j = pair_list[p]
        w = xf.match_xfeat_star(images[i], images[j], top_k=top_k)
        for arm in diff:
            if not same([outs[arm][p]], [w]):
                diff[arm].append({"pair": p, "images": [i, j], "n": len(outs[arm][p][0]), "n_single": len(w[0])})
    res["sample_pairs"] = len(sel)
    res["differs_from_single_pair_calls"] = diff
    res["arms_identical"] = same(outs["star_pairs_one_call"], outs["star_grouped_64"])
    res["matches_total"] = int(sum(len(r[0]) for r in outs["star_pairs_one_call"]))
    print(name, "differs from single-pair calls:", {k: len(v) for k, v in diff.items()}, flush=True)
    return res


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
    ap.add_argument("--only", default="abcdef")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pairs needs a GPU")
    xf = XFeat()
    with np.load(os.path.join(ROOT, "tests", "golden", "inputs_assets_vga.npz")) as z:
        ref, tgt = z["ref"], z["tgt"]
    rng = np.random.default_rng(0)
    result = {"card": card(), "top_k": TOPK, "reps": args.reps}
    t0 = time.time()

    if any(w in args.only for w in "ade"):
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
    if "e" in args.only:
        result["e_star_megadepth1500"] = star_workload(xf, "e_star_megadepth", md_images, md_pairs, 10_000, args.reps)
    if "f" in args.only:
        result["f_star_exhaustive64"] = star_workload(xf, "f_star_exhaustive", vga, ex_pairs, 4096, args.reps)
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
