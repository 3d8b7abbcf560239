#!/usr/bin/env python
"""Per-kernel profile of bench.py's sparse step on one GPU, with torch.profiler.

    python tools/kernel_profile.py --out /tmp/kernel_profile [--steps 5 --warmup 3]

The step is bench.py's resident sparse step at its shapes: `_detect_sparse_device` on both 64-image VGA sets in one call
(B = 128 through the backbone), then the presplit MNN (`_mnn_presplit_device`) and the keypoint gather.  After warm-up, a
timed window (CUDA events, profiler off) gives the step time; a second window runs under the profiler.  Writes
OUT/kernels.md (one row per kernel: launches per step, us per step, share of the summed kernel time of the step) and
OUT/kernels.json, and prints the card's name, power limit and maximum SM clock.

For the wgmma convolution kernels the table also gives the algorithmic FLOPs of the layers they run (2 * MACs of the real
channels, as the model defines them) and the tensor-core rate with the 3 split-fp16 terms counted: 3 * FLOPs / time against
the H100 SXM data-sheet figure of 989 TFLOP/s dense FP16 (a share of the data-sheet peak, not a measured peak).  Kernels bound
by bytes rather than by the tensor pipe (the stem tail, the head chains) also get their algorithmic HBM bytes against the 3.35 TB/s data sheet.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOPK, BATCH, H, W = 4096, 64, 480, 640   # bench.py's sparse config
PEAK_FP16 = 989e12                       # H100 SXM data sheet, dense FP16 / BF16, 700 W card

# Layers of xfeat_net (conv impl 2, the default) by the kernel that runs them: (cin, cout, ks, output H, output W) at the
# bench's VGA input; the head chains count their 1x1 layers at 1/8 resolution.
_B = 2 * BATCH
_LAYERS = {
    "stem_tail_halo_kernel": [(8, 8, 3, H // 2, W // 2), (8, 24, 3, H // 4, W // 4)],                # block1.2, block1.3
    "conv_tc_halo_kernel<32, 32>": [(24, 24, 3, H // 4, W // 4)] * 2,                                  # block2.0-1
    "conv_tc_kernel<3, 32, 64>": [(24, 64, 3, H // 8, W // 8)],                                        # block3.0
    "conv_tc_halo_kernel<64, 64>": [(64, 64, 3, H // 8, W // 8)] * 3 + [(64, 64, 3, H // 16, W // 16)] * 2,  # 3.1, fusion.0-1, 4.1-2
    "conv_tc_kernel<1, 64, 64>": [(64, 64, 1, H // 8, W // 8)],                                        # block3.2
    "conv_tc_kernel<3, 64, 64>": [(64, 64, 3, H // 16, W // 16), (64, 128, 3, H // 32, W // 32)],      # block4.0, block5.0
    "conv_tc128_kernel<3>": [(128, 128, 3, H // 32, W // 32)] * 2,                                      # block5.1-2
    "conv_tc128_kernel<1>": [(128, 64, 1, H // 32, W // 32)],                                           # block5.3
    "head_chain_rf_kernel<0>": [(64, 64, 1, H // 8, W // 8)] * 3 + [(64, 65, 1, H // 8, W // 8)],      # keypoint head
    "head_chain_rf_kernel<1>": [(64, 64, 1, H // 8, W // 8)] * 3 + [(64, 1, 1, H // 8, W // 8)],       # fusion.2 + reliability head
}


# Bandwidth-bound kernels: the HBM bytes per step their algorithm has to move, read once and written once.  The stem tail reads
# a2 (split fp16, 32 B per half-resolution pixel) and the gray image (4 B per pixel) and writes x1s (128 B per quarter-resolution
# pixel).  The keypoint head reads the gray image and writes the heat-map (4 B per full-resolution pixel each); the reliability
# head, with block_fusion.2 in front, reads fusion.1's split output (256 B per cell) and writes the fp32 features (256 B) and
# the reliability (4 B).
_BYTES = {
    "stem_tail_halo_kernel": _B * (H // 2 * W // 2 * 32 + H * W * 4 + H // 4 * W // 4 * 128),
    "head_chain_rf_kernel<0>": _B * H * W * 8,
    "head_chain_rf_kernel<1>": _B * (H // 8 * W // 8) * (256 + 256 + 4),
}
PEAK_HBM = 3.35e12                       # H100 SXM data sheet, HBM3 bytes/s


def algorithmic_flops(kernel: str) -> float:
    """2 * MACs per step of the layers `kernel` runs (0 for kernels outside the table)."""
    return sum(2.0 * _B * ho * wo * cin * cout * ks * ks for cin, cout, ks, ho, wo in _LAYERS.get(kernel, []))


def short_name(name: str) -> str:
    n = re.sub(r"^void\s+", "", name)
    n = re.sub(r"\(.*$", "", n)          # drop the argument list
    return re.sub(r"^xf::", "", n)


def card_info() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"nvidia-smi failed: {r.stderr.strip()}"
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--steps", type=int, default=5, help="steps in the timed and in the profiled window")
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from accelerated_features_b200 import XFeat, _lib
    from accelerated_features_b200 import weights as _w

    if not torch.cuda.is_available():
        raise SystemExit("kernel_profile.py: no CUDA device")
    os.makedirs(a.out, exist_ok=True)
    card = card_info()
    print("card (name, power.limit, clocks.max.sm):", card, flush=True)

    dev = torch.device("cuda", 0)
    xf = XFeat(weights=_w.load_state_dict(_w.DEFAULT_WEIGHTS), top_k=TOPK, device=0)
    lib = _lib.load()
    g = torch.Generator().manual_seed(1000)
    d1 = torch.randn(BATCH, 3, H, W, generator=g).to(dev)
    d2 = torch.randn(BATCH, 3, H, W, generator=g).to(dev)
    presplit = lib.xfeat_get_mnn_impl() in (1, 2, 3)

    def step():
        o = xf._detect_sparse_device([d1, d2], TOPK, xf.detection_threshold, want_split=presplit, want_desc=not presplit)
        k1, k2 = o["keypoints"][:BATCH], o["keypoints"][BATCH:]
        n1, n2 = o["n_valid"][:BATCH], o["n_valid"][BATCH:]
        if presplit:
            sp = o["desc_split"]
            idx0, idx1, cnt = xf._mnn_presplit_device(sp[:BATCH], n1, sp[BATCH:], n2, TOPK, sp.shape[1], BATCH, -1)
        else:
            f1, f2 = o["descriptors"][:BATCH], o["descriptors"][BATCH:]
            idx0, idx1, cnt = xf._mnn_device(f1, n1, TOPK, TOPK * 64, f2, n2, TOPK, TOPK * 64, BATCH, -1, abs_bound=1.0)
        return xf._gather_matches(k1, k2, idx0, idx1, cnt, BATCH, TOPK)

    for _ in range(max(a.warmup, 1)):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.steps

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()

    agg = collections.defaultdict(lambda: [0, 0.0])   # name -> [launches, us]
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        if us <= 0:
            continue
        n = short_name(ev.name)
        agg[n][0] += 1
        agg[n][1] += us
    if not agg:
        raise SystemExit("kernel_profile.py: the profiler recorded no device activity")
    total_us = sum(v[1] for v in agg.values()) / a.steps

    rows = []
    for n, (cnt, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        us_step = us / a.steps
        fl = algorithmic_flops(n)
        rows.append({"kernel": n, "launches_per_step": cnt / a.steps, "us_per_step": us_step, "share": us_step / total_us,
                     "algorithmic_gflop": fl / 1e9 if fl else None,
                     "split3_tflops": 3 * fl / (us_step * 1e-6) / 1e12 if fl else None,
                     "share_of_datasheet_peak": 3 * fl / (us_step * 1e-6) / PEAK_FP16 if fl else None,
                     "algorithmic_gbytes": _BYTES[n] / 1e9 if n in _BYTES else None,
                     "share_of_datasheet_hbm": _BYTES[n] / (us_step * 1e-6) / PEAK_HBM if n in _BYTES else None})
    wg = [r for r in rows if r["kernel"].startswith(("conv_tc", "head_chain"))]
    wg_share = sum(r["share"] for r in wg)

    lines = [f"card (name, power.limit, clocks.max.sm): {card}", "",
             f"step (CUDA events, profiler off, {a.steps} steps after {a.warmup} warm-up): {step_ms:.3f} ms; "
             f"summed kernel time per step under the profiler: {total_us / 1e3:.3f} ms", "",
             f"wgmma convolution + head-chain kernels: {wg_share * 100:.1f} % of the summed kernel time", "",
             "| kernel | launches/step | us/step | share | GFLOP (alg.) | 3-term TFLOP/s | of 989 TFLOP/s data sheet "
             "| GB (alg.) | of 3.35 TB/s data sheet |",
             "|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        fl = (f"{r['algorithmic_gflop']:.1f} | {r['split3_tflops']:.0f} | {r['share_of_datasheet_peak'] * 100:.0f} %"
              if r["algorithmic_gflop"] else " | | ")
        by = (f"{r['algorithmic_gbytes']:.2f} | {r['share_of_datasheet_hbm'] * 100:.0f} %" if r["algorithmic_gbytes"] else " | ")
        lines.append(f"| `{r['kernel'][:110]}` | {r['launches_per_step']:g} | {r['us_per_step']:.1f} | {r['share'] * 100:.2f} % | {fl} | {by} |")
    text = "\n".join(lines) + "\n"
    with open(os.path.join(a.out, "kernels.md"), "w") as f:
        f.write(text)
    with open(os.path.join(a.out, "kernels.json"), "w") as f:
        json.dump({"card": card, "step_ms": step_ms, "kernel_us_per_step": total_us, "steps": a.steps, "kernels": rows}, f, indent=1)
    print(text)


if __name__ == "__main__":
    main()
