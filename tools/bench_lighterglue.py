"""Time LighterGlue (XFeat.match_lighterglue_batch) on B pairs x n points with CUDA events; prints one JSON line.

Inputs: the 4096-point asset pair of tests/golden/lg_assets_4096.npz repeated over the batch (real keypoints and descriptors,
the latter stored to 1/128, so pruning behaves as on real images).  Matcher weights: oracle/_ref/lighterglue_state.npz, staged by
build() (oracle/build_lighterglue.py).  FLOPs are algorithmic, computed from the point counts (multiply-add = 2): the six layers' linears
and attention, and the assignment's similarity matrix; `gflop_per_pair_unpruned` assumes every point survives, and the achieved
rate uses the same unpruned count (so it is an upper bound of useful work when pruning removes points).  `points_after_pruning`
is the mean count per image after the last layer, read back through the xfeat_lg_debug hook in a separate, untimed call."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def flops_per_pair(n0: int, n1: int) -> float:
    D = 96
    lin_self = 2 * (D * 3 * D + D * D + 4 * D * D + 2 * D * D)       # qkv, out, ffn 192x192, ffn 192x96 per point
    lin_cross = 2 * (D * 2 * D + D * D + 4 * D * D + 2 * D * D)
    per_layer = (n0 + n1) * (lin_self + lin_cross)
    per_layer += 2 * 2 * D * (n0 * n0 + n1 * n1)                      # self: q k^T and p v
    per_layer += 2 * 2 * D * (2 * n0 * n1)                            # cross: both directions
    total = 6 * per_layer + (n0 + n1) * 2 * 64 * D                    # + input projection
    total += (n0 + n1) * 2 * D * D + 2 * 2 * D * n0 * n1              # final_proj + the two passes over S
    return float(total)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--prune-min-points", type=int, default=1536, help="-1: no pruning")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lighterglue needs a CUDA device")
    from accelerated_features_b200 import XFeat, _lib
    from oracle import build_lighterglue
    xf = XFeat(device=0, lighterglue_weights=build_lighterglue.path())
    with np.load(os.path.join(ROOT, "tests", "golden", "lg_assets_4096.npz")) as z:
        g = {k: z[k] for k in z.files}
    for s in range(2):
        g[f"desc{s}"] = g[f"desc{s}_q"].astype(np.float32) / np.float32(128)     # the stored int8 descriptors, as the tests read them
    B, n = a.pairs, a.points
    reps = -(-n // len(g["kpts0"]))
    dev = lambda x, dt=torch.float32: torch.as_tensor(np.ascontiguousarray(x)).to("cuda", dt)   # noqa: E731
    side = []
    for s in range(2):
        k = np.tile(g[f"kpts{s}"], (reps, 1))[:n]
        d = np.tile(g[f"desc{s}"], (reps, 1))[:n]
        side.append((dev(np.broadcast_to(k, (B, n, 2))), dev(np.broadcast_to(d, (B, n, 64))),
                     dev(np.full(B, n), torch.int32), dev(np.broadcast_to(g[f"size{s}"].astype(np.float32), (B, 2)))))
    T = None if a.prune_min_points < 0 else a.prune_min_points
    args = (*side[0], *side[1])
    for _ in range(a.warmup):
        xf.match_lighterglue_batch(*args, prune_min_points=T)
    torch.cuda.synchronize()
    times = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, _, _, cnt = xf.match_lighterglue_batch(*args, prune_min_points=T)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    # points left after the last layer (untimed)
    lib = xf._lib
    x = torch.empty((2, B, n, 96), device="cuda")
    ind = torch.empty((2, B, n), dtype=torch.int32, device="cuda")
    left = torch.empty((2, B), dtype=torch.int32, device="cuda")
    ws = xf._workspace(lib.xfeat_lg_workspace_bytes(B, n))
    _lib.check(lib.xfeat_lg_debug(xf._lg().ctx, B, n, *[t.data_ptr() for t in args], -1 if T is None else T, 6, x.data_ptr(),
                                  ind.data_ptr(), left.data_ptr(), None, None, ws.data_ptr(), ws.numel(), xf._stream()),
               "xfeat_lg_debug")
    t = float(np.median(times))
    fl = flops_per_pair(n, n)
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"metric": "lighterglue_pairs_per_s", "value": B / t, "pairs": B, "points": n,
                      "prune_min_points": T, "median_s": t, "step_s": times, "gflop_per_pair_unpruned": fl / 1e9,
                      "tflops_unpruned_count": B * fl / t / 1e12, "points_after_pruning": float(left.float().mean().item()),
                      "matches_mean": float(cnt.float().mean().item()), "device": props.name}))


if __name__ == "__main__":
    main()
