#!/usr/bin/env python
"""Generate tests/golden/megadepth1500_pairs.npz from the reference's MegaDepth-1500 pair list (assets/megadepth_1500.json).

Run where a checkout of the reference is present (its root as the argument or in XFEAT_REFERENCE_ROOT):

    python tools/make_pairs_fixture.py REFERENCE_ROOT

The fixture is derived data only: `sizes` (n_images, 2) int32 (h, w) of each distinct image at the size the benchmark feeds the
matcher (`size0_hw` / `size1_hw`), in order of first appearance, and `pairs` (1500, 2) int32 indices into `sizes`.  Images are
told apart by their `pair_names` entry.  tools/bench_pairs.py replays the benchmark's pair structure from it with synthetic
images.
"""
import json
import os
import sys

import numpy as np

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("XFEAT_REFERENCE_ROOT")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "megadepth1500_pairs.npz")


def main():
    if not REF:
        raise SystemExit("usage: make_pairs_fixture.py REFERENCE_ROOT (or set XFEAT_REFERENCE_ROOT)")
    with open(os.path.join(REF, "assets", "megadepth_1500.json")) as f:
        items = json.load(f)
    index, sizes, pairs = {}, [], []
    for it in items:
        ij = []
        for name, hw in zip(it["pair_names"], (it["size0_hw"], it["size1_hw"])):
            if name not in index:
                index[name] = len(sizes)
                sizes.append(hw)
            elif sizes[index[name]] != hw:
                raise ValueError(f"{name}: two sizes {sizes[index[name]]} and {hw}")
            ij.append(index[name])
        pairs.append(ij)
    sizes, pairs = np.asarray(sizes, np.int32), np.asarray(pairs, np.int32)
    np.savez_compressed(OUT, sizes=sizes, pairs=pairs)
    shapes = {tuple(s) for s in sizes.tolist()}
    print(f"{OUT}: {len(sizes)} images in {len(shapes)} shapes, {len(pairs)} pairs")


if __name__ == "__main__":
    main()
