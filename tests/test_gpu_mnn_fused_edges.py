"""Exact ties of the single-GEMM matcher (implementation 1) on the boundaries of its work split: an item is (pair, 256 columns
of set 2), each of its two 128-column slabs owned by one consumer warpgroup, and the 128-row tiles of set 1 stream past it.
Row arg-maxes merge per slab and item through a global atomic; column arg-maxes run over the tiles in registers and meet
across the 8 row lanes and 4 warps of a slab once per item.  Tied copies sit on each of those boundaries, and the result must
equal implementation 2 and the first-index oracle bit for bit."""
import numpy as np
import pytest
import torch

from tests.test_gpu_mnn_fused import assert_same, match

# set-1 row -> its copies: the lowest row holds every column maximum they tie on.  Rows of tile 8 (1024 ..) by tile-local row
# 16 w + g + 8 (h & 1) + 64 (h >> 1) for warp w, lane group g and fragment row h.
ROW_COPIES = {
    127: (128, 255, 256, 700, 1350),              # across tiles 0 | 1 | 2, tile 5 and the last, partial tile
    1279: (1280, 1399),                           # the last full tile and the partial one
    1042: (1044, 1045, 1062, 1084, 1114, 1151),   # local 18 (w 1, g 2): lane groups 4 and 5, warps 2 and 3, h = 1 and 3
    1033: (1040, 1064, 1090, 1124),               # local 9 (w 0, g 1, h = 1) against later warps and h = 2
}
# the set-2 column that copies each template row (column 899: slab 1 of the last item, four valid columns)
ROW_COLUMN = {127: 127, 1279: 500, 1042: 700, 1033: 899}
# set-2 column -> its copies: the row of set 1 that copies the column ties on all of them, the lowest wins.
# 60 | 190: the two slabs of item 0; 270, 520: items 1 and 2.  150 (slab 1) | 330 (item 1, slab 0) | 640 (item 2, slab 1).
COL_COPIES = {60: (190, 270, 520), 150: (330, 640)}


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@pytest.mark.gpu
def test_fused_exact_ties_on_item_and_tile_edges(xf):
    from oracle import xfeat_oracle as orc
    g = torch.Generator().manual_seed(5)
    n1, n2 = 1400, 900
    f1 = torch.randint(-4, 5, (n1, 64), generator=g).float() / 8
    f2 = torch.randint(-4, 5, (n2, 64), generator=g).float() / 8
    for lo, copies in ROW_COPIES.items():
        for r in copies:
            f1[r] = f1[lo]
    f2[:400] = f1[:400]
    for lo, c in ROW_COLUMN.items():
        f2[c] = f1[lo]
    for c0, copies in COL_COPIES.items():
        for c in copies:
            f2[c] = f2[c0]
    f1b, f2b = f1[None], f2[None]
    got = match(xf, 1, f1b, None, f2b, None)
    assert_same(got, match(xf, 2, f1b, None, f2b, None))
    w0, w1 = orc.mnn_match(f1, f2, -1)
    c = int(got[2][0])
    assert np.array_equal(got[0][0, :c].numpy(), w0.numpy()) and np.array_equal(got[1][0, :c].numpy(), w1.numpy())
    pairs = dict(zip(got[0][0, :c].tolist(), got[1][0, :c].tolist()))
    for lo, col in ROW_COLUMN.items():
        assert pairs.get(lo) == col and not any(r in pairs for r in ROW_COPIES[lo])
    for c0, copies in COL_COPIES.items():
        assert pairs.get(c0) == c0 and not set(copies) & set(pairs.values())
