"""Host side of XFeat.match_xfeat_pairs (no GPU): the extraction plan (buckets, chunks, table slots, remapped pairs), the
validation of `pairs`, and the MegaDepth-1500 pair-structure fixture that tools/bench_pairs.py replays."""
import types

import numpy as np
import pytest
import torch

from accelerated_features_b200.xfeat import PairPlan, XFeat, check_pairs, pair_image_key
from tests.conftest import load_golden


def u8(h, w, c=3):
    return np.zeros((h, w, c), np.uint8)


def test_image_keys_follow_parse_input():
    assert pair_image_key(u8(480, 640)) == (3, 480, 640, "uint8", True)
    assert pair_image_key(np.zeros((480, 640, 3), np.float64)) == (3, 480, 640, "float32", False)   # "/255" on the host
    assert pair_image_key(np.zeros((96, 128), np.uint8)) == (1, 96, 128, "uint8", True)               # (H,W) -> (H,W,1)
    assert pair_image_key(torch.zeros(3, 64, 96)) == (3, 64, 96, "float32", False)
    assert pair_image_key(torch.zeros(1, 1, 64, 96, dtype=torch.uint8)) == (1, 64, 96, "uint8", False)
    for bad in (np.zeros((2, 4, 4, 3), np.uint8), torch.zeros(2, 3, 64, 64), torch.zeros(64, 64), [1, 2]):
        with pytest.raises(RuntimeError):
            pair_image_key(bad)


def test_plan_buckets_slots_and_remap():
    keys = ["a", "b", "a", "c", "b", "a", "a", "d"]          # image 3 ("c") and 7 ("d") are never referenced
    pairs = [[5, 0], [1, 4], [0, 0], [6, 2], [4, 1], [2, 5], [0, 5]]
    plan = PairPlan(keys, pairs, chunk=3)
    # buckets in order of first referenced image, images ascending within a bucket, chunks of at most 3
    assert plan.chunks == [[0, 2, 5], [6], [1, 4]]
    assert plan.n_slots == 6
    assert plan.slot.tolist() == [0, 4, 1, -1, 5, 2, 3, -1]
    assert plan.table_pairs.dtype == np.int32
    assert plan.table_pairs.tolist() == [[plan.slot[i], plan.slot[j]] for i, j in pairs]
    for ch in plan.chunks:
        assert len({keys[i] for i in ch}) == 1
    # matching order: by (j, i) in table slots, every pair exactly once
    order = plan.match_order()
    tp = plan.table_pairs[order]
    assert sorted(order.tolist()) == list(range(len(pairs)))
    assert [tuple(r) for r in tp[:, ::-1]] == sorted(tuple(r) for r in tp[:, ::-1])


def test_plan_default_chunk_is_64():
    plan = PairPlan(["k"] * 130, [[i, 129 - i] for i in range(130)])
    assert [len(c) for c in plan.chunks] == [64, 64, 2]
    assert sorted(plan.slot.tolist()) == list(range(130))


@pytest.mark.parametrize("pairs,exc", [
    (np.zeros((3,), np.int64) + 1, ValueError),                # not (P, 2)
    (np.zeros((2, 3), np.int64), ValueError),
    (np.zeros((2, 2, 1), np.int64), ValueError),
    (np.array([[0.0, 1.0]]), TypeError),                        # float indices
    (np.array([[True, False]]), TypeError),
    ([[0, -1]], ValueError),                                    # negative
    ([[0, 1], [3, 0]], ValueError),                             # out of range (3 images)
])
def test_bad_pairs_rejected(pairs, exc):
    with pytest.raises(exc):
        check_pairs(pairs, 3)


def test_bad_pairs_raise_before_any_launch_and_empty_returns_empty():
    """The host checks run before the method touches the library: a stand-in without one shows that nothing was launched."""
    fake = types.SimpleNamespace(top_k=128)
    imgs = [u8(64, 64), u8(64, 96)]
    for bad in ([[0, 2]], [[0.0, 1.0]], [[0, 1, 1]]):
        with pytest.raises((ValueError, TypeError)):
            XFeat.match_xfeat_pairs(fake, imgs, bad)
        with pytest.raises((ValueError, TypeError)):
            XFeat.match_xfeat_lighterglue_pairs(fake, imgs, bad)
    for empty in ([], np.zeros((0, 2), np.int64)):
        assert XFeat.match_xfeat_pairs(fake, imgs, empty) == []
        assert XFeat.match_xfeat_lighterglue_pairs(fake, imgs, empty) == []
    assert check_pairs([[1, 0]], 2).dtype == np.int64


def test_megadepth1500_fixture():
    z = load_golden("megadepth1500_pairs.npz")
    sizes, pairs = z["sizes"], z["pairs"]
    assert sizes.shape == (806, 2) and sizes.dtype == np.int32
    assert pairs.shape == (1500, 2) and pairs.dtype == np.int32
    assert (sizes % 32 == 0).all() and sizes.max() == 1184 and sizes.min() > 0
    assert pairs.min() == 0 and pairs.max() == 805
    assert len(np.unique(pairs)) == 806                          # every image is used
    assert len({tuple(s) for s in sizes.tolist()}) == 20
    keys = [(3, h, w, "uint8", True) for h, w in sizes.tolist()]
    plan = PairPlan(keys, pairs)
    assert plan.n_slots == 806 and len(plan.chunks) >= 20
