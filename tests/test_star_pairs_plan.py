"""Host side of XFeat.match_xfeat_star_pairs (no GPU): the dense row count of an image against the oracle's extract_dualscale,
the byte budget of the matcher chunks, and the checks that run before anything is launched."""
import types

import numpy as np
import pytest
import torch

from accelerated_features_b200 import xfeat as X
from accelerated_features_b200.xfeat import PairPlan, XFeat, dense_counts, pair_image_key, star_match_chunks, star_pair_bytes
from tests.conftest import load_golden

TOPKS = [-1, 0, 1, 4, 5, 4096, 10_000]


@pytest.mark.parametrize("hw", [(64, 96), (96, 160), (130, 90), (200, 330)])
def test_dense_counts_match_oracle_extract_dualscale(hw, oracle_state):
    from oracle import xfeat_oracle as orc
    H, W = hw
    x = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(H * W))
    for top_k in TOPKS:
        with torch.inference_mode():
            kp, sc, feats = orc.extract_dualscale(oracle_state, x, top_k)
        k1, k2 = dense_counts(H, W, top_k)
        assert kp.shape[1] == feats.shape[1] == k1 + k2, (hw, top_k)
        assert int((sc[0] == 1 / 0.6).sum()) == k1, (hw, top_k)   # the first scale's rows carry 1/s1


def test_dense_counts_reference_quirks():
    cells1, cells2 = (288 // 8) * (384 // 8), (608 // 8) * (832 // 8)   # 480x640 at 0.6 and 1.3, cropped to 32
    assert dense_counts(480, 640, 4096) == (819, 3276)                   # int(4096*0.2), int(4096*0.8)
    assert dense_counts(480, 640, 4) == (cells1, 3)                      # int(0.8) = 0: the first scale is unlimited
    assert dense_counts(480, 640, 1) == (cells1, cells2)                 # both caps below 1
    assert dense_counts(480, 640, -1) == (cells1, cells2)
    assert dense_counts(480, 640, 5) == (1, 4)
    assert dense_counts(50, 640, 4096)[0] == 0                           # floor(50*0.6) = 30 < 32


def test_megadepth_sizes_all_give_10000_rows():
    sizes = load_golden("megadepth1500_pairs.npz")["sizes"]
    assert {sum(dense_counts(h, w, 10_000)) for h, w in sizes.tolist()} == {10_000}


def test_star_pair_bytes_covers_the_library_workspaces():
    from accelerated_features_b200 import _lib
    from accelerated_features_b200.build import build_library
    build_library()
    lib = _lib.load()
    for k in (1, 511, 4095, 10_000):
        for B in (1, 7, 39):
            need = (lib.xfeat_mnn_pairs_f32_workspace_bytes(B, k) + lib.xfeat_refine_pairs_workspace_bytes(B, k)
                    + B * k * (8 + 8 + 16) + 3 * B * 4)             # idx0, idx1, matches, counts
            assert need <= B * star_pair_bytes(k), (k, B)
    assert 4.5e3 < X._REFINE_ROW_BYTES < 5e3                              # ~4.8 KB per coarse-row slot


def test_star_match_chunks_follow_the_budget():
    per = star_pair_bytes(10_000)
    for P, budget in ((1500, 2 << 30), (100, 10 * per), (100, 10 * per + per - 1), (5, 1 << 40), (3, per - 1), (4, 1)):
        ch = star_match_chunks(P, 10_000, budget)
        step = max(1, budget // per)
        assert ch[0][0] == 0 and ch[-1][1] == P
        assert all(a[1] == b[0] for a, b in zip(ch, ch[1:]))                # contiguous, in order, every pair once
        assert all(1 <= e - s <= step for s, e in ch)
        assert all(e - s == min(step, P) for s, e in ch[:-1])
        assert all((e - s) * per <= budget for s, e in ch) or step == 1       # within the budget, or one pair larger than it
    assert [e - s for s, e in star_match_chunks(3, 10_000, 1)] == [1, 1, 1]    # a single pair above the budget still runs
    assert star_match_chunks(0, 10_000) == []
    assert len(star_match_chunks(1500, 10_000)) == -(-1500 // ((2 << 30) // per))
    assert max(e - s for s, e in star_match_chunks(200_000, 1, 1 << 50)) == 65535


def u8(h, w, c=3):
    return np.zeros((h, w, c), np.uint8)


def test_bad_pairs_and_small_images_raise_before_any_launch():
    """A stand-in without the library shows that nothing was launched."""
    fake = types.SimpleNamespace(top_k=4096)
    imgs = [u8(64, 64), u8(64, 96), u8(50, 640), np.zeros((640, 40), np.uint8)]
    for bad in ([[0, 4]], [[0.0, 1.0]], [[0, 1, 1]], [[-1, 0]]):
        with pytest.raises((ValueError, TypeError)):
            XFeat.match_xfeat_star_pairs(fake, imgs, bad)
    for i in (2, 3):
        with pytest.raises(RuntimeError, match=rf"image {i} \(.*image smaller than 32 pixels"):
            XFeat.match_xfeat_star_pairs(fake, imgs, [[0, 1], [1, i]])
    for empty in ([], np.zeros((0, 2), np.int64)):
        assert XFeat.match_xfeat_star_pairs(fake, imgs, empty) == []


def test_star_pair_rows_per_slot():
    imgs = [u8(480, 640), u8(64, 96), u8(50, 640), u8(320, 448)]   # image 2 is too small but not referenced
    keys = [pair_image_key(x) for x in imgs]
    plan = PairPlan(keys, [[0, 1], [3, 0], [1, 1]])
    rows = X.star_pair_rows(keys, plan, 4096)
    assert rows.dtype == np.int32 and len(rows) == plan.n_slots == 3
    for i in (0, 1, 3):
        assert rows[plan.slot[i]] == sum(dense_counts(*imgs[i].shape[:2], 4096))
