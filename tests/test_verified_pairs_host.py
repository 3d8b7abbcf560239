"""Host-side checks of XFeat.match_xfeat_verified_pairs that need no GPU: they run before the method touches the library, so a
stand-in instance without one shows that nothing was extracted or launched."""
import types

import numpy as np
import pytest

from accelerated_features_b200.xfeat import XFeat


def u8(h, w):
    return np.zeros((h, w, 3), np.uint8)


@pytest.mark.parametrize("top_k", [8193, 100_000])
def test_top_k_above_ransac_cache_is_refused(top_k):
    fake = types.SimpleNamespace(top_k=4096)
    with pytest.raises(ValueError, match="8192"):
        XFeat.match_xfeat_verified_pairs(fake, [u8(64, 64)], [(0, 0)], top_k=top_k)
    with pytest.raises(ValueError, match="8192"):
        XFeat.match_xfeat_verified_pairs(types.SimpleNamespace(top_k=top_k), [u8(64, 64)], [(0, 0)])


def test_bad_pairs_raise_and_empty_returns_empty():
    fake = types.SimpleNamespace(top_k=128)
    imgs = [u8(64, 64), u8(64, 96)]
    for bad in ([[0, 2]], [[0.0, 1.0]], [[0, 1, 1]]):
        with pytest.raises((ValueError, TypeError)):
            XFeat.match_xfeat_verified_pairs(fake, imgs, bad)
    for empty in ([], np.zeros((0, 2), np.int64)):
        assert XFeat.match_xfeat_verified_pairs(fake, imgs, empty) == []
