"""Host-side logic of XFeat.tracker that needs no GPU: argument checks made before anything touches the device, and the step
that turns one replay's downloaded buffers into result dicts (inlier gate, NMS overflow naming the frame)."""
from types import SimpleNamespace

import numpy as np
import pytest

from accelerated_features_b200 import _lib
from accelerated_features_b200.tracker import MAX_TOP_K, Tracker
from accelerated_features_b200.xfeat import XFeat


@pytest.mark.parametrize("top_k", [0, -3, MAX_TOP_K + 1, 100_000])
def test_top_k_outside_ransac_cache_is_refused(top_k):
    with pytest.raises(ValueError, match="top_k"):
        Tracker(SimpleNamespace(top_k=4096), None, top_k=top_k)


def test_default_top_k_of_the_instance_is_checked_too():
    with pytest.raises(ValueError, match=str(MAX_TOP_K)):
        Tracker(SimpleNamespace(top_k=10_000), None)


def unpacker(min_inliers):
    tr = Tracker.__new__(Tracker)
    tr.xf = SimpleNamespace(_check_counts=XFeat._check_counts)
    tr.min_inliers = min_inliers
    return tr


def buffers(cnt, n_inl, k=16):
    B = len(cnt)
    rng = np.random.default_rng(0)
    return (rng.random((B, k, 2), dtype=np.float32), rng.random((B, k, 2), dtype=np.float32), np.array(cnt, np.int32),
            rng.random((B, 3, 3), dtype=np.float32), rng.random((B, k)) > 0.5, np.array(n_inl, np.int32))


def test_results_slice_and_gate():
    args = buffers([9, 12, 0, 5], [8, 3, 0, 5])
    res = unpacker(5)._results(*args)
    assert len(res) == 4
    for b, r in enumerate(res):
        n = args[2][b]
        assert np.array_equal(r["mkpts0"], args[0][b, :n]) and np.array_equal(r["mkpts1"], args[1][b, :n])
        assert np.array_equal(r["inliers"], args[4][b, :n]) and r["n_inliers"] == args[5][b]
    assert res[0]["H"].dtype == np.float64 and np.array_equal(res[0]["H"], args[3][0].astype(np.float64))
    assert res[1]["H"] is None and res[2]["H"] is None and res[3]["H"] is not None
    # a homography needs four inliers whatever min_inliers says
    res = unpacker(0)._results(*buffers([9, 9], [3, 4]))
    assert res[0]["H"] is None and res[1]["H"] is not None


def test_overflow_names_the_frames():
    with pytest.raises(_lib.XFeatLibraryError, match=r"frame 1, frame 3$|frame 1, frame 3;"):
        unpacker(50)._results(*buffers([4, _lib.N_OVERFLOW, 2, _lib.N_OVERFLOW], [0, 0, 0, 0]))
