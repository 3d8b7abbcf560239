"""The homography, essential- and fundamental-matrix RANSAC, bit for bit: every call stored in tests/golden/ransac_pinned.npz
(tools/make_golden_ransac.py) is replayed from its stored inputs through the public batch API, and the model (as uint32 bits),
the packed mask and the inlier counts must equal the stored ones.  The float64 reference tests in test_gpu_ransac_models.py
allow any sample stream that converges; these pin the stream itself (hash constants, hypothesis and pair ids) and the order of
every reduction.  The 7-point solver hook is pinned the same way."""
import numpy as np
import pytest
import torch

from accelerated_features_b200.geometry import find_essential_batch, find_fundamental_batch, find_homography_batch
from tests.test_gpu_ransac_models import run_seven_point

pytestmark = pytest.mark.gpu


def run(kind, p0, p1, cnt, thr, iters, seed, ids=None):
    """One call of the public batch API: (model (B, 9) float32, mask (B, n_max) bool, counts (B) int32)."""
    a, b, c = (torch.from_numpy(x).cuda() for x in (p0, p1, cnt))
    if kind == "h":
        out = find_homography_batch(a, b, c, thr=thr, iters=iters, seed=seed)
    elif kind == "e":
        out = find_essential_batch(a, b, c, thr=thr, iters=iters, seed=seed)
    else:
        out = find_fundamental_batch(a, b, c, thr=thr, iters=iters, seed=seed, pair_ids=ids)
    model, mask, n = (t.cpu().numpy() for t in out)
    return model.reshape(len(cnt), 9), mask, n


@pytest.fixture(scope="module")
def pinned(golden):
    return golden("ransac_pinned.npz")


@pytest.mark.parametrize("kind", ["h", "e", "f"])
def test_ransac_outputs_pinned(pinned, kind):
    calls = [f"call{i:03d}." for i in range(int(pinned["n_calls"])) if str(pinned[f"call{i:03d}.kind"]) == kind]
    assert calls
    for pre in calls:
        name, thr = str(pinned[pre + "set"]), float(pinned[pre + "thr"])
        iters, seed = int(pinned[pre + "iters"]), int(pinned[pre + "seed"])
        p0, p1, cnt = (pinned[f"{kind}_{name}.{k}"] for k in ("p0", "p1", "cnt"))
        ids = pinned.get(pre + "pair_ids")
        model, mask, n = run(kind, p0, p1, cnt, thr, iters, seed, ids)
        what = f"{kind} {name} iters={iters} seed={seed:#x} pair_ids={ids is not None}"
        assert np.array_equal(model.view(np.uint32), pinned[pre + "model"].view(np.uint32)), what
        assert np.array_equal(np.packbits(mask, axis=1), pinned[pre + "mask"]), what
        assert np.array_equal(n, pinned[pre + "n_inliers"]), what


def test_seven_point_pinned(pinned):
    Fc, nc = run_seven_point(pinned["seven.samples"])
    assert np.array_equal(nc, pinned["seven.count"])
    assert np.array_equal(Fc.reshape(len(nc), 3, 9).view(np.uint32), pinned["seven.F"].view(np.uint32))
