"""Self-checks of helpers_ref.py on the CPU: each reference equals the oracle's ATen form, and each derived bound covers ATen's
own fp32 result (a different evaluation order than the kernels', so a bound that fails here is too tight to be a bound)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import xfeat_oracle as orc
from tests import helpers_ref as hr


def test_heatmap_ref_and_bound():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 65, 7, 13, generator=g) * 20
    x[0, 64] = 60.0                                              # the dustbin dominant
    x[1, :, 0, 0] = 3.0                                          # all equal
    for t in (1.0, 2.0, 0.5, 0.0, -1.0):
        ref = hr.heatmap_ref(x, t)
        aten = orc.kpts_heatmap(x, t).double()
        r = float(((aten - ref).abs() / hr.heatmap_bound(x, t)).max())
        print(f"temp {t}: ATen fp32 / bound {r:.3f}")
        assert r <= 1.0


def test_nms_ref_is_maxpool_with_nan_and_inf():
    g = torch.Generator().manual_seed(2)
    h = torch.rand(3, 37, 41, generator=g)
    h[0, 5, 5] = float("nan")
    h[0, 5, 6] = 0.99
    h[1, 10, 10] = float("inf")
    h[1, 10, 12] = float("inf")
    h[2, 3:9, 3:9] = 0.5
    h[2, 20, 20] = -float("inf")
    for k in (1, 3, 5, 7, 31):
        for thr in (0.05, 0.5):
            want = orc.nms(h[:, None], thr, k)
            cnt = orc.nms_counts(h[:, None], thr, k)
            for b, p in enumerate(hr.nms_ref(h.numpy(), thr, k)):
                assert np.array_equal(p, want[b, :cnt[b]].numpy()), (k, thr, b)
    assert [6, 5] not in hr.nms_ref(h.numpy(), 0.05, 5)[0].tolist()     # a NaN neighbour suppresses the 0.99 peak


@pytest.mark.parametrize("mode", ["nearest", "bilinear", "bicubic"])
def test_sample_ref_against_grid_sample(mode):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 5, 9, 14, generator=g)
    H, W = 77, 101
    pos = torch.rand(2, 300, 2, generator=g) * torch.tensor([W + 20.0, H + 20.0]) - 10
    pos[0, :40] = torch.randint(0, 100, (40, 2), generator=g).float()
    want = orc.sample_sparse(x, pos, H, W, mode).double().numpy()
    got, bound = hr.sample_ref(x.numpy(), pos.numpy(), H, W, mode)
    err = np.abs(got - want).max()
    print(f"{mode}: ATen fp32 against the float64 reference, worst error {err:.2e}")
    if mode == "nearest":
        assert np.array_equal(got, want)
    else:
        # ATen's CPU kernel rounds the source coordinate in its own order (with FMAs), so it samples a few ulp away from
        # source_coord; the derived bound is for the same coordinate and is checked against the CUDA kernel, which uses it
        assert err < 1e-5


def test_subpix_ref_and_bound():
    g = torch.Generator().manual_seed(4)
    m = torch.randn(500, 64, generator=g) * 3
    m[:8] = 0
    for i, c in enumerate((0, 7, 56, 63)):
        m[i, c] = 1e3
        m[4 + i, c] = -1e3
    for t in (3.0, 1.0, 0.0, -3.0, 50.0):
        ref = hr.subpix_ref(m, t)
        aten = orc.subpix_softmax2d(m.view(-1, 8, 8), t).double()
        r = float(((aten - ref).abs().max(1)[0] / hr.subpix_bound(m, t)).max())
        print(f"temp {t}: ATen fp32 / bound {r:.3f}")
        assert r <= 1.0
    assert torch.equal(hr.subpix_ref(m[:1], 0.0), torch.tensor([[-0.5, -0.5]], dtype=torch.float64))
