"""CPU checks of tests/ingest_ref.py, the host reference of image ingest: its float32 emulation against ATen's CPU bilinear
upsample (both the size and the scale-factor form), ATen's copy of an axis that keeps its size, and its InstanceNorm against
F.instance_norm in float64.  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import ingest_ref as ir

F32 = np.float32
MAX_ULPS = 4     # ATen's CPU kernel contracts the interpolation's products and sums into FMAs; the emulation rounds each one


def bilinear_ulps(got: np.ndarray, want: np.ndarray, x: np.ndarray, out, sh, sw, fma: bool) -> float:
    """Largest |got - want| in float32 ulps of the interpolation's magnitude (the same bilinear of |x|): the unit of the
    rounding error of a sum of products, which stays meaningful where neighbours of opposite sign cancel."""
    mag = ir.resize(np.abs(x), out[0], out[1], sh, sw, fma=fma)
    return float((np.abs(got.astype(np.float64) - want) / np.spacing(mag)).max())


def randn(shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


# (input shape, F.interpolate keyword arguments, output size)
CASES = [
    ((2, 3, 300, 400), dict(size=(288, 384)), (288, 384)),          # preprocess_tensor's resize to multiples of 32 (down)
    ((1, 3, 100, 150), dict(size=(96, 160)), (96, 160)),            # down in H, up in W
    ((2, 3, 480, 640), dict(scale_factor=0.6), (288, 384)),         # extract_dualscale s1
    ((2, 3, 480, 640), dict(scale_factor=1.3), (624, 832)),         # extract_dualscale s2
    ((1, 3, 960, 1280), dict(scale_factor=0.6), (576, 768)),
    ((1, 2, 37, 53), dict(scale_factor=2.7), (99, 143)),            # edge taps: src past in - 1 at the bottom and right
    ((2, 3, 480, 640), dict(scale_factor=1.0018), (480, 641)),      # H keeps its size and is copied, W is interpolated
]


@pytest.mark.parametrize("shape,kw,out", CASES, ids=lambda c: str(c).replace(" ", ""))
def test_emulation_matches_aten_bilinear(shape, kw, out):
    """With ATen's fused source index the emulation is ATen's CPU result up to FMA contraction of the interpolation itself.
    The kernels' unfused source index is the same value or one float32 ulp of src away; the outputs then agree exactly at
    every pixel whose row and column indices agree."""
    x = randn(shape, seed=sum(shape))
    want = F.interpolate(x, mode="bilinear", align_corners=False, **kw).numpy()
    assert tuple(want.shape[-2:]) == out
    Hi, Wi = shape[-2:]
    if "size" in kw:
        sh, sw = ir.size_scale(Hi, out[0]), ir.size_scale(Wi, out[1])
    else:
        sh = sw = ir.factor_scale(kw["scale_factor"])
    xs = x.numpy()
    got_fma = ir.resize(xs, out[0], out[1], sh, sw, fma=True)
    d = bilinear_ulps(got_fma, want, xs, out, sh, sw, True)
    got = ir.resize(xs, out[0], out[1], sh, sw)
    d_kernel = bilinear_ulps(got, want, xs, out, sh, sw, False)
    esh, esw = ir.effective_scales(Hi, Wi, out[0], out[1], sh, sw)
    rows = ir.lin_taps(out[0], Hi, esh)[3] == ir.lin_taps(out[0], Hi, esh, fma=True)[3]
    cols = ir.lin_taps(out[1], Wi, esw)[3] == ir.lin_taps(out[1], Wi, esw, fma=True)[3]
    print(f"emulation vs ATen CPU {shape} {kw}: max {d:g} ulp with ATen's fused source index; kernels' arithmetic: max "
          f"{d_kernel:g} ulp, source index rounded apart in {(~rows).sum()} of {rows.size} rows, {(~cols).sum()} of "
          f"{cols.size} columns")
    assert d <= MAX_ULPS, d
    assert np.array_equal(got[..., rows[:, None] & cols[None, :]], got_fma[..., rows[:, None] & cols[None, :]])
    f64 = np.stack([ir.bilinear_f64(xs[b], out[0], out[1], sh, sw) for b in range(shape[0])])
    assert bilinear_ulps(got, f64, xs, out, sh, sw, False) <= 3      # 1 - l1, two products and a sum per axis


def test_same_size_axis_is_a_copy():
    """ATen copies along an axis whose output size equals its input size, whatever the scale factor; the emulation samples
    that axis at scale 1, which is an exact copy."""
    x = randn((2, 3, 480, 640), seed=5)
    want = F.interpolate(x, scale_factor=1.001, mode="bilinear", align_corners=False)
    assert torch.equal(want, x)
    s = ir.factor_scale(1.001)
    got = ir.resize(x.numpy(), 480, 640, s, s)
    assert np.array_equal(got.view(np.uint32), x.numpy().view(np.uint32))
    assert (ir.lin_taps(480, 480, s)[3] != 0).any()          # the same scale without the rule resamples
    # one axis changes size (480 x 641): W is interpolated with 1/s, H is still copied
    want = F.interpolate(x, scale_factor=1.0018, mode="bilinear", align_corners=False).numpy()
    assert want.shape[-2:] == (480, 641)
    s = ir.factor_scale(1.0018)
    assert ir.effective_scales(480, 640, 480, 641, s, s) == (F32(1), s)
    got = ir.resize(x.numpy(), 480, 641, s, s, fma=True)
    d = bilinear_ulps(got, want, x.numpy(), (480, 641), F32(1), s, True)
    print(f"one axis resized: max {d:g} ulp")
    assert d <= MAX_ULPS
    i0, i1, l0, l1 = ir.lin_taps(480, 480, s, fma=True)
    both = l0[:, None] * got[..., i0, :] + l1[:, None] * got[..., i1, :]     # H interpolated as well: not what ATen does
    assert np.abs(both - want).max() > 1e-3
    # uint8 input with "/255": the copy is float(u8) / 255, as parse_input computes it on the CPU
    u8 = torch.randint(0, 256, (1, 3, 64, 96), dtype=torch.uint8, generator=torch.Generator().manual_seed(6))
    got = ir.resize(u8.numpy(), 64, 96, s, s, div255=True)
    assert np.array_equal(got, (u8 / 255).numpy())


def test_div255_matches_parse_input():
    """parse_input's `tensor / 255` (ATen CPU true division) is the kernels' per-tap __fdiv_rn(float(u8), 255)."""
    u8 = np.arange(256, dtype=np.uint8)
    assert np.array_equal((torch.from_numpy(u8) / 255).numpy().view(np.uint32), ir.values(u8, True).view(np.uint32))


@pytest.mark.parametrize("C", [1, 3, 4, 5])
def test_gray_is_channel_sum_over_C(C):
    x = randn((2, C, 64, 96), seed=C)
    g = ir.gray(x.numpy(), 64, 96)
    want = x.numpy()[:, 0].copy()
    for c in range(1, C):
        want = want + x.numpy()[:, c]
    if C != 1:
        want = want / F32(C)
    assert np.array_equal(g, want)
    assert np.abs(ir.gray_f64(x.numpy(), 64, 96) - x.numpy().astype(np.float64).mean(1)).max() < 1e-6


@pytest.mark.parametrize("kind", ["randn", "assets_like", "low_contrast", "constant"])
def test_instnorm_matches_torch_f64(kind):
    g = torch.Generator().manual_seed(11)
    if kind == "randn":
        x = torch.randn(3, 96, 128, generator=g)
    elif kind == "assets_like":
        x = torch.rand(3, 96, 128, generator=g)
    elif kind == "low_contrast":
        x = 200 + 0.01 * torch.randn(3, 96, 128, generator=g)     # sum_sq / n - mean^2 cancels to 1e-4 of 4e4
    else:
        x = torch.full((3, 96, 128), 0.37)
    gx = x.numpy().astype(F32)
    want = F.instance_norm(torch.from_numpy(gx).double()[:, None], eps=1e-5)[:, 0].numpy()
    ref = ir.instnorm_f64(gx)
    assert np.abs(ref - want).max() < 1e-10
    stats = ir.stats_f64(gx)
    got = ir.instnorm_f32(gx, stats)
    err = np.abs(got.astype(np.float64) - ref)
    bound = ir.instnorm_f32_bound(gx, stats)
    print(f"instnorm {kind}: max err {err.max():.3g}, max bound {bound.max():.3g}")
    assert (err <= bound).all()
    if kind == "constant":
        assert (got == 0).all()
