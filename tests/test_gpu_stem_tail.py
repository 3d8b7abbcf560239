"""The fused stem tail (stem_tail_halo_kernel: block1.2, then block1.3 + skip1, with block1.2's output kept in shared memory)
against the per-layer tensor-core kernels it replaces in xfeat_net: xfeat_debug_conv_layer_tc_ex for block1.2 (fp32 out), then
for block1.3 with the skip input (split out).  The split x1s must match bit for bit, and its padded channels 24-31 must be
exact zeros, at the production shapes, at partial tiles on the right and bottom edges, on an image narrower than one tile,
and on inputs with exact zeros and constant images (where out-of-image a3 positions differ from relu(bias))."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


def make_inputs(kind, B, H2, W2, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "constant":
        x = torch.full((B, H2, W2, 8), 0.75, device="cuda")
        xn = torch.full((B, 2 * H2, 2 * W2), -0.3, device="cuda")
        return x, xn
    x = torch.relu(torch.randn(B, H2, W2, 8, generator=g, device="cuda") * 2.0)
    xn = torch.randn(B, 2 * H2, 2 * W2, generator=g, device="cuda")
    if kind == "zeros":   # whole zero pixels, a zero band through every image, and a zero patch of the gray image
        x[torch.rand(B, H2, W2, generator=g, device="cuda") < 0.3] = 0.0
        x[:, H2 // 3: H2 // 3 + 5] = 0.0
        x[:, :, :7] = 0.0
        xn[:, : 2 * H2 // 2, : 2 * W2 // 3] = 0.0
    return x, xn


def two_kernel_chain(xf, x, xn):
    from accelerated_features_b200 import _lib
    B, H2, W2, _ = x.shape
    st = torch.cuda.current_stream().cuda_stream
    scratch = torch.empty(B * H2 * W2 * 32, dtype=torch.uint8, device="cuda")
    a3 = torch.empty(B, H2, W2, 8, device="cuda")
    out = torch.full((B, H2 // 2, W2 // 2, 64), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(xf._lib.xfeat_debug_conv_layer_tc_ex(xf._ctx, 2, x.data_ptr(), B, H2, W2, a3.data_ptr(), None, None,
                                                    scratch.data_ptr(), scratch.numel(), st), "block1.2")
    _lib.check(xf._lib.xfeat_debug_conv_layer_tc_ex(xf._ctx, 3, a3.data_ptr(), B, H2, W2, None, out.data_ptr(), xn.data_ptr(),
                                                    scratch.data_ptr(), scratch.numel(), st), "block1.3")
    return out


def fused(xf, x, xn):
    from accelerated_features_b200 import _lib
    B, H2, W2, _ = x.shape
    scratch = torch.empty(B * H2 * W2 * 32, dtype=torch.uint8, device="cuda")
    out = torch.full((B, H2 // 2, W2 // 2, 64), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(xf._lib.xfeat_debug_stem_tail(xf._ctx, x.data_ptr(), xn.data_ptr(), B, H2, W2, out.data_ptr(), scratch.data_ptr(),
                                             scratch.numel(), torch.cuda.current_stream().cuda_stream), "stem tail")
    return out


# (B, H2, W2): half-resolution shapes (block1.1's output); x1s is (H2/2, W2/2) in tiles of 8 x 15
SHAPES = [
    (2, 240, 320),    # VGA
    (2, 288, 384),    # star, 768 x 576
    (1, 624, 832),    # star, 1664 x 1248
    (3, 22, 38),      # 11 x 19 outputs: partial tiles on the right and at the bottom
    (2, 34, 30),      # 17 x 15: a partial bottom row of tiles
    (2, 16, 16),      # 8 x 8: narrower than one tile
    (2, 16, 64),      # 8 x 32: a ragged last tile column
]


@pytest.mark.parametrize("kind", ["relu_randn", "zeros", "constant"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B{}_{}x{}".format(*s))
def test_stem_tail_matches_two_kernels(xf, shape, kind):
    assert xf._lib.xfeat_get_conv_impl() == 2
    B, H2, W2 = shape
    x, xn = make_inputs(kind, B, H2, W2, seed=B * 7919 + H2 * 31 + W2)
    want = two_kernel_chain(xf, x, xn)
    got = fused(xf, x, xn)
    torch.cuda.synchronize()
    gb, wb = got.view(torch.int16), want.view(torch.int16)
    assert torch.equal(gb, wb), f"{int((gb != wb).any(-1).sum())} of {gb[..., 0].numel()} pixels differ"
    assert bool((gb[..., 24:32] == 0).all() and (gb[..., 56:64] == 0).all()), "padded channels 24-31 are not +0"
    assert bool((gb[..., :24] != 0).any()), "no nonzero output"


def test_stem_tail_production_batch(xf):
    """bench.py's backbone batch: 128 VGA images, 21 120 tiles over the persistent grid."""
    B, H2, W2 = 128, 240, 320
    x, xn = make_inputs("relu_randn", B, H2, W2, seed=128)
    want = two_kernel_chain(xf, x, xn)
    got = fused(xf, x, xn)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    assert bool((got.view(torch.int16)[..., 24:32] == 0).all() and (got.view(torch.int16)[..., 56:64] == 0).all())
