"""What xfeat_net runs after block_fusion.1 (xfeat_debug_heads variant 1: head_chain_rf_kernel<1>, block_fusion.2 and the
reliability head in one kernel, and head_chain_rf_kernel<0>, the keypoint head; activations handed from layer to layer in
registers, two warpgroups per CTA on independent tiles) against the separate kernels (variant 0: block_fusion.2 on
conv_tc_kernel<1,64,64>, then head_chain_kernel<1> and head_chain_kernel<0>, which keep each layer's activations in shared
memory).  feats, reliability, heat and the raw keypoint logits must match bit for bit: at the production batch (many tiles
per warpgroup, so the ring, cp.async and store-piece parities wrap), at both star scales, on a ragged last tile, with fewer
tiles than SMs, on a grid smaller than one tile (one warpgroup idle), and on inputs with many exact zeros and on constant
inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


def make_inputs(kind, B, Hc, Wc, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "constant":
        return (torch.full((B, Hc, Wc, 64), 0.75, device="cuda"),
                torch.full((B, 8 * Hc, 8 * Wc), -0.3, device="cuda"))
    f1 = torch.relu(torch.randn(B, Hc, Wc, 64, generator=g, device="cuda") * 2.0)
    xn = torch.randn(B, 8 * Hc, 8 * Wc, generator=g, device="cuda")
    if kind == "zeros":   # whole zero cells, a zero band through every image, and a zero patch of the gray image
        f1[torch.rand(B, Hc, Wc, generator=g, device="cuda") < 0.3] = 0.0
        f1[:, Hc // 3: Hc // 3 + 2] = 0.0
        xn[:, : 4 * Hc, : 8 * Wc // 3] = 0.0
    return f1, xn


def run_heads(xf, variant, f1, xn):
    from accelerated_features_b200 import _lib
    B, Hc, Wc, _ = f1.shape
    npix = B * Hc * Wc
    scratch = torch.empty(npix * 512, dtype=torch.uint8, device="cuda")
    nan = float("nan")
    feats = torch.full((B, Hc, Wc, 64), nan, device="cuda")
    heat = torch.full((B, 8 * Hc, 8 * Wc), nan, device="cuda")
    rel = torch.full((npix,), nan, device="cuda")
    logits = torch.full((npix, 65), nan, device="cuda")
    _lib.check(xf._lib.xfeat_debug_heads(xf._ctx, variant, f1.data_ptr(), xn.data_ptr(), B, Hc, Wc, feats.data_ptr(),
                                         heat.data_ptr(), rel.data_ptr(), logits.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                         torch.cuda.current_stream().cuda_stream), f"heads variant {variant}")
    return {"feats": feats, "heat": heat, "reliability": rel, "logits": logits}


def assert_same_bits(xf, f1, xn):
    want = run_heads(xf, 0, f1, xn)
    got = run_heads(xf, 1, f1, xn)
    torch.cuda.synchronize()
    for name in want:
        w, g = want[name].view(torch.int32), got[name].view(torch.int32)
        assert not torch.isnan(want[name]).any(), f"{name}: reference left unwritten values"
        assert torch.equal(g, w), f"{name}: {int((g != w).sum())} of {w.numel()} values differ"


# (B, Hc, Wc) in 1/8-resolution cells
SHAPES = [
    (2, 60, 80),      # VGA
    (2, 72, 96),      # star, 768 x 576
    (1, 156, 208),    # star, 1664 x 1248
    (52, 28, 36),     # 52 416 cells: a ragged last tile
    (1, 60, 80),      # B = 1 at VGA: 38 tiles, fewer than SMs
    (1, 5, 7),        # 35 cells: a grid smaller than one tile, the CTA's second warpgroup idle
]


@pytest.mark.parametrize("kind", ["relu_randn", "zeros", "constant"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B{}_{}x{}".format(*s))
def test_heads_match_reference(xf, shape, kind):
    assert xf._lib.xfeat_get_conv_impl() == 2
    B, Hc, Wc = shape
    f1, xn = make_inputs(kind, B, Hc, Wc, seed=B * 7919 + Hc * 31 + Wc)
    assert_same_bits(xf, f1, xn)


def test_heads_production_batch(xf):
    """bench.py's backbone batch: 128 VGA images, 4 800 tiles over the persistent grid."""
    f1, xn = make_inputs("relu_randn", 128, 60, 80, seed=128)
    assert_same_bits(xf, f1, xn)
