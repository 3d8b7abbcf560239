"""Halo-patch variant of the wgmma conv (3x3 stride 1): taps addressed by shifting the shared-memory descriptor."""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import xfeat_oracle as orc  # noqa: E402


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@contextlib.contextmanager
def conv_impl(xf, impl, mode=0):
    old = xf._lib.xfeat_get_conv_impl()
    xf._lib.xfeat_set_conv_impl(impl)
    xf._lib.xfeat_set_halo_desc_mode(mode)
    try:
        yield
    finally:
        xf._lib.xfeat_set_conv_impl(old)
        xf._lib.xfeat_set_halo_desc_mode(0)


def relerr(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


CASES = [(8, "block3.1", 60, 80), (8, "block3.1", 13, 21), (17, "block_fusion.0", 36, 48), (11, "block4.1", 30, 40),
         (12, "block4.2", 15, 20), (5, "block2.0", 120, 160), (6, "block2.1", 9, 13), (8, "block3.1", 156, 208),
         (2, "block1.2", 240, 320), (2, "block1.2", 11, 27)]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"L{c[0]}_{c[2]}x{c[3]}")
def test_halo_layer_vs_oracle(xf, oracle_state, case, mode):
    from accelerated_features_b200 import _lib
    layer, prefix, H, W = case
    sd = oracle_state
    cout, cin = sd[prefix + ".layer.0.weight"].shape[:2]
    g = torch.Generator().manual_seed(layer * 1000 + H)
    B = 3
    x = torch.randn(B, cin, H, W, generator=g) * 2.0
    want = orc._basic_layer(sd, prefix, x, 1, 1)
    xin = x.permute(0, 2, 3, 1).contiguous().cuda()
    out = torch.zeros((B, H, W, cout), device="cuda")
    scratch = torch.empty(B * H * W * 512, dtype=torch.uint8, device="cuda")
    with conv_impl(xf, 2, mode):
        _lib.check(xf._lib.xfeat_debug_conv_layer_tc(xf._ctx, layer, xin.data_ptr(), B, H, W, out.data_ptr(), scratch.data_ptr(),
                                                     scratch.numel(), torch.cuda.current_stream().cuda_stream), "conv_tc_halo")
        torch.cuda.synchronize()
    err = relerr(out.permute(0, 3, 1, 2).cpu(), want)
    print(f"halo mode {mode} {prefix} {H}x{W}: rel err {err:.2e}")
    if mode == 0:
        assert err < 1e-5, (prefix, err)     # shifted descriptor, base_offset 0: correct (swizzle follows physical address bits)
    elif layer != 2:
        assert err > 1e-2                    # base_offset = (addr>>7)&7 double-applies the phase: documented negative result


def test_halo_net_and_e2e(xf, oracle_state, assets_vga):
    ref, tgt = assets_vga
    x = torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0)
    want = orc.detect_and_compute(oracle_state, x, 4096)
    with conv_impl(xf, 2, 0):
        got = xf.detectAndCompute(x, top_k=4096)
    for b in range(2):
        gs = {(float(a), float(c)) for a, c in got[b]["keypoints"].cpu().numpy()}
        ws_ = {(float(a), float(c)) for a, c in want[b]["keypoints"].numpy()}
        frac = len(gs & ws_) / len(ws_)
        print(f"halo e2e image {b}: common keypoints {frac:.4f}")
        assert frac >= 0.995
