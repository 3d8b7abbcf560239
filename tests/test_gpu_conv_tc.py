"""wgmma implicit-GEMM conv (64->64, 3x3 / 1x1, stride 1; split-fp16 operands, fp32 accumulation) against the oracle,
layer by layer, through the whole network, and end to end."""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import xfeat_oracle as orc  # noqa: E402


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@contextlib.contextmanager
def conv_impl(xf, impl):
    old = xf._lib.xfeat_get_conv_impl()
    xf._lib.xfeat_set_conv_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_conv_impl(old)


def relerr(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


CASES = [  # (layer id, oracle prefix, basic layer?, H_in, W_in, pad, stride)
    (8, "block3.1", True, 60, 80, 1, 1), (8, "block3.1", True, 13, 21, 1, 1), (8, "block3.1", True, 8, 16, 1, 1),
    (9, "block3.2", True, 60, 80, 0, 1), (11, "block4.1", True, 30, 40, 1, 1), (12, "block4.2", True, 15, 20, 1, 1),
    (17, "block_fusion.0", True, 36, 48, 1, 1), (19, "block_fusion.2", False, 12, 16, 0, 1),
    (20, "heatmap_head.0", True, 7, 130, 0, 1), (25, "keypoint_head.2", True, 60, 80, 0, 1),
    # channel-padded (24 -> 32) and strided (TMA element strides) variants
    (5, "block2.0", True, 120, 160, 1, 1), (6, "block2.1", True, 24, 40, 1, 1), (5, "block2.0", True, 9, 13, 1, 1),
    (7, "block3.0", True, 120, 160, 1, 2), (7, "block3.0", True, 24, 40, 1, 2),
    (10, "block4.0", True, 60, 80, 1, 2), (10, "block4.0", True, 20, 80, 1, 2),
    (13, "block5.0", True, 30, 40, 1, 2), (13, "block5.0", True, 10, 40, 1, 2),
    # 128 input channels: weights streamed per tap
    (14, "block5.1", True, 15, 20, 1, 1), (15, "block5.2", True, 5, 7, 1, 1), (16, "block5.3", True, 15, 20, 0, 1),
    (14, "block5.1", True, 39, 52, 1, 1),
    # stem tail: 8 input channels, 32-byte operand rows (SWIZZLE_32B), stride 2 (skip branch is covered by the net tests)
    (3, "block1.3", True, 240, 320, 1, 2), (3, "block1.3", True, 22, 38, 1, 2),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"L{c[0]}_{c[1]}_{c[3]}x{c[4]}s{c[6]}")
def test_conv_tc_layer_vs_oracle(xf, oracle_state, case):
    from accelerated_features_b200 import _lib
    layer, prefix, basic, H, W, pad, stride = case
    sd = oracle_state
    wkey = prefix + (".layer.0.weight" if basic else ".weight")
    cout, cin = sd[wkey].shape[0], sd[wkey].shape[1]
    g = torch.Generator().manual_seed(layer * 1000 + H)
    B = 3
    x = torch.randn(B, cin, H, W, generator=g) * 2.0
    x[0, :, 0, 0] = 0.0                      # exact zeros and tiny values exercise the lo-term range
    x[1, :, -1, -1] *= 1e-3
    want = orc._basic_layer(sd, prefix, x, stride, pad) if basic else F.conv2d(x, sd[prefix + ".weight"], sd[prefix + ".bias"])
    Ho, Wo = want.shape[2], want.shape[3]
    xin = x.permute(0, 2, 3, 1).contiguous().cuda()
    out = torch.empty((B, Ho, Wo, cout), device="cuda")
    scratch = torch.empty(B * H * W * 512, dtype=torch.uint8, device="cuda")
    _lib.check(xf._lib.xfeat_debug_conv_layer_tc(xf._ctx, layer, xin.data_ptr(), B, H, W, out.data_ptr(), scratch.data_ptr(),
                                                 scratch.numel(), torch.cuda.current_stream().cuda_stream), "conv_tc")
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2).cpu()
    err = relerr(got, want)
    print(f"{prefix} {H}x{W} s{stride}: rel err {err:.2e}")
    assert err < 1e-5, (prefix, err)         # 3-term fp16 split: ~2^-21 operand error + fp32 accumulation


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("which", ["g3_small", "vga"])
def test_net_tc_vs_oracle(xf, oracle_state, golden, assets_vga, which, impl):
    """impl 2: the tensor-core schedule.  impl 1 has no schedule of its own: like every value but 0 it selects the tensor-core
    schedule, reported as 2, with bit-identical outputs."""
    if which == "g3_small":
        x = torch.from_numpy(golden("g3_randn_small.npz")["x"])
    else:
        ref, tgt = assets_vga
        x = torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0)
    st = orc.backbone(oracle_state, x)
    B, _, H, W = x.shape
    xn = st["xn"][:, 0].contiguous().cuda()
    with conv_impl(xf, impl):
        assert xf._lib.xfeat_get_conv_impl() == 2
        feats, heat, rel, logits = xf._run_net(xn, B, H, W, want_logits=True)
        torch.cuda.synchronize()
    if impl != 2:
        with conv_impl(xf, 2):
            default = xf._run_net(xn, B, H, W, want_logits=True)
            torch.cuda.synchronize()
        for name, a, b in zip(("feats", "heat", "reliability", "logits"), (feats, heat, rel, logits), default):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"impl {impl}: {name} differs from the default schedule"
    with conv_impl(xf, 0):
        feats0, heat0, rel0, logits0 = xf._run_net(xn, B, H, W, want_logits=True)
        torch.cuda.synchronize()
    e_feats = relerr(feats.permute(0, 3, 1, 2).cpu(), st["feats"])
    e_log = (logits.permute(0, 3, 1, 2).cpu() - st["kpt_logits"]).abs().max().item()
    e_rel = (rel.cpu() - st["reliability"][:, 0]).abs().max().item()
    e_heat = (heat.cpu() - orc.kpts_heatmap(st["kpt_logits"])[:, 0]).abs().max().item()
    print(f"[{which}] tensor-core impl {impl}: feats rel {e_feats:.2e} logits abs {e_log:.2e} reliability abs {e_rel:.2e} heat abs {e_heat:.2e}; "
          f"vs simt feats rel {relerr(feats, feats0):.2e}")
    # 3-term fp16 split carries 22 mantissa bits per operand (fp32: 24): a few 1e-5 after ~20 layers, 1e-3 is the budget
    assert e_feats < 1e-4 and e_log < 5e-4 and e_rel < 5e-5 and e_heat < 5e-5


def test_e2e_tc_detect_and_match(xf, oracle_state, assets_vga, golden):
    ref, tgt = assets_vga
    x = torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0)
    want = orc.detect_and_compute(oracle_state, x, 4096)
    got = xf.detectAndCompute(x, top_k=4096)
    mk0, mk1 = xf.match_xfeat(ref, tgt, top_k=4096)
    for b in range(2):
        gk, wk = got[b]["keypoints"].cpu().numpy(), want[b]["keypoints"].numpy()
        gs = {(float(a), float(c)) for a, c in gk}; ws_ = {(float(a), float(c)) for a, c in wk}
        common = gs & ws_
        frac = len(common) / len(wk)
        gi = {(float(a), float(c)): i for i, (a, c) in enumerate(gk)}
        wi = {(float(a), float(c)): i for i, (a, c) in enumerate(wk)}
        ia = np.array([gi[c] for c in common]); ib = np.array([wi[c] for c in common])
        derr = np.abs(got[b]["descriptors"].cpu().numpy()[ia] - want[b]["descriptors"].numpy()[ib]).max()
        print(f"tensor-core convs, image {b}: common keypoints {len(common)}/{len(wk)} ({frac:.4f}), desc max err {derr:.2e}")
        assert frac >= 0.995 and derr < 1e-3
    g = golden("g1_sparse_vga.npz")
    wantm = {(float(a), float(b), float(c), float(d)) for (a, b), (c, d) in zip(g["mkpts0"], g["mkpts1"])}
    gotm = {(float(a), float(b), float(c), float(d)) for (a, b), (c, d) in zip(mk0, mk1)}
    frac = len(wantm & gotm) / len(wantm)
    print(f"tensor-core convs: matches {len(gotm)} vs golden {len(wantm)}, common {frac:.4f}")
    assert frac >= 0.98


def test_star_tc(xf, assets_vga, golden):
    ref, tgt = assets_vga
    g = golden("g4_star_vga.npz")
    a0, a1 = xf.match_xfeat_star(ref, tgt, top_k=4096)
    want0, want1 = g["b1_mk0"], g["b1_mk1"]
    wd = {(float(r[0]), float(r[1])): s for r, s in zip(want1, want0)}
    hit = sum(1 for s, r in zip(a0, a1) if (float(r[0]), float(r[1])) in wd and np.abs(wd[(float(r[0]), float(r[1]))] - s).max() < 0.05)
    print(f"star (tensor-core convs): {len(a0)} vs {len(want0)} refined matches, agreeing {hit}")
    assert hit >= 0.95 * len(want0)
