"""Tile-count edges of the wgmma convolution kernels, whose consumer keeps one wgmma group in flight across pipeline stages
(conv_tc_kernel with >= 3 stages; the hi and lo passes of the 64-channel halo kernel) and whose epilogues read the accumulator
32 channels at a time: a single tile, fewer tiles than CTAs, one tile more than a whole number of waves, a ragged last tile
and block5.0's two N tiles.  Each case compares against float64 with the split_ref tolerance, checks the split output bit for
bit and the padded channels for exact zeros.  The CPU test reads the ptxas logs of the build."""
import glob
import os
import re

import pytest
import torch

from tests import split_ref as sr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_layer(xf, sd, layer, B, Ho, Wo):
    from accelerated_features_b200 import _lib, weights
    ks, stride, _, _ = sr.layer_geometry(layer)
    cout, cin = sd[weights.LAYERS[layer][0] + ".weight"].shape[:2]
    H, W = Ho * stride, Wo * stride
    cinp = 8 if cin <= 8 else (32 if cin <= 32 else (64 if cin <= 64 else 128))
    cs = 8 if (cin == 8 and cout == 8) else (32 if cout == 24 else cout)
    g = torch.Generator(device="cuda").manual_seed(layer * 7919 + B * 31 + Ho)
    x = torch.randn(B, H, W, cin, generator=g, device="cuda") * 2.0
    skip = torch.randn(B, 4 * Ho, 4 * Wo, generator=g, device="cuda") if layer == 3 else None
    out = torch.full((B, Ho, Wo, cout), float("nan"), device="cuda")
    split = torch.full((B, Ho, Wo, 2 * cs), float("nan"), dtype=torch.float16, device="cuda")
    scratch = torch.empty(B * H * W * 4 * cinp, dtype=torch.uint8, device="cuda")
    _lib.check(xf._lib.xfeat_debug_conv_layer_tc_ex(xf._ctx, layer, x.data_ptr(), B, H, W, out.data_ptr(), split.data_ptr(),
                                                    None if skip is None else skip.data_ptr(), scratch.data_ptr(),
                                                    scratch.numel(), torch.cuda.current_stream().cuda_stream), "conv_tc_ex")
    torch.cuda.synchronize()
    xc = x.permute(0, 3, 1, 2)
    ref = sr.reference(sd, layer, xc, skip)
    got = out.permute(0, 3, 1, 2)
    assert torch.isfinite(got).all()
    err = float((got.double() - ref).abs().max() / ref.abs().max())
    assert err < sr.CONV_TC_TOL, f"layer {layer} B={B} {Ho}x{Wo}: error {err:.3e} >= {sr.CONV_TC_TOL:.1e}"
    hi, lo = split[..., :cs], split[..., cs:]
    want_hi = out.half()
    want_lo = (out - want_hi.float()).half()
    assert torch.equal(hi[..., :cout].view(torch.int16), want_hi.view(torch.int16)), "hi half differs"
    assert torch.equal(lo[..., :cout].view(torch.int16), want_lo.view(torch.int16)), "lo half differs"
    if cs > cout:
        assert bool((hi[..., cout:] == 0).all() and (lo[..., cout:] == 0).all()), "padded channels are not zero"


# (layer, kernel family, name): the halo kernels and each conv_tc / conv_tc128 instantiation; "3x3 64-ch per tap" is block4.0
# (conv_tc_kernel<3,64,64>, stride 2)
LAYERS = [
    (5, "halo", "halo 32-ch"), (8, "halo", "halo 64-ch"), (9, "conv_tc", "1x1 64-ch"), (10, "conv_tc", "3x3 64-ch per tap"),
    (7, "conv_tc", "3x3 stride 2 32->64"), (3, "conv_tc", "stem tail + skip1"), (13, "conv_tc", "block5.0 two N tiles"),
    (14, "conv_tc", "128-ch 3x3"), (16, "conv_tc", "128-ch 1x1"),
]
# output sizes of ONE tile per image: 4 x 8 fits the smallest halo tile (TW 8, TH 12), 8 x 16 one 128-pixel conv_tc tile
ONE_TILE = {"halo": (4, 8), "conv_tc": (8, 16)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", LAYERS, ids=lambda c: c[2].replace(" ", "_"))
@pytest.mark.parametrize("edge", ["one_tile", "fewer_tiles_than_ctas", "waves_plus_one", "ragged"])
def test_tile_count_edges(xf, oracle_state, sms, case, edge):
    layer, family, _ = case
    ho, wo = ONE_TILE[family]
    if edge == "one_tile":
        B = 1
    elif edge == "fewer_tiles_than_ctas":
        B = 3
    elif edge == "waves_plus_one":
        B = 2 * sms + 1        # one tile per image: n_tiles = 2 * grid + 1, so the first CTA runs one tile more than the rest
    else:
        B, ho, wo = 5, 37, 53  # neither dimension a multiple of any tile shape
    run_layer(xf, oracle_state, layer, B, ho, wo)


def test_build_logs_no_serialised_wgmma_or_epilogue_spills():
    """ptxas reports for the wgmma convolution kernels: no wgmma serialisation (C7519 / C7520) and, since the epilogues stopped
    copying all accumulator columns, at most a few bytes of spill stores (the copy used to spill 192-260 B)."""
    logs = {os.path.basename(p): open(p).read() for p in glob.glob(os.path.join(ROOT, "accelerated_features_b200", "build", "*.o.log"))}
    if not {"conv_tc.o.log", "conv_tc_halo.o.log", "head_chain_tc.o.log"} <= set(logs):
        from accelerated_features_b200.build import build_library
        build_library(force=True)
        logs = {n: open(os.path.join(ROOT, "accelerated_features_b200", "build", n)).read()
                for n in ("conv_tc.o.log", "conv_tc_halo.o.log", "head_chain_tc.o.log")}
    for name in ("conv_tc.o.log", "conv_tc_halo.o.log", "head_chain_tc.o.log"):
        text = logs[name]
        assert "C7519" not in text and "C7520" not in text, f"{name}: ptxas serialises wgmma:\n" + "\n".join(
            l for l in text.splitlines() if "C75" in l)
        kernels = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes spill stores", text, re.S)
        assert kernels, f"{name}: no ptxas -v output"
        for fn, spill in kernels:
            limit = 0 if ("halo" in fn or "head_chain" in fn) else 16
            assert int(spill) <= limit, f"{name}: {fn} spills {spill} B (limit {limit})"
