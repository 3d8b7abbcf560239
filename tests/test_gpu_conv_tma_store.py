"""The wgmma convolution kernels write their outputs as TMA tensor-store boxes {channels, TW, TH, 1}.  A box the TMA places
outside its tensor overwrites memory silently, so these cases put the fp32 and split outputs inside larger buffers whose
margins hold a sentinel, and check that the margins survive and that the outputs are bit-identical to a run into plain
buffers.  They cover the tile-count edges and layers of test_gpu_conv_overlap.py: ragged tiles, one tile, 2 * grid + 1 tiles,
block5.0's two N tiles, and 8-, 24-, 64- and 128-channel layers, the 8-channel one (block1.2) on the halo kernel.  Output
pointers that are not 16-byte aligned are refused with an error."""
import pytest
import torch

from tests import split_ref as sr
from tests.test_gpu_conv_overlap import LAYERS, ONE_TILE

MARGIN = 4096   # elements before and after each output (16-byte multiples for both dtypes)
CASES = LAYERS + [(2, "halo", "halo 8-ch")]


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def geometry(sd, layer):
    from accelerated_features_b200 import weights
    ks, stride, _, _ = sr.layer_geometry(layer)
    cout, cin = sd[weights.LAYERS[layer][0] + ".weight"].shape[:2]
    cinp = 8 if cin <= 8 else (32 if cin <= 32 else (64 if cin <= 64 else 128))
    cs = 8 if (cin == 8 and cout == 8) else (32 if cout == 24 else cout)
    return stride, cin, cout, cinp, cs


def call(xf, layer, x, B, H, W, out_ptr, split_ptr, skip, scratch):
    rc = xf._lib.xfeat_debug_conv_layer_tc_ex(xf._ctx, layer, x.data_ptr(), B, H, W, out_ptr, split_ptr,
                                               None if skip is None else skip.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                               torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def inputs(layer, B, Ho, Wo, stride, cin, cinp):
    H, W = Ho * stride, Wo * stride
    g = torch.Generator(device="cuda").manual_seed(layer * 7919 + B * 31 + Ho)
    x = torch.randn(B, H, W, cin, generator=g, device="cuda") * 2.0
    skip = torch.randn(B, 4 * Ho, 4 * Wo, generator=g, device="cuda") if layer == 3 else None
    scratch = torch.empty(B * H * W * 4 * cinp, dtype=torch.uint8, device="cuda")
    return H, W, x, skip, scratch


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[2].replace(" ", "_"))
@pytest.mark.parametrize("edge", ["one_tile", "fewer_tiles_than_ctas", "waves_plus_one", "ragged"])
def test_outputs_stay_inside_their_tensors(xf, oracle_state, sms, case, edge):
    from accelerated_features_b200 import _lib
    layer, family, _ = case
    ho, wo = ONE_TILE[family]
    B = {"one_tile": 1, "fewer_tiles_than_ctas": 3, "waves_plus_one": 2 * sms + 1, "ragged": 5}[edge]
    if edge == "ragged":
        ho, wo = 37, 53
    stride, cin, cout, cinp, cs = geometry(oracle_state, layer)
    H, W, x, skip, scratch = inputs(layer, B, ho, wo, stride, cin, cinp)
    n_out, n_split = B * ho * wo * cout, B * ho * wo * 2 * cs
    out_buf = torch.full((n_out + 2 * MARGIN,), -12345.0, device="cuda")
    split_buf = torch.full((n_split + 2 * MARGIN,), -1234.0, dtype=torch.float16, device="cuda")
    out_keep, split_keep = out_buf.clone(), split_buf.clone()
    _lib.check(call(xf, layer, x, B, H, W, out_buf[MARGIN:].data_ptr(), split_buf[MARGIN:].data_ptr(), skip, scratch),
               "conv_tc_ex")
    for buf, keep, n, name in ((out_buf, out_keep, n_out, "fp32"), (split_buf, split_keep, n_split, "split")):
        assert torch.equal(buf[:MARGIN], keep[:MARGIN]), f"{name} output: write before the tensor"
        assert torch.equal(buf[MARGIN + n:], keep[MARGIN + n:]), f"{name} output: write past the tensor"

    out = torch.empty(B, ho, wo, cout, device="cuda")
    split = torch.empty(B, ho, wo, 2 * cs, dtype=torch.float16, device="cuda")
    _lib.check(call(xf, layer, x, B, H, W, out.data_ptr(), split.data_ptr(), skip, scratch), "conv_tc_ex")
    assert torch.equal(out_buf[MARGIN:MARGIN + n_out].view(torch.int32), out.reshape(-1).view(torch.int32))
    assert torch.equal(split_buf[MARGIN:MARGIN + n_split].view(torch.int16), split.reshape(-1).view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(8, "halo"), (9, "conv_tc"), (14, "conv_tc128")], ids=lambda c: c[1])
@pytest.mark.parametrize("which", ["fp32", "split"])
def test_misaligned_output_is_an_error(xf, oracle_state, case, which):
    layer, _ = case
    stride, cin, cout, cinp, cs = geometry(oracle_state, layer)
    B, ho, wo = 1, 8, 16
    H, W, x, skip, scratch = inputs(layer, B, ho, wo, stride, cin, cinp)
    out = torch.zeros(B * ho * wo * cout + 64, device="cuda")
    split = torch.zeros(B * ho * wo * 2 * cs + 64, dtype=torch.float16, device="cuda")
    out_ptr, split_ptr = out.data_ptr(), split.data_ptr()
    if which == "fp32":
        out_ptr += 4
    else:
        split_ptr += 2
    rc = call(xf, layer, x, B, H, W, out_ptr, split_ptr, skip, scratch)
    assert rc != 0
    assert "16-byte aligned" in xf._lib.xfeat_last_error().decode()
    assert bool((out == 0).all() and (split == 0).all()), "a refused call wrote its outputs"
