"""GPU parity of the reference's helper surface (SURVEY 8b) and of the round-2 API additions: every helper method of
modules/xfeat.py that callers may use directly, mixed numpy / tensor inputs, the streaming pipeline, the NMS overflow status,
and two devices in one process."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import xfeat_oracle as orc  # noqa: E402
from tests import split_ref  # noqa: E402


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


def test_is_module_with_reference_attributes(xf):
    import torch.nn as nn
    assert isinstance(xf, nn.Module) and isinstance(xf.net, nn.Module) and isinstance(xf.net.fine_matcher, nn.Module)
    assert isinstance(xf.interpolator, nn.Module) and xf.interpolator.mode == "bicubic"
    assert xf.eval() is xf and xf.top_k == 4096 and xf.detection_threshold == 0.05
    assert xf.dev.type == "cuda"


def test_preprocess_tensor(xf, assets_vga):
    ref, _ = assets_vga
    crop = np.ascontiguousarray(ref[10:310, 5:405])                                  # 300 x 400 -> 288 x 384
    want, rh, rw = orc.preprocess_tensor(crop)
    got, grh, grw = xf.preprocess_tensor(crop)
    assert (grh, grw) == (rh, rw) and got.shape == want.shape and got.dtype == torch.float32
    assert (got.cpu() - want).abs().max().item() < 2e-3                              # values up to 255 (no /255 here, xfeat.py:221-233): 1e-5 relative
    x = torch.rand(2, 3, 64, 96)
    got, grh, grw = xf.preprocess_tensor(x)                                          # identity resize still runs (xfeat.py:239)
    assert grh == 1.0 and grw == 1.0 and (got.cpu() - x).abs().max().item() < 1e-6
    with pytest.raises(RuntimeError):
        xf.preprocess_tensor(np.zeros((2, 3, 4, 5), np.float32))


def test_get_kpts_heatmap_and_nms(xf, oracle_state, assets_vga):
    ref, tgt = assets_vga
    x = torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0)
    st = orc.backbone(oracle_state, x)
    want_heat = orc.kpts_heatmap(st["kpt_logits"])
    got_heat = xf.get_kpts_heatmap(st["kpt_logits"].cuda())
    assert got_heat.shape == want_heat.shape
    assert (got_heat.cpu() - want_heat).abs().max().item() < 1e-6
    got_t = xf.get_kpts_heatmap(st["kpt_logits"].cuda(), softmax_temp=2.0)
    assert (got_t.cpu() - orc.kpts_heatmap(st["kpt_logits"], 2.0)).abs().max().item() < 1e-6
    # NMS on the ORACLE heat-map: integer output, bit-exact including the zero padding and the raster order
    want_pos = orc.nms(want_heat, 0.05, 5)
    got_pos = xf.NMS(want_heat.cuda(), threshold=0.05, kernel_size=5)
    assert got_pos.dtype == torch.long and torch.equal(got_pos.cpu(), want_pos)
    want3 = orc.nms(want_heat, 0.1, 3)
    assert torch.equal(xf.NMS(want_heat.cuda(), threshold=0.1, kernel_size=3).cpu(), want3)


def test_interpolator_modes(xf):
    from accelerated_features_b200.xfeat import InterpolateSparse2d
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 5, 12, 16, generator=g)
    pos = torch.stack([torch.randint(0, 128, (2, 50), generator=g), torch.randint(0, 96, (2, 50), generator=g)], -1)
    pos[0, 0] = torch.tensor([127, 95]); pos[0, 1] = torch.tensor([0, 0])           # borders: zero padding / rounding quirks
    for mode in ("nearest", "bilinear", "bicubic"):
        want = orc.sample_sparse(x, pos, 96, 128, mode)
        got = InterpolateSparse2d(mode)(x.cuda(), pos.cuda(), 96, 128)
        assert got.shape == want.shape
        assert (got.cpu() - want).abs().max().item() < 2e-6, mode


def test_fine_matcher_and_subpix(xf, oracle_state):
    g = torch.Generator().manual_seed(9)
    x = torch.randn(300, 128, generator=g) * 4
    want = orc.fine_matcher(oracle_state, x)
    got = xf.net.fine_matcher(x.cuda())
    assert got.shape == (300, 64)
    assert (got.cpu() - want).abs().max().item() < split_ref.FINE_MATCHER_TOL   # sees a dropped split term (test_split_error_model)
    want_xy = orc.subpix_softmax2d(want.view(-1, 8, 8))
    got_xy = xf.subpix_softmax2d(want.view(-1, 8, 8).cuda())
    assert (got_xy.cpu() - want_xy).abs().max().item() < 1e-5
    assert xf.net.fine_matcher(torch.zeros(0, 128)).shape == (0, 64)


def test_dense_helpers_and_refine_matches(xf, oracle_state, assets_vga):
    ref, tgt = assets_vga
    x = torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0)
    mk, sc, ft = xf.extract_dualscale(x, 4096)
    assert mk.shape == (2, 4095, 2) and sc.shape == (2, 4095) and ft.shape == (2, 4095, 64)
    mk1, ft1 = xf.extractDense(x, top_k=1000)
    wk1, wf1 = orc.extract_dense(oracle_state, x, 1000)
    assert mk1.shape == wk1.shape
    common = {(float(a), float(b)) for a, b in mk1[0].cpu().numpy()} & {(float(a), float(b)) for a, b in wk1[0].numpy()}
    assert len(common) >= 1000 - 2
    # top_k < 1 means "all cells" (xfeat.py:357-358)
    mk_all, _ = xf.extractDense(x, top_k=0)
    assert mk_all.shape[1] == 60 * 80
    assert torch.equal(xf.create_xy(3, 4, xf.dev).cpu(), orc.create_xy(3, 4))
    # refine_matches on the oracle's coarse features and matches
    d1 = orc.detect_and_compute_dense(oracle_state, x, 2000)
    d2 = orc.detect_and_compute_dense(oracle_state, torch.flip(x, dims=[0]), 2000)
    idxs = orc.batch_match(d1["descriptors"], d2["descriptors"])
    dd1 = {k: v.cuda() for k, v in d1.items()}
    dd2 = {k: v.cuda() for k, v in d2.items()}
    for b in range(2):
        want, stg = orc.refine_matches(oracle_state, d1, d2, idxs, b, return_stages=True)
        got = xf.refine_matches(dd1, dd2, [(i0.cuda(), i1.cuda()) for i0, i1 in idxs], b)
        borderline = int((np.abs(stg["conf"].numpy() - 0.25) <= 1e-4).sum())
        assert abs(len(got) - len(want)) <= borderline
        if borderline == 0:
            np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), atol=2e-3)


def test_mixed_numpy_and_tensor_inputs(xf, assets_vga):
    """parse_input divides numpy images by 255 and passes tensors through (xfeat.py:396-403): the flag is per image set."""
    ref, tgt = assets_vga
    t_ref = torch.from_numpy(ref).permute(2, 0, 1)[None].float() / 255
    t_tgt = torch.from_numpy(tgt).permute(2, 0, 1)[None].float() / 255
    base = xf.match_xfeat(ref, tgt, top_k=2048)
    for a, b in ((ref, t_tgt), (t_ref, tgt), (t_ref, t_tgt)):
        mk0, mk1 = xf.match_xfeat(a, b, top_k=2048)
        assert np.array_equal(mk0, base[0]) and np.array_equal(mk1, base[1])
    s0 = xf.match_xfeat_star(ref, tgt, top_k=2048)
    s1 = xf.match_xfeat_star(ref, t_tgt, top_k=2048)
    assert np.array_equal(s0[0], s1[0]) and np.array_equal(s0[1], s1[1])


def test_star_different_resolutions(xf, oracle_state, assets_vga):
    """batch_match works with K1 != K2 (xfeat.py:265-290): a small second image yields fewer coarse features."""
    ref, tgt = assets_vga
    x1 = orc.parse_input(ref)
    x2 = F.interpolate(orc.parse_input(tgt), size=(160, 224), mode="bilinear", align_corners=False)
    with torch.inference_mode():
        d1 = orc.detect_and_compute_dense(oracle_state, x1, 4096)
        d2 = orc.detect_and_compute_dense(oracle_state, x2, 4096)
        assert d1["descriptors"].shape[1] != d2["descriptors"].shape[1]
        idxs = orc.batch_match(d1["descriptors"], d2["descriptors"])
        want = orc.refine_matches(oracle_state, d1, d2, idxs, 0)
    g0, g1 = xf.match_xfeat_star(x1, x2, top_k=4096)
    assert abs(len(g0) - len(want)) <= 6
    wd = {(float(r[2]), float(r[3])): r[:2].numpy() for r in want}
    hit = sum(1 for a, b in zip(g0, g1) if (float(b[0]), float(b[1])) in wd and np.abs(wd[(float(b[0]), float(b[1]))] - a).max() < 0.05)
    assert len(want) - hit <= 6


def test_stream_equals_batch_and_single(xf, assets_vga):
    ref, tgt = assets_vga
    b1 = np.stack([ref, tgt, ref, tgt]); b2 = np.stack([tgt, ref, ref, tgt])
    single = [xf.match_xfeat(a, b, top_k=1500) for a, b in zip(b1, b2)]
    pinned = xf.pinned_like(b1.shape)
    pinned.numpy()[:] = b1
    batches = [(b1, b2), (pinned.numpy(), b2), (b1[:2], b2[:2]), (b1, b2)]     # pageable, pinned (numpy view), other shape
    outs = list(xf.match_xfeat_stream(batches, top_k=1500))
    assert len(outs) == 4 and [len(o) for o in outs] == [4, 4, 2, 4]
    for o in outs:
        for b, (mk0, mk1) in enumerate(o):
            assert np.array_equal(mk0, single[b][0]) and np.array_equal(mk1, single[b][1])
    # float tensors, (B,C,H,W), on the host and on the device
    t1 = torch.from_numpy(b1).permute(0, 3, 1, 2).float() / 255
    t2 = torch.from_numpy(b2).permute(0, 3, 1, 2).float() / 255
    o = xf.match_xfeat_batch(t1, t2.cuda(), top_k=1500)
    for b in range(4):
        assert np.array_equal(o[b][0], single[b][0]) and np.array_equal(o[b][1], single[b][1])
    assert list(xf.match_xfeat_stream([], top_k=100)) == []


def test_nms_overflow_is_reported(xf):
    """More than H*W/4 maxima above the threshold (an equal-valued plateau passes `x == local_max`, xfeat.py:252): the image
    reports XF_N_OVERFLOW instead of an arbitrary subset, and the Python layer raises."""
    from accelerated_features_b200 import _lib
    lib = _lib.load()
    B, H, W, k = 2, 64, 96, 128
    heat = torch.full((B, H, W), 0.5, device="cuda")
    heat[1] = 0.0
    heat[1, 10, 10] = 0.9                                             # image 1 is ordinary: one keypoint
    feats = torch.randn(B, H // 8, W // 8, 64, device="cuda")
    rel = torch.full((B, H // 8, W // 8), 0.7, device="cuda")
    kpts = torch.empty((B, k, 2), device="cuda"); scores = torch.empty((B, k), device="cuda")
    desc = torch.empty((B, k, 64), device="cuda"); nv = torch.empty((B,), dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.xfeat_sparse_workspace_bytes(B, H, W, k), dtype=torch.uint8, device="cuda")
    _lib.check(lib.xfeat_detect_sparse(xf._ctx, feats.data_ptr(), heat.data_ptr(), rel.data_ptr(), B, H, W, k, 0.05, 1.0, 1.0,
                                       kpts.data_ptr(), scores.data_ptr(), desc.data_ptr(), nv.data_ptr(), None, None,
                                       ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), "detect_sparse")
    assert nv.tolist() == [_lib.N_OVERFLOW, 1]
    assert float(desc[0].abs().sum()) == 0.0
    with pytest.raises(_lib.XFeatLibraryError):
        xf._check_counts(nv.tolist(), "test")
    # the matcher propagates the status instead of reporting "no matches"
    idx0, idx1, cnt = xf._mnn_device(desc, nv, k, k * 64, desc, nv, k, k * 64, B, -1, abs_bound=1.0)
    assert cnt.tolist() == [_lib.N_OVERFLOW, 1]


def test_two_devices_in_one_process(assets_vga):
    """cudaFuncAttributeMaxDynamicSharedMemorySize is per device: a second context on another GPU must launch the >48 KB
    kernels too, and creating / destroying contexts must not move the caller's current device."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from accelerated_features_b200 import XFeat
    ref, tgt = assets_vga
    cur = torch.cuda.current_device()
    a = XFeat(device=0)
    b = XFeat(device=1)
    assert torch.cuda.current_device() == cur
    ra = a.match_xfeat(ref, tgt, top_k=1024)
    rb = b.match_xfeat(ref, tgt, top_k=1024)
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
    sa = a.match_xfeat_star(ref, tgt, top_k=1024)
    sb = b.match_xfeat_star(ref, tgt, top_k=1024)
    assert np.array_equal(sa[0], sb[0])
    del b
    assert torch.cuda.current_device() == cur
