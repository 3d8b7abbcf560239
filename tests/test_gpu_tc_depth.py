"""Tensor-core kernels against float64 at production batch sizes, where every CTA of the persistent launches wraps its
shared-memory ring (the mbarrier wait parity flips on each wrap) -- the oracle comparisons elsewhere stop at one or two tiles per
CTA.  Each case first asserts its depth with split_ref.min_tiles_per_cta (a lower bound: a tile covers at most 128 pixels or
rows and a launch has at most one CTA per SM), then compares with the split_ref tolerances, and prints the emulated error of
the exact three-term split and of the split with one term dropped next to the measured error."""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import xfeat_oracle as orc  # noqa: E402
from tests import split_ref as sr  # noqa: E402
from tests.parity_util import assert_keypoints_exact_modulo_ties, assert_matches_exact_modulo_ties, match_set  # noqa: E402


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def conv_impl(xf, impl):
    old = xf._lib.xfeat_get_conv_impl()
    xf._lib.xfeat_set_conv_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_conv_impl(old)


def assert_depth(name, rows, sms, need):
    d = sr.min_tiles_per_cta(rows, sms)
    print(f"{name}: {rows} rows on {sms} SMs -> >= {d} tiles per CTA")
    assert d >= need, f"{name}: only {d} tiles per CTA guaranteed, the case needs {need}"


def report(name, err, bound, model):
    print(f"{name}: error {err:.3e} (bound {bound:.1e}); emulated {sr.fmt_model(model)}")
    assert err < bound, f"{name}: error {err:.3e} >= {bound:.1e}"


# (layer, name, B, H_in, W_in, tiles per CTA needed).  `need` = ring slots + 1 where the ring advances once per tile (halo patch
# rings: 16 / 4 / 2 slots; 1x1 per-tap ring: 6 stages; stem tail: 4 stages of 9 taps), else 3.
CONV_CASES = [
    (2, "block1.2 halo 8-ch", 6, 240, 320, 17),
    (5, "block2.0 halo 32-ch", 6, 120, 160, 5),
    (8, "block3.1 halo 64-ch", 12, 60, 80, 3),
    (9, "block3.2 1x1 per-tap", 32, 60, 80, 7),
    (10, "block4.0 stride 2", 48, 60, 80, 3),
    (7, "block3.0 stride 2", 12, 120, 160, 3),
    (3, "block1.3 + skip1 stride 2", 6, 240, 320, 5),
    (13, "block5.0 two N tiles", 180, 30, 40, 3),
    (14, "block5.1 128-ch 3x3", 26, 39, 52, 3),
    (16, "block5.3 128-ch 1x1", 26, 39, 52, 3),        # 52,728 pixels: the last tile is ragged
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: c[1].replace(" ", "_"))
def test_conv_layer_depth(xf, oracle_state, sms, case):
    from accelerated_features_b200 import _lib, weights
    layer, name, B, H, W, need = case
    sd = oracle_state
    ks, stride, _, _ = sr.layer_geometry(layer)
    cout, cin = sd[weights.LAYERS[layer][0] + ".weight"].shape[:2]
    Ho, Wo = H // stride, W // stride
    assert_depth(name, B * Ho * Wo, sms, need)
    cinp = 8 if cin <= 8 else (32 if cin <= 32 else (64 if cin <= 64 else 128))
    cs = 8 if (cin == 8 and cout == 8) else (32 if cout == 24 else cout)      # split channels of the output tensor
    g = torch.Generator(device="cuda").manual_seed(layer * 1000 + B)
    x = torch.randn(B, H, W, cin, generator=g, device="cuda") * 2.0
    x[0, 0, 0] = 0.0                                 # exact zeros and tiny values exercise the lo-term range
    x[-1, -1, -1] *= 1e-3
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
    scale = ref.abs().max()
    got = out.permute(0, 3, 1, 2)
    assert torch.isfinite(got).all()
    err = float((got.double() - ref).abs().max() / scale)
    model = sr.error_model(lambda t: sr.emulate(sd, layer, xc, t, skip), lambda y: (y - ref).abs().max() / scale)
    report(name, err, sr.CONV_TC_TOL, model)
    # the split the next layer reads: hi = fp16_rn(y), lo = fp16_rn(y - hi) bit for bit, padded channels exact zeros; for
    # block5.0 this also places the two N tiles at channels [0,64) and [64,128) of the [hi(128) | lo(128)] row
    hi, lo = split[..., :cs], split[..., cs:]
    want_hi = out.half()
    want_lo = (out - want_hi.float()).half()
    assert torch.equal(hi[..., :cout].view(torch.int16), want_hi.view(torch.int16)), f"{name}: hi half differs"
    assert torch.equal(lo[..., :cout].view(torch.int16), want_lo.view(torch.int16)), f"{name}: lo half differs"
    if cs > cout:
        assert bool((hi[..., cout:] == 0).all() and (lo[..., cout:] == 0).all()), f"{name}: padded channels are not zero"


def _xn(x):
    return torch.nn.functional.instance_norm(x.mean(dim=1, keepdim=True), eps=orc.IN_EPS)[:, 0]


@pytest.mark.parametrize("B,H,W", [(12, 480, 640), (52, 224, 288)], ids=["12xVGA", "52x224x288"])
def test_head_chains_depth(xf, oracle_state, sms, B, H, W):
    """Fused keypoint / reliability head chains (conv impl 2) of xfeat_net, each against float64 on the GPU's own input, so the
    backbone's error does not enter; 52 x 224 x 288 gives 52,416 cells, a ragged last tile."""
    sd = oracle_state
    Hc, Wc = H // 8, W // 8
    assert_depth(f"head chains {B}x{H}x{W}", B * Hc * Wc, sms, 3)
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, 3, H, W, generator=g)
    xn = _xn(x)
    with conv_impl(xf, 2):
        feats, heat, rel, logits = xf._run_net(xn.cuda(), B, H, W, want_logits=True)
    torch.cuda.synchronize()
    u = orc.unfold8(xn.cuda()[:, None])
    ref_log = sr.reference_chain(sd, sr.KEYPOINT_HEAD, u)
    ref_heat = orc.kpts_heatmap(ref_log)[:, 0]
    err = float((logits.permute(0, 3, 1, 2).double() - ref_log).abs().max())
    report("keypoint logits", err, sr.KPT_LOGITS_TOL,
           sr.error_model(lambda t: sr.emulate_chain(sd, sr.KEYPOINT_HEAD, u, t), lambda y: (y - ref_log).abs().max()))
    err = float((heat.double() - ref_heat).abs().max())
    report("heat", err, sr.HEAT_TOL, sr.error_model(lambda t: orc.kpts_heatmap(sr.emulate_chain(sd, sr.KEYPOINT_HEAD, u, t))[:, 0],
                                                    lambda y: (y - ref_heat).abs().max()))
    f = feats.permute(0, 3, 1, 2)
    ref_rel = torch.sigmoid(sr.reference_chain(sd, sr.HEATMAP_HEAD, f))[:, 0]
    err = float((rel.double() - ref_rel).abs().max())
    report("reliability", err, sr.RELIABILITY_TOL,
           sr.error_model(lambda t: torch.sigmoid(sr.emulate_chain(sd, sr.HEATMAP_HEAD, f, t))[:, 0],
                          lambda y: (y - ref_rel).abs().max()))
    # the whole network on three images of the batch against the oracle, at the network budgets of test_gpu_conv_tc.py
    pick = [0, B // 2, B - 1]
    with torch.inference_mode():
        st = orc.backbone(sd, x[pick])
    gf = feats[pick].permute(0, 3, 1, 2).cpu().double()
    e_feats = float((gf - st["feats"]).abs().max() / st["feats"].abs().max())
    e_log = float((logits[pick].permute(0, 3, 1, 2).cpu() - st["kpt_logits"]).abs().max())
    e_rel = float((rel[pick].cpu() - st["reliability"][:, 0]).abs().max())
    e_heat = float((heat[pick].cpu() - orc.kpts_heatmap(st["kpt_logits"])[:, 0]).abs().max())
    print(f"images {pick} vs oracle: feats rel {e_feats:.2e} logits {e_log:.2e} reliability {e_rel:.2e} heat {e_heat:.2e}")
    assert e_feats < 1e-4 and e_log < 5e-4 and e_rel < 5e-5 and e_heat < 5e-5


@pytest.fixture(scope="module")
def asset_feats(oracle_state, assets_vga):
    ref, tgt = assets_vga
    with torch.inference_mode():
        st = orc.backbone(oracle_state, torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0))
    return st["feats"]


def test_fine_matcher_depth(xf, oracle_state, sms, asset_feats):
    """60,001 rows: the last layer (one N tile) runs >= 3 tiles per CTA, the 512-wide hidden layers (8 N tiles) >= 28."""
    n = 60001
    assert_depth("fine matcher, last layer", n, sms, 3)
    assert_depth("fine matcher, hidden layers", 8 * n, sms, 28)
    f0 = asset_feats[0].reshape(64, -1).t()
    f1 = asset_feats[1].reshape(64, -1).t()
    mnn = sr.coarse_pairs(asset_feats[0], asset_feats[1])
    g = torch.Generator().manual_seed(5)
    i = torch.randint(0, len(f0), (n - len(mnn),), generator=g)
    j = torch.randint(0, len(f1), (n - len(mnn),), generator=g)
    x = torch.cat([mnn, torch.cat([f0[i], f1[j]], 1)], 0)
    x[torch.randperm(n, generator=g)[:1000]] = 0.0           # all-zero rows, the last one included
    x[-1] = 0.0
    xg = x.cuda()
    got = xf.net.fine_matcher(xg)
    torch.cuda.synchronize()
    ref = sr.reference_chain(oracle_state, sr.FINE_MATCHER, xg)
    err = float((got.double() - ref).abs().max())
    model = sr.error_model(lambda t: sr.emulate_chain(oracle_state, sr.FINE_MATCHER, xg, t), lambda y: (y - ref).abs().max())
    report(f"fine matcher logits, {n} rows", err, sr.FINE_MATCHER_TOL, model)
    last = slice((n - 1) // 128 * 128, n)
    assert float((got[last].double() - ref[last]).abs().max()) < sr.FINE_MATCHER_TOL


def test_refine_depth(xf, oracle_state, sms):
    """xfeat_refine on 64 pairs x 4,096 coarse matches with ragged counts (0 and n_max included): the live rows are read on the
    device.  Sampled pairs against a float64 fine matcher + subpix_softmax2d; rows whose confidence is within 1e-4 of the
    threshold may go either way and are skipped."""
    B, n_max, conf_thr = 64, 4096, 0.25
    g = torch.Generator().manual_seed(11)
    cnt = torch.randint(0, n_max + 1, (B,), generator=g, dtype=torch.int32)
    cnt[0], cnt[1], cnt[63] = 0, n_max, n_max
    assert_depth("refine, last layer", int(cnt.sum()), sms, 3)
    d0 = torch.randn(B, n_max, 64, generator=g)
    d1 = torch.randn(B, n_max, 64, generator=g)
    k0 = torch.rand(B, n_max, 2, generator=g) * torch.tensor([640.0, 480.0])
    ar = torch.arange(n_max)
    k1 = torch.stack([(ar % 64).float() + 0.5, (ar // 64).float() + 0.25], 1).expand(B, -1, -1).contiguous()  # row id in k1
    sc0 = torch.where(torch.rand(B, n_max, generator=g) < 0.2, 1 / 0.6, 1 / 1.3).float()
    idx0 = torch.stack([torch.randperm(n_max, generator=g) for _ in range(B)])
    idx1 = torch.stack([torch.randperm(n_max, generator=g) for _ in range(B)])
    dd0 = {"descriptors": d0.cuda(), "keypoints": k0.cuda(), "scales": sc0.cuda()}
    dd1 = {"descriptors": d1.cuda(), "keypoints": k1.cuda(), "scales": torch.ones(B, n_max, device="cuda")}
    matches, n_ref = xf._refine_device(dd0, dd1, idx0.cuda(), idx1.cuda(), cnt.cuda(), conf_thr)
    torch.cuda.synchronize()
    matches, n_ref = matches.cpu(), n_ref.cpu()
    tol = sr.SUBPIX_TOL * float(sc0.max()) + 1e-4            # + fp32 rounding of x0 + dx * s at x0 < 1024
    for b in (0, 1, 2, 31, 63):
        m = int(cnt[b])
        x = torch.cat([d0[b, idx0[b, :m]], d1[b, idx1[b, :m]]], 1).cuda()
        logits = sr.reference_chain(oracle_state, sr.FINE_MATCHER, x).cpu()
        conf = torch.softmax(3 * logits, -1).max(-1)[0]
        xy = k0[b, idx0[b, :m]].double() + orc.subpix_softmax2d(logits.view(-1, 8, 8)) * sc0[b, idx0[b, :m], None].double()
        good, unsure = conf > conf_thr, (conf - conf_thr).abs() < 1e-4
        got = matches[b, :int(n_ref[b])]
        row_of = torch.full((n_max,), -1, dtype=torch.long)
        row_of[idx1[b, :m]] = torch.arange(m)                  # idx1 is a permutation: k1 identifies the coarse match
        rows = row_of[(got[:, 3] - 0.25).long() * 64 + (got[:, 2] - 0.5).long()]
        assert bool((rows >= 0).all()), f"pair {b}: a refined row that is not one of the live coarse matches"
        assert bool((rows[1:] > rows[:-1]).all()), f"pair {b}: refined rows out of order"
        assert not bool((~good[rows] & ~unsure[rows]).any()), f"pair {b}: a row below the confidence threshold was kept"
        missing = good & ~unsure
        missing[rows] = False
        assert not bool(missing.any()), f"pair {b}: {int(missing.sum())} confident rows were dropped"
        err = float((got[:, :2].double() - xy[rows]).abs().max()) if len(rows) else 0.0
        print(f"refine pair {b}: {m} coarse, {len(rows)} refined, {int(unsure.sum())} at the threshold, coord error {err:.2e} px "
              f"(bound {tol:.1e})")
        assert err < tol
        assert torch.equal(got[:, 2:], k1[b, idx1[b, :m]][rows])


def test_production_batch_end_to_end(xf, oracle_state, sms):
    """The 64-pair seed-0 randn VGA workload with two different image sets; pairs 0, 31 and 63 against the oracle run on
    just those images."""
    g = torch.Generator().manual_seed(0)
    x1 = torch.randn(64, 3, 480, 640, generator=g)
    x2 = torch.randn(64, 3, 480, 640, generator=g)
    assert_depth("64 VGA pairs, head chains", 128 * 60 * 80, sms, 3)
    got1 = xf.detectAndCompute(x1, top_k=4096)
    got2 = xf.detectAndCompute(x2, top_k=4096)
    out = xf.match_xfeat_batch(x1, x2, top_k=4096)
    pick = [0, 31, 63]
    with torch.inference_mode():
        w1, st1 = orc.detect_and_compute(oracle_state, x1[pick], 4096, return_stages=True)
        w2, st2 = orc.detect_and_compute(oracle_state, x2[pick], 4096, return_stages=True)
    for k, b in enumerate(pick):
        nd = []
        for got, want, st, tag in ((got1, w1, st1, "set1"), (got2, w2, st2, "set2")):
            gk, wk = got[b]["keypoints"].cpu().numpy(), want[k]["keypoints"].numpy()
            nd.append(assert_keypoints_exact_modulo_ties(f"pair{b}_{tag}", gk, wk, st, k, 4096))
            gi = {(float(p), float(q)): i for i, (p, q) in enumerate(gk)}
            wi = {(float(p), float(q)): i for i, (p, q) in enumerate(wk)}
            common = sorted(set(gi) & set(wi))
            ia = np.array([gi[c] for c in common]); ib = np.array([wi[c] for c in common])
            derr = float(np.abs(got[b]["descriptors"].cpu().numpy()[ia] - want[k]["descriptors"].numpy()[ib]).max())
            assert derr < 1e-3, (b, tag, derr)
        i0, i1 = orc.mnn_match(w1[k]["descriptors"], w2[k]["descriptors"], -1)
        want = match_set(w1[k]["keypoints"][i0].numpy(), w2[k]["keypoints"][i1].numpy())
        dm = assert_matches_exact_modulo_ties(f"pair{b}", match_set(*out[b]), want, w1[k]["keypoints"].numpy(), w1[k]["descriptors"],
                                              w2[k]["keypoints"].numpy(), w2[k]["descriptors"], nd[0], nd[1])
        print(f"pair {b}: {len(want)} matches, keypoint differences {nd}, match differences {dm} (all at near-ties)")


@pytest.mark.parametrize("impl", [4, 1, 3])
def test_mnn_depth(xf, sms, impl):
    """64 x 4,096 distinct unit descriptors per side through the matcher implementations; pairs 0, 31, 63 against the oracle's
    MNN, differences allowed only on rows / columns whose top-1 / top-2 gap is below 1e-5."""
    B, n = 64, 4096
    assert_depth(f"mnn impl {impl}", B * n, sms, 3)
    g = torch.Generator().manual_seed(17)
    f1 = torch.nn.functional.normalize(torch.randn(B, n, 64, generator=g), dim=-1)
    f2 = torch.nn.functional.normalize(torch.randn(B, n, 64, generator=g), dim=-1)
    old = xf._lib.xfeat_get_mnn_impl()
    xf._lib.xfeat_set_mnn_impl(impl)
    try:
        got = xf.batch_match(f1, f2)
    finally:
        xf._lib.xfeat_set_mnn_impl(old)
    for b in (0, 31, 63):
        w0, w1 = orc.mnn_match(f1[b], f2[b], -1)
        gs = {(int(i), int(j)) for i, j in zip(got[b][0].cpu(), got[b][1].cpu())}
        ws = {(int(i), int(j)) for i, j in zip(w0, w1)}
        rgap, cgap = orc.mnn_ambiguity(f1[b], f2[b])
        diff = gs ^ ws
        for i, j in diff:
            assert float(rgap[i]) < 1e-5 or float(cgap[j]) < 1e-5, f"impl {impl} pair {b}: robust match {(i, j)} differs"
        print(f"mnn impl {impl} pair {b}: {len(ws)} matches, {len(diff)} differences at near-ties")
