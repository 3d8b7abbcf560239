"""The stand-alone helper kernels (csrc/helpers.cu) against the float64 / exact references of helpers_ref.py at their edges:
get_kpts_heatmap at odd shapes, temperatures and extreme logits; NMS exactly against the numpy MaxPool rule (kernel sizes up to
larger than the image, plateaus, a threshold equal to a pixel, +-inf and NaN pixels, W > 1024, W = 1, H = 1, 1248 x 1664 = 2028
chunks so the chunk scan loops, empty images, pos_cap below a count); subpix_softmax2d from n = 0 to 2^20 + 3; InterpolateSparse2d
at fractional and out-of-frame positions in all three modes; the fine matcher at ragged row counts and input magnitudes.

Bounds are the derived per-element bounds of helpers_ref.py; each test prints its worst error / bound ratio."""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from accelerated_features_b200 import _lib  # noqa: E402
from tests import helpers_ref as hr  # noqa: E402
from tests import split_ref as sr  # noqa: E402


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat(device=0)


@contextlib.contextmanager
def conv_impl(xf, impl):
    old = xf._lib.xfeat_get_conv_impl()
    xf._lib.xfeat_set_conv_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_conv_impl(old)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------------
# get_kpts_heatmap
# ---------------------------------------------------------------------------------------------------------------------------
def heat_logits(kind, B, Hc, Wc, g):
    x = torch.randn(B, 65, Hc, Wc, generator=g) * 3
    if kind == "pm60":
        x = torch.where(torch.rand(B, 65, Hc, Wc, generator=g) < 0.5, -60.0, 60.0) + torch.randn(B, 65, Hc, Wc, generator=g)
    elif kind == "dominant":
        x[:, 17] += 40
    elif kind == "dustbin":
        x[:, 64] += 40
    elif kind == "equal":
        x[:] = 1.25
    elif kind == "neginf":
        x[:, ::3] = -float("inf")
        x[:, :, 0, 0] = -float("inf")                     # one cell all -inf: NaN in the reference and the kernel
    return x


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 1, 257), (3, 7, 13), (2, 60, 80), (128, 60, 80)],
                         ids=["1x1", "1x257", "7x13", "60x80", "B128_vga"])
@pytest.mark.parametrize("temp", [1.0, 2.0, 0.5, 0.0, -1.0])
def test_kpts_heatmap(xf, shape, temp):
    B, Hc, Wc = shape
    g = torch.Generator().manual_seed(B * 1000 + Hc + Wc)
    kinds = ["randn"] if B == 128 else ["randn", "pm60", "dominant", "dustbin", "equal", "neginf"]
    worst = 0.0
    for kind in kinds:
        x = heat_logits(kind, B, Hc, Wc, g).cuda()
        heat = torch.full((B, 1, 8 * Hc, 8 * Wc), -3.0, device="cuda")
        _lib.check(xf._lib.xfeat_kpts_heatmap(x.data_ptr(), B, Hc, Wc, temp, heat.data_ptr(), _stream()), "kpts_heatmap")
        torch.cuda.synchronize()
        ref = hr.heatmap_ref(x, temp)
        nan = torch.isnan(ref)
        assert torch.equal(torch.isnan(heat), nan), f"{kind} temp {temp}: NaN cells differ from the reference"
        bound = hr.heatmap_bound(x, temp)
        ok = ~nan
        r = float(((heat.double() - ref).abs()[ok] / bound[ok]).max()) if bool(ok.any()) else 0.0
        worst = max(worst, r)
        assert r <= 1.0, f"{kind} temp {temp}: error / bound {r:.3f}"
        if kind == "equal" or temp == 0.0:
            want = torch.tensor(1 / 65, dtype=torch.float32).item()
            assert bool((heat[ok] == want).all()), f"{kind} temp {temp}: equal logits must give fp32(1/65) exactly"
    print(f"heatmap {shape} temp {temp}: worst error / bound {worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------------------
# NMS
# ---------------------------------------------------------------------------------------------------------------------------
def nms_run(xf, heat, k, thr, want_counts, pos_cap=None):
    """xfeat_nms_count, checked against want_counts before anything is written (the writer places each chunk at the scanned
    offsets), then xfeat_nms_write into a buffer pre-filled with -5 and one spare row past B * pos_cap."""
    lib = xf._lib
    B, H, W = heat.shape
    h = heat.cuda().contiguous()
    ws = torch.empty(lib.xfeat_nms_workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    cnt = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    _lib.check(lib.xfeat_nms_count(h.data_ptr(), B, H, W, k, thr, cnt.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "nms_count")
    assert cnt.tolist() == want_counts, f"counts {cnt.tolist()}, want {want_counts}"
    cap = max(want_counts) if pos_cap is None else pos_cap
    pos = torch.full((B, 0, 2), -5, dtype=torch.int64)
    if cap:
        buf = torch.full((B * cap + 1, 2), -5, dtype=torch.int64, device="cuda")
        _lib.check(lib.xfeat_nms_write(h.data_ptr(), B, H, W, k, thr, buf.data_ptr(), cap, ws.data_ptr(), ws.numel(), _stream()),
                   "nms_write")
        torch.cuda.synchronize()
        assert buf[-1].tolist() == [-5, -5], "nms_write wrote past B * pos_cap"
        pos = buf[:-1].view(B, cap, 2).cpu()
    return cnt.cpu().tolist(), pos.numpy(), cap


def nms_check(xf, heat, k, thr, tag):
    want = hr.nms_ref(heat.numpy(), thr, k)
    cnt, pos, cap = nms_run(xf, heat, k, thr, [len(w) for w in want])
    for b, w in enumerate(want):
        assert np.array_equal(pos[b, :len(w)], w), f"{tag}: image {b} positions differ"
        assert (pos[b, len(w):cap] == -5).all(), f"{tag}: image {b} wrote past its count"
    got = xf.NMS(heat[:, None].cuda(), threshold=thr, kernel_size=k)        # the public form: zero padded to the batch maximum
    assert tuple(got.shape) == (heat.shape[0], max(cnt), 2)
    for b, w in enumerate(want):
        assert np.array_equal(got[b, :len(w)].cpu().numpy(), w) and bool((got[b, len(w):] == 0).all())
    return cnt


NMS_SHAPES = [(2, 37, 41), (1, 33, 31), (2, 3, 1500), (2, 700, 1), (2, 1, 900), (1, 1248, 1664)]


@pytest.mark.parametrize("shape", NMS_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("k", [1, 3, 5, 7, 31])
def test_nms_exact(xf, shape, k):
    B, H, W = shape
    g = torch.Generator().manual_seed(H * W + k)
    heat = torch.rand(B, H, W, generator=g) ** 4
    heat[0].view(-1)[torch.randint(0, H * W, (max(1, H * W // 50),), generator=g)] = 0.5        # plateaus of equal values
    if H > 8 and W > 8:
        heat[0, 2:7, 2:7] = 0.75
    thr = 0.05
    cnt = nms_check(xf, heat, k, thr, f"{shape} k={k}")
    # the threshold equal to a pixel value: strict >
    v = float(heat[0].view(-1)[H * W // 2])
    nms_check(xf, heat, k, v, f"{shape} k={k} thr=pixel")
    if shape == (1, 1248, 1664):
        print(f"1248 x 1664 ({(H * W + 1023) // 1024} chunks), k={k}: {cnt[0]} maxima")


def test_nms_inf_nan_and_empty(xf):
    g = torch.Generator().manual_seed(8)
    heat = torch.rand(4, 40, 50, generator=g)
    heat[0, 10, 10] = float("inf")
    heat[0, 10, 11] = float("inf")                              # two +inf neighbours: both kept (inf == max)
    heat[0, 30, 30] = -float("inf")
    heat[1, 20, 20] = float("nan")                              # NaN suppresses its window and is never kept
    heat[1, 20, 22] = 0.999
    heat[1, 0, 0] = float("nan")
    heat[2] = 0.0                                               # an empty image in the batch
    heat[3, :, 25] = float("nan")
    for k in (3, 5):
        nms_check(xf, heat, k, 0.05, f"inf/nan k={k}")
    want = hr.nms_ref(heat.numpy(), 0.05, 5)
    assert [22, 20] not in want[1].tolist()
    empty = torch.zeros(3, 17, 19)
    got = xf.NMS(empty[:, None].cuda(), threshold=0.05, kernel_size=5)
    assert tuple(got.shape) == (3, 0, 2)


def test_nms_pos_cap_below_count(xf):
    g = torch.Generator().manual_seed(9)
    heat = torch.rand(3, 64, 80, generator=g)
    want = hr.nms_ref(heat.numpy(), 0.05, 3)
    cap = min(len(w) for w in want) - 7
    cnt, pos, _ = nms_run(xf, heat, 3, 0.05, [len(w) for w in want], pos_cap=cap)
    for b, w in enumerate(want):
        assert np.array_equal(pos[b], w[:cap]), f"image {b}: the first pos_cap positions differ"


# ---------------------------------------------------------------------------------------------------------------------------
# subpix_softmax2d
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 7, 2 ** 20 + 3])
@pytest.mark.parametrize("temp", [3.0, 1.0, 0.0, -3.0, 50.0])
def test_subpix_softmax2d(xf, n, temp):
    g = torch.Generator(device="cuda").manual_seed(n + 1)
    maps = torch.randn(n, 64, generator=g, device="cuda") * 3
    for i, c in enumerate((0, 7, 56, 63)):                      # one dominant entry at each corner, both signs, |x| = 1e3
        if 2 * i + 1 < n:
            maps[2 * i] = 0.0
            maps[2 * i, c] = 1e3
            maps[2 * i + 1, c] = -1e3
    out = torch.full((max(n, 1), 2), -7.0, device="cuda")
    _lib.check(xf._lib.xfeat_subpix_softmax2d(maps.data_ptr(), n, temp, out.data_ptr(), _stream()), "subpix_softmax2d")
    torch.cuda.synchronize()
    if n == 0:
        assert bool((out == -7.0).all())
        return
    ref = hr.subpix_ref(maps, temp)
    if temp == 0.0:
        assert bool((out == -0.5).all()), "temp 0 must give (-0.5, -0.5) exactly"
    r = float(((out.double() - ref).abs().max(1)[0] / hr.subpix_bound(maps, temp)).max())
    print(f"subpix n={n} temp {temp}: worst error / bound {r:.3f}")
    assert r <= 1.0
    if n >= 8 and temp == 50.0:
        corners = out[:8:2].cpu().tolist()
        assert corners == [[-4.0, -4.0], [3.0, -4.0], [-4.0, 3.0], [3.0, 3.0]], corners


# ---------------------------------------------------------------------------------------------------------------------------
# InterpolateSparse2d
# ---------------------------------------------------------------------------------------------------------------------------
INTERP_CASES = [  # (B, C, Hm, Wm, H, W, N)
    (2, 64, 12, 16, 96, 128, 400),
    (3, 65, 9, 14, 77, 101, 300),          # H, W != 8 Hm, 8 Wm
    (1, 1, 1, 20, 8, 160, 200),            # Hm = 1
    (2, 3, 17, 1, 130, 9, 200),            # Wm = 1
    (2, 5, 10, 10, 80, 80, 0),             # N = 0
]


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["nearest", "bilinear", "bicubic"])
@pytest.mark.parametrize("case", INTERP_CASES, ids=lambda c: "B{}C{}_{}x{}_in_{}x{}_N{}".format(*c))
def test_interpolate_sparse(xf, case, mode):
    B, C, Hm, Wm, H, W, N = case
    g = torch.Generator().manual_seed(B * C + Hm * Wm + N)
    x = torch.randn(B, C, Hm, Wm, generator=g)
    pos = torch.rand(B, N, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])             # fractional, per image
    if N:
        k = N // 8
        far = torch.tensor([[-40.0, H / 2], [W + 40.0, H / 2], [W / 2, -40.0], [W / 2, H + 40.0]])       # wholly outside
        near = torch.tensor([[-3.3, 5.0], [W + 2.7, 5.0], [5.0, -2.2], [5.0, H + 1.9], [-0.6, -0.4]])  # partly outside
        pos[:, :4] = far
        pos[:, 4:9] = near
        # exact .5 ties of the source coordinate: p = (W - 1) (2 c + 1) / (2 Wm) hits c + 0.5 where that is exact in fp32
        c = torch.arange(k).float() % max(Wm, 1)
        pos[0, 9:9 + k, 0] = (W - 1) * (c + 1.0) / Wm
        pos[:, 9 + k:9 + 2 * k] = torch.randint(0, 1000, (B, k, 2), generator=g).float() % torch.tensor([W, H]).float()
    out = torch.full((B, N, C), -7.0, device="cuda")
    if N:
        xc, pc = x.cuda(), pos.cuda()
        _lib.check(xf._lib.xfeat_interpolate_sparse(xc.data_ptr(), pc.data_ptr(), B, C, Hm, Wm, N, H, W, mode, out.data_ptr(),
                                                    _stream()), "interpolate_sparse")
    else:
        _lib.check(xf._lib.xfeat_interpolate_sparse(x.cuda().data_ptr(), pos.cuda().data_ptr(), B, C, Hm, Wm, 0, H, W, mode,
                                                    out.data_ptr(), _stream()), "interpolate_sparse")
    torch.cuda.synchronize()
    if N == 0:
        return
    name = ["nearest", "bilinear", "bicubic"][mode]
    want, bound = hr.sample_ref(x.numpy(), pos.numpy(), H, W, name)
    got = out.cpu().double().numpy()
    if mode == 0:
        ties = int((hr.source_coord(pos[0, 9:9 + k, 0].numpy(), W, Wm) % 1 == 0.5).sum())
        print(f"nearest: {ties} exact .5 ties of the source x")
        assert ties > 0 or Wm != 16
        assert np.array_equal(got, want), f"nearest: {int((got != want).sum())} values differ"
        return
    r = float((np.abs(got - want) / bound).max())
    print(f"{name} {case}: worst error / bound {r:.3f}")
    assert r <= 1.0
    assert (got[:, :4] == 0).all(), f"{name}: positions wholly outside the frame must sample zeros"


# ---------------------------------------------------------------------------------------------------------------------------
# fine matcher
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fm_rows(oracle_state, assets_vga):
    from oracle import xfeat_oracle as orc
    ref, tgt = assets_vga
    with torch.inference_mode():
        f = orc.backbone(oracle_state, torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0))["feats"]
    x = sr.coarse_pairs(f[0], f[1])
    g = torch.Generator().manual_seed(12)
    a, b = f[0].reshape(64, -1).t(), f[1].reshape(64, -1).t()
    i, j = torch.randint(0, len(a), (1000,), generator=g), torch.randint(0, len(b), (1000,), generator=g)
    return torch.cat([x, torch.cat([a[i], b[j]], 1)], 0)[:1000].contiguous()


def fine_matcher_run(xf, x):
    n = x.shape[0]
    out = torch.full((max(n, 1), 64), -7.0, device="cuda")
    ws = torch.empty(xf._lib.xfeat_fine_matcher_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    _lib.check(xf._lib.xfeat_fine_matcher(xf._ctx, x.data_ptr(), n, out.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
               "fine_matcher")
    torch.cuda.synchronize()
    return out[:n]


@pytest.mark.parametrize("impl", [2, 0])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 1000])
def test_fine_matcher_rows(xf, oracle_state, fm_rows, n, impl):
    x = fm_rows[-n:].cuda().contiguous()
    with conv_impl(xf, impl):
        got = fine_matcher_run(xf, x)
    ref = sr.reference_chain(oracle_state, sr.FINE_MATCHER, x)
    err = float((got.double() - ref).abs().max())
    print(f"fine matcher n={n} impl {impl}: error {err:.2e} (bound {sr.FINE_MATCHER_TOL:.0e})")
    assert err < sr.FINE_MATCHER_TOL


# Inputs in the fine matcher's domain (include/xfeat_b200.h: max |x| <= 2^13) give finite logits within FINE_MATCHER_TOL times the
# gain: the split is relative, so the error grows with the activations.  Outside it the tensor-core schedule's fp16 split of the
# input overflows; the gains below find where.
FM_DOMAIN = 2.0 ** 13


@pytest.mark.parametrize("impl", [2, 0])
def test_fine_matcher_magnitudes(xf, oracle_state, fm_rows, impl):
    x0 = fm_rows.cuda()
    for gain in (1.0, 10.0, 100.0, 1000.0, 2.0 ** 15):
        x = (x0 * gain).contiguous()
        with conv_impl(xf, impl):
            got = fine_matcher_run(xf, x)
        ref = sr.reference_chain(oracle_state, sr.FINE_MATCHER, x)
        finite = bool(torch.isfinite(got).all())
        err = float((got.double() - ref).abs().max()) if finite else float("inf")
        inside = float(x.abs().max()) <= FM_DOMAIN
        print(f"fine matcher impl {impl} gain {gain:g} (max |x| {float(x.abs().max()):.3g}, max |logit| {float(ref.abs().max()):.3g}): "
              f"finite {finite}, error {err:.2e}, error / gain {err / gain:.2e} (bound {sr.FINE_MATCHER_TOL:.0e}), "
              f"{'inside' if inside else 'outside'} the domain")
        if inside or impl == 0:
            assert finite and err / gain < sr.FINE_MATCHER_TOL
