"""Image ingest (csrc/prep.cu) and block1.0 + block1.1 (csrc/stem.cu) against exact host references.

Ingest: xfeat_preprocess / xfeat_preprocess_scaled pick one of several kernel forms from the dtype, the strides, the pointer
alignment, the image size and two environment switches.  Every form is reached here by an input built from its dispatch
conditions; the launch count of the call tells the one-kernel cluster form from the two-kernel forms.  The gray image is
emulated bit for bit in float32 (tests/ingest_ref.py), the returned fp64 sums are checked against it, and xn must equal the
emulated InstanceNorm of those sums bit for bit.  The 8-CTA cluster and the two-kernel fallback run in a child process under
XFEAT_PREP_CLUSTER_MAX=8 and XFEAT_PREP_TWO_PASS=1.

An axis whose size does not change is copied whatever scale the caller passes, as in ATen; every form must agree on that.

Stem: stem01_kernel (what xfeat_net runs) against the stem_conv_kernel pair, bit for bit, and both against float64
BasicLayers from the oracle state."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import ingest_ref as ir

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SWITCHES = ("XFEAT_PREP_CLUSTER_MAX", "XFEAT_PREP_TWO_PASS")
LAUNCHES = {"cluster16": 1, "identity_f32": 2, "u8hwc": 2, "f32x4": 2, "generic_f32": 2, "generic_u8": 2}


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


def load_assets():
    with np.load(os.path.join(ROOT, "tests", "golden", "inputs_assets_vga.npz")) as z:
        return z["ref"], z["tgt"]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype.itemsize == 4 else np.uint16)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
class Case:
    def __init__(self, cid, dtype, C, B, Hi, Wi, layout, kind, H, W, form, scale=None, div255=False):
        self.id, self.dtype, self.C, self.B, self.Hi, self.Wi = cid, dtype, C, B, Hi, Wi
        self.layout, self.kind, self.H, self.W, self.form, self.scale, self.div255 = layout, kind, H, W, form, scale, div255

    def __repr__(self):
        return self.id


def host_pixels(c: Case) -> np.ndarray:
    """(B, Hi, Wi, C) numpy uint8 or float32 image batch."""
    rng = np.random.default_rng(sum(map(ord, c.id)))
    shape = (c.B, c.Hi, c.Wi, c.C)
    if c.kind == "assets":
        ref, tgt = load_assets()
        imgs = np.stack([(ref, tgt)[b % 2] for b in range(c.B)])[:, :c.Hi, :c.Wi, :c.C]
        return imgs if c.dtype == "u8" else imgs.astype(np.float32) / np.float32(255)
    if c.kind == "randn":
        return rng.standard_normal(shape, dtype=np.float32)
    if c.kind == "u8":           # uint8 values, also as float32 values 0..255 for div255 on fp32 input
        v = rng.integers(0, 256, shape, dtype=np.uint8)
        return v if c.dtype == "u8" else v.astype(np.float32)
    if c.kind == "constant":
        return np.full(shape, 77 if c.dtype == "u8" else 0.37, np.uint8 if c.dtype == "u8" else np.float32)
    if c.kind == "lowcontrast":  # 200 + 0.01 randn, no /255: sum_sq / n - mean^2 cancels to 1e-4 of 4e4
        return (200 + 0.01 * rng.standard_normal(shape)).astype(np.float32)
    raise ValueError(c.kind)


def device_input(c: Case) -> torch.Tensor:
    """(B, C, Hi, Wi) view on the device in the case's layout: nchw, hwc / channels_last, or nchw one float past a 16-byte
    boundary."""
    px = host_pixels(c)
    if c.layout == "hwc":
        return torch.from_numpy(px).cuda().permute(0, 3, 1, 2)
    nchw = torch.from_numpy(px).permute(0, 3, 1, 2)
    if c.layout == "nchw":     # row-major strides, also for C = 1 (channel stride H*W)
        return torch.empty(nchw.shape, dtype=nchw.dtype, device="cuda").copy_(nchw)
    if c.layout == "misaligned":
        buf = torch.empty(nchw.numel() + 4, dtype=nchw.dtype, device="cuda")
        x = buf[1:1 + nchw.numel()].view(nchw.shape)
        x.copy_(nchw)
        return x
    raise ValueError(c.layout)


def expected_form(x: torch.Tensor, H: int, W: int) -> str:
    """The form xfeat_preprocess_scaled dispatches to (prep.cu), from the same conditions."""
    B, C, Hi, Wi = x.shape
    sb, sc, sh, sw = x.stride()
    same = (Hi, Wi) == (H, W)
    if (x.dtype == torch.float32 and same and sw == 1 and x.data_ptr() % 16 == 0 and sb % 4 == 0 and sc % 4 == 0
            and sh % 4 == 0):
        return "cluster16" if H * W * 4 // 16 <= 100 * 1024 else "identity_f32"
    if (x.dtype == torch.uint8 and same and C == 3 and sc == 1 and sw == 3 and x.data_ptr() % 4 == 0 and sb % 4 == 0
            and sh % 4 == 0):
        return "u8hwc"
    if x.dtype == torch.float32 and sw == 1:
        return "f32x4"
    return "generic_f32" if x.dtype == torch.float32 else "generic_u8"


def run_prep(xf, x: torch.Tensor, H: int, W: int, div255: bool, scale=None):
    """One xfeat_preprocess (scale None) or xfeat_preprocess_scaled (scale or (scale_h, scale_w)) call on x addressed in place
    by its strides -> (xn, stats, kernels launched), outputs prefilled with NaN."""
    from accelerated_features_b200 import _lib
    B, C, Hi, Wi = x.shape
    sb, sc, sh, sw = x.stride()
    code = 1 if x.dtype == torch.uint8 else 0
    xn = torch.full((B, H, W), float("nan"), device="cuda")
    stats = torch.full((B, 2), float("nan"), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    n0 = xf._lib.xfeat_launch_count()
    if scale is None:
        rc = xf._lib.xfeat_preprocess(x.data_ptr(), code, B, C, Hi, Wi, sb, sc, sh, sw, int(div255), H, W, xn.data_ptr(),
                                      stats.data_ptr(), _stream())
    else:
        s_h, s_w = scale if isinstance(scale, tuple) else (scale, scale)
        rc = xf._lib.xfeat_preprocess_scaled(x.data_ptr(), code, B, C, Hi, Wi, sb, sc, sh, sw, int(div255), H, W, float(s_h),
                                             float(s_w), xn.data_ptr(), stats.data_ptr(), _stream())
    _lib.check(rc, "preprocess")
    n = xf._lib.xfeat_launch_count() - n0
    torch.cuda.synchronize()
    return xn.cpu().numpy(), stats.cpu().numpy(), n


def emulated_gray(c: Case, x: torch.Tensor, scale=None) -> np.ndarray:
    s_h, s_w = (None, None) if scale is None else (scale if isinstance(scale, tuple) else (scale, scale))
    return ir.gray(x.cpu().numpy(), c.H, c.W, s_h, s_w, c.div255)


def check_against_emulation(label: str, g: np.ndarray, xn: np.ndarray, stats: np.ndarray):
    """The fp64 sums within 1e-12 of the float64 sums of the emulated gray, and xn bit for bit the emulated InstanceNorm of
    the returned sums (so the fp64 summation order stays out of the comparison)."""
    want = ir.stats_f64(g)
    g64 = np.asarray(g, np.float64).reshape(g.shape[0], -1)
    assert (np.abs(stats[:, 0] - want[:, 0]) <= 1e-12 * np.abs(g64).sum(1)).all(), (label, stats, want)
    assert (np.abs(stats[:, 1] - want[:, 1]) <= 1e-12 * want[:, 1]).all(), (label, stats, want)
    xw = ir.instnorm_f32(g, stats)
    diff = bits(xn) != bits(xw)
    assert not diff.any(), f"{label}: {int(diff.sum())} of {diff.size} xn values differ from the emulation"


F06, F13 = float(ir.factor_scale(0.6)), float(ir.factor_scale(1.3))
CASES = [
    # fp32 at network resolution
    Case("f32_vga_b1_assets", "f32", 3, 1, 480, 640, "nchw", "assets", 480, 640, "cluster16"),
    Case("f32_vga_b3_randn", "f32", 3, 3, 480, 640, "nchw", "randn", 480, 640, "cluster16"),
    Case("f32_vga_b64_randn", "f32", 3, 64, 480, 640, "nchw", "randn", 480, 640, "cluster16"),      # cluster grid.y = 64
    Case("f32_vga_b2_constant", "f32", 3, 2, 480, 640, "nchw", "constant", 480, 640, "cluster16"),
    Case("f32_vga_b3_lowcontrast", "f32", 3, 3, 480, 640, "nchw", "lowcontrast", 480, 640, "cluster16"),
    Case("f32_32x32_b2_randn", "f32", 3, 2, 32, 32, "nchw", "randn", 32, 32, "cluster16"),          # W/4 = 8: partial block
    Case("f32_vga_c1_b2_randn", "f32", 1, 2, 480, 640, "nchw", "randn", 480, 640, "cluster16"),
    Case("f32_vga_c4_b2_randn", "f32", 4, 2, 480, 640, "nchw", "randn", 480, 640, "cluster16"),
    Case("f32_vga_c5_b2_randn", "f32", 5, 2, 480, 640, "nchw", "randn", 480, 640, "cluster16"),      # partial 4-channel group
    Case("f32_vga_b2_div255", "f32", 3, 2, 480, 640, "nchw", "u8", 480, 640, "cluster16", div255=True),
    Case("f32_1248x1664_b2_randn", "f32", 3, 2, 1248, 1664, "nchw", "randn", 1248, 1664, "identity_f32"),
    Case("f32_704x640_b2_randn", "f32", 3, 2, 704, 640, "nchw", "randn", 704, 640, "identity_f32"),
    Case("f32_704x640_b2_lowcontrast", "f32", 3, 2, 704, 640, "nchw", "lowcontrast", 704, 640, "identity_f32"),
    Case("f32_vga_b2_misaligned_randn", "f32", 3, 2, 480, 640, "misaligned", "randn", 480, 640, "f32x4"),
    Case("f32_vga_b2_channels_last_assets", "f32", 3, 2, 480, 640, "hwc", "assets", 480, 640, "generic_f32"),
    Case("f32_vga_c5_b2_channels_last_randn", "f32", 5, 2, 480, 640, "hwc", "randn", 480, 640, "generic_f32"),
    # uint8
    Case("u8_vga_b2_hwc_assets", "u8", 3, 2, 480, 640, "hwc", "assets", 480, 640, "u8hwc", div255=True),
    Case("u8_vga_b2_hwc_constant", "u8", 3, 2, 480, 640, "hwc", "constant", 480, 640, "u8hwc", div255=True),
    Case("u8_vga_b2_nchw_assets", "u8", 3, 2, 480, 640, "nchw", "assets", 480, 640, "generic_u8", div255=True),
    Case("u8_vga_b2_rgba_random", "u8", 4, 2, 480, 640, "hwc", "u8", 480, 640, "generic_u8", div255=True),
    # resizes
    Case("f32_300x400_to_288x384_b2_assets", "f32", 3, 2, 300, 400, "nchw", "assets", 288, 384, "f32x4"),
    Case("f32_480x650_to_480x640_b2_randn", "f32", 3, 2, 480, 650, "nchw", "randn", 480, 640, "f32x4"),
    Case("u8_300x400_to_288x384_b2_hwc_assets", "u8", 3, 2, 300, 400, "hwc", "assets", 288, 384, "generic_u8", div255=True),
    Case("f32_960x1280_s0.6_b2_randn", "f32", 3, 2, 960, 1280, "nchw", "randn", 576, 768, "f32x4", scale=F06),
    Case("f32_960x1280_s1.3_b2_randn", "f32", 3, 2, 960, 1280, "nchw", "randn", 1248, 1664, "f32x4", scale=F13),
    Case("u8_960x1280_s0.6_b2_hwc", "u8", 3, 2, 960, 1280, "hwc", "u8", 576, 768, "generic_u8", scale=F06, div255=True),
    Case("u8_960x1280_s1.3_b2_hwc", "u8", 3, 2, 960, 1280, "hwc", "u8", 1248, 1664, "generic_u8", scale=F13, div255=True),
]
BY_ID = {c.id: c for c in CASES}


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_preprocess_form_matches_emulation(xf, c):
    x = device_input(c)
    assert expected_form(x, c.H, c.W) == c.form
    xn, stats, n = run_prep(xf, x, c.H, c.W, c.div255, c.scale)
    assert n == LAUNCHES[c.form], f"{c.id}: {n} kernels launched, the {c.form} form launches {LAUNCHES[c.form]}"
    g = emulated_gray(c, x, c.scale)
    check_against_emulation(c.id, g, xn, stats)
    if c.kind == "constant":
        assert (bits(xn) == 0).all(), "a constant image normalises to +0 everywhere"
    if c.kind == "lowcontrast":
        ref = ir.instnorm_f64(g)
        err = np.abs(xn.astype(np.float64) - ref)
        bound = ir.instnorm_f32_bound(g, stats)
        print(f"{c.id}: |xn - float64 InstanceNorm| max {err.max():.3g} (bound {bound.max():.3g}); std "
              f"{np.sqrt(ir.instnorm_f64(g).var()):.3g}")
        assert (err <= bound).all()


# ---------------------------------------------------------------------------------------------------------------------
# an axis that keeps its size is copied whatever its scale (this failed for the resize forms before the fix)
S1001 = float(ir.factor_scale(1.001))
SAME_SIZE = ["f32_vga_b3_randn", "f32_704x640_b2_randn", "f32_vga_b2_misaligned_randn", "f32_vga_b2_channels_last_assets",
             "u8_vga_b2_hwc_assets", "u8_vga_b2_nchw_assets", "u8_vga_b2_rgba_random"]


@pytest.mark.parametrize("cid", SAME_SIZE)
def test_same_size_scaled_is_the_identity(xf, cid):
    c = BY_ID[cid]
    x = device_input(c)
    ident, _, _ = run_prep(xf, x, c.H, c.W, c.div255)
    got, stats, n = run_prep(xf, x, c.H, c.W, c.div255, scale=S1001)
    assert n == LAUNCHES[c.form]
    check_against_emulation(cid, emulated_gray(c, x, S1001), got, stats)
    diff = bits(got) != bits(ident)
    assert not diff.any(), f"{cid}: scale {S1001} on a same-size image changed {int(diff.sum())} of {diff.size} values"


def test_one_axis_keeps_its_size(xf):
    """480 x 650 -> 480 x 640 with a non-unit H scale: H is copied, W is resampled with its own scale."""
    c = BY_ID["f32_480x650_to_480x640_b2_randn"]
    x = device_input(c)
    scale = (S1001, float(ir.size_scale(650, 640)))
    got, stats, _ = run_prep(xf, x, 480, 640, False, scale=scale)
    check_against_emulation(c.id, emulated_gray(c, x, scale), got, stats)
    want, _, _ = run_prep(xf, x, 480, 640, False)
    assert np.array_equal(bits(got), bits(want))


# ---------------------------------------------------------------------------------------------------------------------
# the forms only an environment switch reaches: 8-CTA cluster, two-kernel fallback
FORCED = [c for c in CASES if c.form == "cluster16" and c.B <= 3]


def child_main(outdir):
    from accelerated_features_b200 import XFeat
    xf = XFeat()
    for c in FORCED:
        xn, stats, n = run_prep(xf, device_input(c), c.H, c.W, c.div255, c.scale)
        np.savez(os.path.join(outdir, c.id + ".npz"), xn=xn, stats=stats, n=n)


@pytest.mark.parametrize("env,launches", [({"XFEAT_PREP_CLUSTER_MAX": "8"}, 1), ({"XFEAT_PREP_TWO_PASS": "1"}, 2)],
                         ids=["cluster8", "two_pass"])
def test_forced_forms_give_the_same_bits(xf, tmp_path, env, launches):
    for s in SWITCHES:
        assert s not in os.environ          # this process runs the default forms
    r = subprocess.run([sys.executable, "-c", f"from tests.test_gpu_ingest import child_main; child_main({str(tmp_path)!r})"],
                       cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    for c in FORCED:
        x = device_input(c)
        mine, _, _ = run_prep(xf, x, c.H, c.W, c.div255, c.scale)
        with np.load(tmp_path / (c.id + ".npz")) as z:
            xn, stats, n = z["xn"], z["stats"], int(z["n"])
        assert n == launches, (c.id, n)
        check_against_emulation(c.id, emulated_gray(c, x, c.scale), xn, stats)
        # the low-contrast variance cancels to where the fp64 summation order shows in invstd: compared via its own sums above
        if c.kind != "lowcontrast":
            assert np.array_equal(bits(xn), bits(mine)), c.id


# ---------------------------------------------------------------------------------------------------------------------
# the dual-scale fold and xfeat_resize_bilinear
def run_resize(xf, x: torch.Tensor, Ho: int, Wo: int, div255: bool, scale: float) -> np.ndarray:
    from accelerated_features_b200 import _lib
    B, C, Hi, Wi = x.shape
    out = torch.full((B, C, Ho, Wo), float("nan"), device="cuda")
    _lib.check(xf._lib.xfeat_resize_bilinear(x.data_ptr(), 1 if x.dtype == torch.uint8 else 0, B, C, Hi, Wi, *x.stride(),
                                             int(div255), out.data_ptr(), Ho, Wo, scale, scale, _stream()), "resize")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("s", [0.6, 1.3])
@pytest.mark.parametrize("dtype", ["f32", "u8"])
def test_fold_equals_resize_then_preprocess(xf, dtype, s):
    Ho, Wo = int(math.floor(960 * s)), int(math.floor(1280 * s))
    c = Case("fold", dtype, 3, 2, 960, 1280, "nchw" if dtype == "f32" else "hwc", "randn" if dtype == "f32" else "u8", Ho, Wo,
             "", div255=dtype == "u8")
    x = device_input(c)
    sc = float(ir.factor_scale(s))
    fold, _, _ = run_prep(xf, x, Ho, Wo, c.div255, scale=sc)
    r = run_resize(xf, x, Ho, Wo, c.div255, sc)
    two_step, _, _ = run_prep(xf, r, Ho, Wo, False)
    assert np.array_equal(bits(fold), bits(two_step))


@pytest.mark.parametrize("Ho,Wo,s", [(624, 832, 1.3), (480, 640, 1.001), (480, 641, 1.0018)])
@pytest.mark.parametrize("dtype,layout", [("f32", "nchw"), ("f32", "hwc"), ("u8", "hwc"), ("u8", "nchw")])
def test_resize_matches_emulation(xf, dtype, layout, Ho, Wo, s):
    """B * C = 9 planes; 624 x 832 is extract_dualscale's s = 1.3 on VGA, not a multiple of 32."""
    c = Case("resize", dtype, 3, 3, 480, 640, layout, "randn" if dtype == "f32" else "u8", Ho, Wo, "", div255=dtype == "u8")
    x = device_input(c)
    sc = float(ir.factor_scale(s))
    got = run_resize(xf, x, Ho, Wo, c.div255, sc).cpu().numpy()
    want = ir.resize(x.cpu().numpy(), Ho, Wo, sc, sc, c.div255)
    diff = bits(got) != bits(want)
    assert not diff.any(), f"{int(diff.sum())} of {diff.size} values differ from the emulation"
    if (Ho, Wo) == (480, 640):
        assert np.array_equal(bits(got), bits(ir.values(x.cpu().numpy(), c.div255))), "a same-size resize is a copy"


# ---------------------------------------------------------------------------------------------------------------------
# public entry points: one image batch as numpy uint8, as parse_input's float tensor, and channels_last
def test_input_layouts_give_identical_bits(xf):
    ref, tgt = load_assets()
    u8 = np.stack([ref, tgt])
    f = xf.parse_input(u8)                                    # /255 on the CPU
    f_nchw, f_cl = f.contiguous(), f.contiguous(memory_format=torch.channels_last)
    assert f_cl.stride()[1] == 1 and f_nchw.stride()[3] == 1
    t_u8, flag = xf._parse_input(u8)
    assert flag and t_u8.dtype == torch.uint8
    with torch.inference_mode():
        # match_xfeat's extraction of a numpy batch: uint8 HWC, "/255" on the device
        s_u8 = xf._detect_sparse_device(t_u8, 4096, xf.detection_threshold, div255=True)
        n = s_u8["n_valid"].tolist()
        sparse_u8 = [{k: s_u8[k][b, :n[b]] for k in ("keypoints", "scores", "descriptors")} for b in range(2)]
        # match_xfeat_star's extraction of a numpy batch
        dense_u8 = xf._dense_device(t_u8, 4096, True, div255=True)
    for t in (f_nchw, f_cl):
        got = xf.detectAndCompute(t, top_k=4096)
        for b in range(2):
            for k in ("keypoints", "scores", "descriptors"):
                assert torch.equal(got[b][k].view(torch.int32), sparse_u8[b][k].view(torch.int32)), (b, k)
        got = xf.detectAndComputeDense(t, top_k=4096)
        for k in ("keypoints", "descriptors", "scales"):
            assert torch.equal(got[k].view(torch.int32), dense_u8[k].view(torch.int32)), k
    m_u8 = xf.match_xfeat_star(ref, tgt)
    m_f = xf.match_xfeat_star(xf.parse_input(ref).contiguous(), xf.parse_input(tgt).contiguous())
    assert len(m_u8[0]) > 100
    for a, b in zip(m_u8, m_f):
        assert np.array_equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# block1.0 + block1.1
def stem01(xf, variant: int, xn: torch.Tensor) -> torch.Tensor:
    from accelerated_features_b200 import _lib
    B, H, W = xn.shape
    scratch = torch.empty(B * H * W * 16, dtype=torch.uint8, device="cuda")
    out = torch.full((B, H // 2, W // 2, 16), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(xf._lib.xfeat_debug_stem01(xf._ctx, variant, xn.data_ptr(), B, H, W, out.data_ptr(), scratch.data_ptr(),
                                          scratch.numel(), _stream()), f"stem01 variant {variant}")
    torch.cuda.synchronize()
    return out


def stem_inputs(kind: str, B: int, H: int, W: int, xf) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(B * 7919 + H * 31 + W)
    if kind == "assets":
        ref, tgt = load_assets()
        return xf._preprocess(torch.from_numpy(np.stack([ref, tgt])).permute(0, 3, 1, 2).cuda(), H, W, div255=True)
    if kind == "randn":
        return torch.randn(B, H, W, generator=g, device="cuda")
    xn = torch.zeros(B, H, W, device="cuda")
    if kind == "impulse":       # one pixel at each corner and edge midpoint, and the centre: every border tap of the window
        for b in range(B):
            for i, (y, x) in enumerate([(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (0, W // 2), (H - 1, W // 2),
                                        (H // 2, 0), (H // 2, W - 1), (H // 2, W // 2)]):
                xn[b, y, x] = (3.0 + i) * (-1) ** (b + i)
    return xn


STEM_CASES = [("assets", 2, 480, 640), ("randn", 64, 480, 640), ("randn", 1, 32, 32), ("randn", 3, 64, 96),
              ("randn", 2, 1248, 1664), ("impulse", 2, 64, 96), ("impulse", 1, 32, 32), ("zeros", 2, 64, 96)]


@pytest.mark.parametrize("kind,B,H,W", STEM_CASES)
def test_stem01_matches_pair_and_float64(xf, oracle_state, kind, B, H, W):
    from oracle import xfeat_oracle as orc
    xn = stem_inputs(kind, B, H, W, xf)
    ref_pair = stem01(xf, 0, xn)
    fused = stem01(xf, 1, xn)
    a, b = ref_pair.view(torch.int16), fused.view(torch.int16)
    assert torch.equal(a, b), f"{int((a != b).any(-1).sum())} of {a[..., 0].numel()} pixels differ"
    sd = {k: v.double().cuda() for k, v in oracle_state.items() if k.startswith(("block1.0.", "block1.1."))}
    with torch.no_grad():
        t = orc._basic_layer(sd, "block1.0", xn.double()[:, None], 1)
        want = orc._basic_layer(sd, "block1.1", t, 2).permute(0, 2, 3, 1)
    got = fused[..., :8].double() + fused[..., 8:].double()
    scale = want.abs().max().item()
    err = (got - want).abs().max().item()
    print(f"stem01 {kind} {B}x{H}x{W}: max |hi + lo - float64| = {err:.3g} = {err / scale:.3g} of max|ref| {scale:.3g}")
    assert scale > 0 and err <= 1e-6 * scale
