"""CPU checks of tests/select_ref.py, the host reference the GPU selection tests (test_gpu_select.py) compare against."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import xfeat_oracle as orc
from tests import select_ref as ref

U = 2.0 ** -24          # unit roundoff of float32


@pytest.fixture(scope="module")
def vga_maps(oracle_state, assets_vga):
    """Heat-map and reliability map of the two VGA asset images, computed by the oracle network."""
    x = torch.cat([orc.parse_input(a) for a in assets_vga], 0)
    with torch.inference_mode():
        st = orc.backbone(oracle_state, x)
        heat = orc.kpts_heatmap(st["kpt_logits"])
    return heat[:, 0].numpy(), st["reliability"][:, 0].numpy()


def random_maps(seed, B, H, W):
    g = np.random.default_rng(seed)
    heat = g.random((B, H, W), dtype=np.float32) * np.float32(0.3)
    rel = g.random((B, H // 8, W // 8), dtype=np.float32)
    return heat, rel


MAPS = [("vga", None), ("random_96x160", (1, 96, 160)), ("random_480x416", (2, 480, 416)), ("random_32x1024", (3, 32, 1024))]


def get_maps(vga_maps, which, shape):
    if shape is None:
        return vga_maps
    return random_maps(*shape[:1], 2, *shape[1:])


def all_pixels(H, W):
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return xs.reshape(-1), ys.reshape(-1)


def aten_scalar_scores(heat, rel, xs, ys):
    """xfeat.py:77-80 through ATen's scalar grid sampler (`_grid_sampler_2d_cpu_fallback`): grid_sampler_unnormalize
    ((g + 1) * size - 1) / 2, the formula of ATen's CUDA kernel and of the oracle's source_coord."""
    B, H, W = heat.shape
    pos = torch.from_numpy(np.stack([xs, ys], -1)).float()
    grid = (2.0 * (pos / torch.tensor([W - 1, H - 1], dtype=torch.float32)) - 1.0)[None, :, None].expand(B, -1, -1, -1)
    near = torch._grid_sampler_2d_cpu_fallback(torch.from_numpy(heat)[:, None], grid, 1, 0, False)[:, 0, :, 0]
    bil = torch._grid_sampler_2d_cpu_fallback(torch.from_numpy(rel)[:, None], grid, 0, 0, False)[:, 0, :, 0]
    s = (near * bil).numpy()
    s[:, (xs == 0) & (ys == 0)] = -1
    return s


def f64_bound(heat, rel, xs, ys, s32):
    """|s32 - s64| <= |kv| * Rmax * u * (9 (Wm + Hm) + 8) + u |s32|, u = 2^-24, Rmax = max |reliability| of the image.
    Derivation, following the float32 operations of sparse_src_coord for a map of size M:
      q = p / (n - 1) in [0, 1]: error <= u;  g = 2 q - 1: 2q exact, rounding <= u |g| <= u, so |dg| <= 3u;
      g + 1 in [0, 2]: + 2u -> 5u;  * M: 5uM + rounding 2uM -> 7uM;  - 1: + 2uM -> 9uM;  / 2 exact: |d ix| <= 4.5 u M.
    Bilinear interpolation with zero padding is Lipschitz in (ix, iy) with constant 2 Rmax per axis, so the coordinate error
    moves the sample by <= 9 u Rmax (Wm + Hm); the float32 evaluation adds <= u for the weight (fx + 1) - ix, u for wx * wy,
    u for R * w and 3u for the three sums of terms bounded by Rmax: <= 8 u Rmax (a loose count).  The nearest tap kv is a
    stored heat value, exact in both; the final product rounds once more: u |s32|."""
    H, W = heat.shape
    kv = np.abs(heat[ys, xs]).astype(np.float64)
    return kv * float(np.abs(rel).max()) * U * (9 * (W // 8 + H // 8) + 8) + U * np.abs(s32.astype(np.float64))


@pytest.mark.parametrize("which,shape", MAPS, ids=[m[0] for m in MAPS])
def test_score_emulation_equals_aten(vga_maps, which, shape):
    """The float32 emulation of nms_score_key equals ATen's scalar grid sampler (nearest * bilinear) bit for bit at every
    pixel of the map, (0, 0) -> -1 and the out-of-range last row / column included: 0 positions differ.

    The oracle's sparse_scores runs F.grid_sample, whose vectorised CPU kernel computes the source coordinate in a different
    operation order.  Measured here: about 23 % of the scores differ from it (71 709 of 307 200 on the first VGA map; 3 902 of
    15 360 at 96 x 160), by up to 63 ulp on VGA and 225 ulp at 480 x 416 -- more than 1 ulp, because an ulp of the coordinate
    moves the bilinear weights by many ulps of the weight.  Both stay inside the float64 bound of f64_bound (worst 0.08 of it),
    which this test checks for the oracle; the GPU tests compare the kernels with the exact emulation, not with this bound."""
    heat, rel = get_maps(vga_maps, which, shape)
    B, H, W = heat.shape
    xs, ys = all_pixels(H, W)
    want = aten_scalar_scores(heat, rel, xs, ys)
    pos = torch.from_numpy(np.stack([xs, ys], -1)).long()[None].expand(B, -1, -1).contiguous()
    oracle = orc.sparse_scores(torch.from_numpy(heat)[:, None], torch.from_numpy(rel)[:, None], pos).numpy()
    for b in range(B):
        got = ref.scores_f32(heat[b], rel[b], xs, ys)
        assert got.dtype == np.float32
        diff = got.view(np.int32) != want[b].view(np.int32)
        assert int(diff.sum()) == 0, f"b={b}: {int(diff.sum())} of {diff.size} scores differ from ATen"
        s64 = ref.scores_f64(heat[b], rel[b], xs, ys)
        assert (np.abs(oracle[b] - s64) <= f64_bound(heat[b], rel[b], xs, ys, oracle[b])).all()
        n_vec = int((got.view(np.int32) != oracle[b].view(np.int32)).sum())
        print(f"[{which} b={b}] vectorised F.grid_sample differs at {n_vec} of {diff.size} pixels")
    # the quirks are present: (0, 0) is -1 and the last row and column read the nearest tap out of range -> 0
    s = ref.scores_f32(heat[0], rel[0], xs, ys).reshape(H, W)
    assert s[0, 0] == -1.0 and not s[-1, :].any() and not s[:, -1].any()


@pytest.mark.parametrize("which,shape", MAPS, ids=[m[0] for m in MAPS])
def test_score_emulation_within_float64_bound(vga_maps, which, shape):
    """The emulation is within f64_bound (derived in its docstring) of the same formula evaluated in float64."""
    heat, rel = get_maps(vga_maps, which, shape)
    B, H, W = heat.shape
    xs, ys = all_pixels(H, W)
    worst = 0.0
    for b in range(B):
        s32 = ref.scores_f32(heat[b], rel[b], xs, ys)
        s64 = ref.scores_f64(heat[b], rel[b], xs, ys)
        bound = f64_bound(heat[b], rel[b], xs, ys, s32)
        err = np.abs(s32.astype(np.float64) - s64)
        assert (err <= bound).all(), f"b={b}: {int((err > bound).sum())} scores outside the bound"
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    print(f"[{which}] worst |s32 - s64| / bound = {worst:.3f}")


def test_nms_mask_equals_oracle(vga_maps):
    heat, _ = vga_maps
    for thr in (0.05, 0.0):
        want = torch.from_numpy(heat)[:, None]
        local = F.max_pool2d(want, 5, stride=1, padding=2)
        want = ((want == local) & (want > thr))[:, 0].numpy()
        assert np.array_equal(ref.nms_mask(heat, thr), want)
        assert np.array_equal(np.stack(np.nonzero(want[0])[::-1], -1), orc.nms_numpy(heat[0], thr))


def test_sparse_select_order_and_capacity():
    """Ties on the score resolve by raster index; more than H*W/4 positive candidates is an overflow."""
    H, W = 64, 64
    heat = np.zeros((H, W), np.float32)
    heat[10:13, 20:23] = 0.5                      # a 3x3 plateau: nine maxima with one score
    heat[40, 40] = 0.75
    rel = np.ones((H // 8, W // 8), np.float32)
    sel = ref.sparse_select(heat, rel, 0.05, 5)
    assert sel["n_cand"] == 10 and sel["n_valid"] == 5
    assert (sel["x"][0], sel["y"][0]) == (40, 40)
    lin = sel["y"][1:] * W + sel["x"][1:]
    assert np.all(np.diff(lin) > 0) and np.all(sel["score"][1:] == sel["score"][1])
    flat = np.full((H, W), 0.5, np.float32)
    assert ref.sparse_select(flat, rel, 0.05, 5)["n_valid"] == -1


def test_dense_select_signed_zero_ties():
    rel = np.array([[0.0, -0.0, 1.0, -1.0], [-0.0, 0.0, 1.0, np.float32(-1e-30)]], np.float32)
    assert ref.dense_select(rel, 8).tolist() == [2, 6, 0, 1, 4, 5, 7, 3]


def test_bicubic_reference_equals_aten_grid_sample():
    """descriptors_f64 is ATen grid_sampler_2d (bicubic, zeros, align_corners=False) in float64 at the float32 source
    coordinate, followed by F.normalize: checked against ATen itself run in float64, border keypoints included."""
    g = np.random.default_rng(5)
    H, W = 96, 160
    feats = g.standard_normal((H // 8, W // 8, 64)).astype(np.float32)
    xs = np.concatenate([g.integers(0, W, 300), [0, 1, 2, W - 3, W - 2, W - 1, 0, W - 1]])
    ys = np.concatenate([g.integers(0, H, 300), [0, 1, 2, H - 3, H - 2, H - 1, H - 1, 0]])
    got, _, _ = ref.descriptors_f64(feats, xs, ys, H, W)
    M = F.normalize(torch.from_numpy(feats).double().permute(2, 0, 1)[None], dim=1)
    gx = ref.src_coord_f32(xs, W, W // 8).astype(np.float64)
    gy = ref.src_coord_f32(ys, H, H // 8).astype(np.float64)
    grid = torch.from_numpy(np.stack([(2 * gx + 1) / (W // 8) - 1, (2 * gy + 1) / (H // 8) - 1], -1))[None, :, None]
    want = F.grid_sample(M, grid, mode="bicubic", align_corners=False)[0, :, :, 0].t()
    want = F.normalize(want, dim=-1).numpy()
    assert np.abs(got - want).max() < 1e-12


def test_split_f16_reconstructs():
    g = np.random.default_rng(7)
    d = g.standard_normal((1000, 64)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    hi, lo = ref.split_f16(d)
    x = d.astype(np.float64) * 8192
    err = np.abs(hi.astype(np.float64) + lo.astype(np.float64) - x)
    # half an fp16 ulp of lo = x - hi (2^-25 where lo is subnormal)
    assert (err <= np.maximum(np.abs(x - hi.astype(np.float64)) * 2.0 ** -11, 2.0 ** -25)).all()


def max_width_at(H):
    """The largest multiple of 32 with H * W * W < 2^40, the host condition of the sorted sampler."""
    W = int(np.sqrt((1 << 40) / H)) // 32 * 32 + 32
    while H * W * W >= (1 << 40):
        W -= 32
    return W


# (H, W): the widest image the host allows at H = 4096, the sorted sampler's tallest (Hm = 512) and widest-at-Hm-1 shapes, and
# narrow and wide shapes of the test suite
MAGIC_SHAPES = [(4096, max_width_at(4096)), (4096, 256), (32, max_width_at(32) // 32 * 32), (480, 640), (2048, 2048), (32, 32),
                (480, 416), (64, 160)]


@pytest.mark.parametrize("H,W", MAGIC_SHAPES, ids=[f"{h}x{w}" for h, w in MAGIC_SHAPES])
def test_magic_division_exact_at_host_bound(H, W):
    """y = (lin * magic(W)) >> 40 equals lin // W for every pixel lin < H * W, and the column-strip division equals x // xw
    for every x < W and every strip count 1..8, wherever the host enables the sorted sampler (H * W * W < 2^40)."""
    assert H * W * W < (1 << 40)
    chunk = 1 << 24
    for lo in range(0, H * W, chunk):
        lin = np.arange(lo, min(H * W, lo + chunk), dtype=np.uint64)
        assert np.array_equal(ref.magic_div(lin, W), lin // np.uint64(W)), (H, W, lo)
    xs = np.arange(W, dtype=np.uint64)
    for nxb in range(1, 9):
        xw = (W + nxb - 1) // nxb
        assert np.array_equal(ref.magic_div(xs, xw), xs // np.uint64(xw)), (W, nxb)


def test_magic_division_bound_is_needed():
    """Past the host bound the reciprocal division goes wrong: with magic(d) * d = 2^40 + e, the first pixel index where it
    fails is the smallest n = -1 (mod d) with n * e >= 2^40.  For W = 65 760 (e = 43 904) that index is on row 380, and any
    image with that row has H * W * W >= 2^40, which makes the host choose the generic sampler."""
    W = 65760
    e = ref.magic(W) * W - (1 << 40)
    n = -(-(1 << 40) // e)
    n += (W - 1 - n % W) % W
    assert ref.magic_div(np.array([n]), W)[0] != n // W
    assert ref.magic_div(np.array([n - W]), W)[0] == (n - W) // W
    H = n // W + 1
    assert H == 381 and H * W * W >= (1 << 40)


def test_sorted_sampler_strips():
    assert [ref.sorted_sampler_strips(h) for h in (12, 60, 64, 65, 128, 256, 257, 512)] == [8, 8, 8, 7, 4, 2, 1, 1]
