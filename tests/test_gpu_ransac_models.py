"""Homography and essential-matrix RANSAC on the GPU (xfeat_ransac_homography / xfeat_ransac_essential,
geometry.find_homography_batch / find_essential_batch) against the float64 references of tests/ransac_ref.py.

The estimators are stochastic only in which minimal sample wins; everything after the winner is deterministic.  So these tests
check, on synthetic scenes with a known answer:
  * exact recovery on noise-free data (the mask is the true inlier set, the model is the true one to float32 rounding);
  * that the returned homography is the float64 least-squares refit of its own mask (normal equations, eigen-solver and
    de-normalisation), which exact data cannot tell from the raw 4-point hypothesis;
  * that the mask is `error < thr` under the returned model, recomputed in float64 from the input points;
  * that the MSAC cost of the returned model is no worse than the true model's;
  * degenerate inputs, determinism and isolation of each pair from the rest of its batch.
Inliers are exact float64 projections rounded to float32 (plus Gaussian noise where stated).  Outliers are redrawn until their
true error is far above the threshold, so no check depends on a point near it.  Rows past a pair's count hold large garbage
values, so a kernel reading past its count is visible.

Measured on one H100 SXM (80 GB): the worst cases behind each tolerance are given beside it."""
import numpy as np
import pytest
import torch

from accelerated_features_b200 import _lib
from accelerated_features_b200.geometry import find_essential_batch, find_homography, find_homography_batch, recover_pose
from tests import ransac_ref as ref

pytestmark = pytest.mark.gpu

F32 = np.float32
SIZES = [(64, 48), (640, 480), (3840, 2160)]
MOTIONS = ["identity", "translation", "rot90", "rot180", "scale0.3", "scale3", "perspective"]


def garbage(rng, shape):
    return (rng.uniform(1e5, 1e6, shape) * rng.choice([-1, 1], shape)).astype(F32)


def grid(W, H):
    return np.stack(np.meshgrid(np.linspace(0, W, 9), np.linspace(0, H, 9)), -1).reshape(-1, 2)


def grid_dist(Ha, Hb, W, H):
    g = grid(W, H)
    return float(np.linalg.norm(ref.apply_h(Ha, g) - ref.apply_h(Hb, g), axis=1).max())


def motion_h(kind, W, H):
    """A homography image 0 -> image 1 of the named kind for a W x H image (rotations and scales about the image centre)."""
    C, Ci = np.array([[1, 0, -W / 2], [0, 1, -H / 2], [0, 0, 1.0]]), np.array([[1, 0, W / 2], [0, 1, H / 2], [0, 0, 1.0]])
    rot = lambda a: np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])  # noqa: E731
    if kind == "identity":
        return np.eye(3)
    if kind == "translation":
        return np.array([[1, 0, 0.13 * W], [0, 1, -0.07 * H], [0, 0, 1.0]])
    if kind == "rot90":
        return Ci @ rot(np.pi / 2) @ C
    if kind == "rot180":
        return Ci @ rot(np.pi) @ C
    if kind.startswith("scale"):
        s = float(kind[5:])
        return Ci @ np.diag([s, s, 1.0]) @ C
    if kind == "perspective":          # w = 1 - 0.5 x / W - 0.3 y / H: from 1 at the origin down to 0.2 at (W, H)
        return np.array([[1.1, 0.05, 0.02 * W], [0.03, 0.95, 0.01 * H], [-0.5 / W, -0.3 / H, 1.0]])
    raise ValueError(kind)


def h_scene(rng, W, H, Ht, n, frac, thr, noise=0.0):
    """n correspondences under Ht in a W x H image: round(frac n) inliers (Gaussian noise of `noise` px on image 1), the rest
    outliers redrawn until their true transfer error is >= 10 thr.  Returns p0, p1 (float32) and the true inlier mask.
    With n <= 5 the points sit near the corners (and the centre): four random points can be close to collinear, and the
    homography they fix is then ill-conditioned away from them, whatever computes it."""
    if n <= 5:
        corners = np.array([[0.1, 0.1], [0.9, 0.12], [0.88, 0.9], [0.12, 0.88], [0.5, 0.45]])[:n]
        p0 = ((corners + rng.uniform(-0.05, 0.05, (n, 2))) * [W, H]).astype(F32)
    else:
        p0 = rng.uniform([0, 0], [W, H], (n, 2)).astype(F32)
    p1 = ref.apply_h(Ht, p0) + rng.normal(0, noise, (n, 2)) if noise else ref.apply_h(Ht, p0)
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:int(round(frac * n))]] = True
    corners = ref.apply_h(Ht, np.array([[0, 0], [W, 0], [0, H], [W, H]], np.float64))
    lo, hi = corners.min(0) - 10 * thr, corners.max(0) + 10 * thr
    p1 = p1.astype(F32)
    bad = ~inl
    while bad.any():
        p1[bad] = rng.uniform(lo, hi, (bad.sum(), 2)).astype(F32)
        bad = ~inl & (ref.transfer_err(Ht, p0, p1) < 10 * thr)
    return p0, p1, inl


def pack(rng, scenes, n_max, counts=None):
    """(B, n_max, 2) arrays of the scenes' points, garbage past each count."""
    B = len(scenes)
    p0, p1 = garbage(rng, (B, n_max, 2)), garbage(rng, (B, n_max, 2))
    cnt = np.array([len(s[0]) for s in scenes] if counts is None else counts, np.int32)
    for b, s in enumerate(scenes):
        p0[b, :len(s[0])], p1[b, :len(s[1])] = s[0], s[1]
    return p0, p1, cnt


def run_h(p0, p1, cnt, thr, iters, seed):
    H, m, n = find_homography_batch(torch.from_numpy(p0).cuda(), torch.from_numpy(p1).cuda(),
                                    None if cnt is None else torch.from_numpy(cnt).cuda(), thr=thr, iters=iters, seed=seed)
    return H.cpu().numpy(), m.cpu().numpy(), n.cpu().numpy()


def run_e(x0, x1, cnt, thr, iters, seed):
    E, m, n = find_essential_batch(torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda(),
                                   None if cnt is None else torch.from_numpy(cnt).cuda(), thr=thr, iters=iters, seed=seed)
    return E.cpu().numpy(), m.cpu().numpy(), n.cpu().numpy()


def assert_mask_rule(err, mask, thr, what):
    """mask == (err < thr) outside a 1e-3 relative band around thr (the float32 rounding of the classification), with at most
    2 points inside the band."""
    clear = np.abs(err - thr) > 1e-3 * thr
    assert np.array_equal(mask[clear], (err < thr)[clear]), what
    assert (~clear).sum() <= 2, what


# ---------------------------------------------------------------------------------------------------------------------------
# homography
# ---------------------------------------------------------------------------------------------------------------------------
H_NW = [(4, 1.0), (5, 1.0)] + [(n, w) for n in (64, 1000) for w in (1.0, 0.7, 0.4)]
H_BIG = [(8192, w) for w in (1.0, 0.7, 0.4)]
H_THR = 3.0
# worst grid distance |H_gpu(x) - H_true(x)| over the 9 x 9 grid, as a fraction of the image diagonal, per image size
GRID_TOL = 1e-5        # measured: 1.1e-6 (64x48), 1.3e-6 (640x480), 2.1e-6 (3840x2160)


@pytest.mark.parametrize("iters", [1024, 700])
def test_homography_exact_recovery(iters):
    """Noise-free scenes over image sizes, motions, counts and inlier fractions: the mask is the true inlier set, H[2,2] = 1,
    and H maps a 9 x 9 grid over the image within 1e-5 of the diagonal of where the true H does."""
    rng = np.random.default_rng(100 + iters)
    worst = {}
    for group, n_max in ((H_NW, 1024), (H_BIG, 8192)):
        keys, scenes = [], []
        for W, H in SIZES:
            for kind in MOTIONS:
                Ht = motion_h(kind, W, H)
                for n, w in group:
                    keys.append((W, H, kind, n, w, Ht))
                    scenes.append(h_scene(rng, W, H, Ht, n, w, H_THR))
        p0, p1, cnt = pack(rng, scenes, n_max)
        Hg, mask, n_inl = run_h(p0, p1, cnt, H_THR, iters, seed=iters)
        for b, ((W, H, kind, n, w, Ht), (_, _, inl)) in enumerate(zip(keys, scenes)):
            what = f"{W}x{H} {kind} n={n} w={w}"
            assert np.array_equal(mask[b, :n], inl) and not mask[b, n:].any(), what
            assert n_inl[b] == inl.sum(), what
            assert Hg[b, 2, 2] == 1.0, what
            d = grid_dist(Hg[b].astype(np.float64), Ht, W, H) / np.hypot(W, H)
            worst[(W, H)] = max(worst.get((W, H), 0.0), d)
            assert d < GRID_TOL, (what, d)
    print(f"iters {iters}: worst grid distance / diagonal " + ", ".join(f"{W}x{H} {d:.2e}" for (W, H), d in worst.items()))


def noisy_h_batch(rng, sizes=((640, 480),), n_list=(300, 1000, 3000), fracs=(0.25, 0.4, 0.7), noises=(0.3, 0.6, 1.0),
                  thr=H_THR, motions=("translation", "rot90", "scale0.3", "scale3", "perspective")):
    keys, scenes = [], []
    for W, H in sizes:
        for kind in motions:
            for n in n_list:
                for w in fracs:
                    noise = noises[len(scenes) % len(noises)]
                    Ht = motion_h(kind, W, H)
                    keys.append((W, H, kind, n, w, noise, Ht))
                    scenes.append(h_scene(rng, W, H, Ht, n, w, thr, noise))
    return keys, scenes


# worst |H_gpu(x) - H_ref(x)| on the grid, in pixels per 800 px of image diagonal (2e-3 px at VGA)
REFIT_TOL = 2e-3       # measured: 9.2e-4 (640x480), 9.7e-4 (3840x2160)


def test_homography_is_refit_of_its_mask():
    """The returned H is the float64 least-squares DLT refit of its own mask, in the Hartley frames of all n points: the mask
    is a fixed point of the refit (its transfer error < thr reproduces the mask), and H agrees with the refit on the grid.

    The kernel refits twice, the second time on the mask of the first refit, and classifies with the second.  When an inlier
    sits near the threshold the two masks can differ, and H is then the refit of a mask a point or two away from the one
    returned: at 1 px noise and thr 3 px this moved H by 0.034 px on the grid for a VGA pair of 1000 correspondences.  The
    noise here stays at or below 0.6 px, where no inlier comes near 3 px."""
    rng = np.random.default_rng(7)
    keys, scenes = noisy_h_batch(rng, sizes=((640, 480), (3840, 2160)), noises=(0.3, 0.45, 0.6))
    p0, p1, cnt = pack(rng, scenes, 3072)
    Hg, mask, n_inl = run_h(p0, p1, cnt, H_THR, 4096, seed=3)
    worst = {}
    for b, (W, H, kind, n, w, noise, Ht) in enumerate(keys):
        what = f"{W}x{H} {kind} n={n} w={w} noise={noise}"
        a, c, m = p0[b, :n], p1[b, :n], mask[b, :n]
        Hr = ref.dlt_refit(a, c, m, ref.hartley(a), ref.hartley(c))
        assert_mask_rule(ref.transfer_err(Hr, a, c), m, H_THR, what)
        d = grid_dist(Hg[b].astype(np.float64), Hr, W, H) * 800 / np.hypot(W, H)
        worst[(W, H)] = max(worst.get((W, H), 0.0), d)
        assert d < REFIT_TOL, (what, d)
    print("worst grid distance H_gpu - H_ref (px per 800 px of diagonal): " +
          ", ".join(f"{W}x{H} {d:.2e}" for (W, H), d in worst.items()))


@pytest.mark.parametrize("thr", [1.0, 3.0, 8.0])
def test_homography_mask_is_transfer_error_below_thr(thr):
    """The mask is `|H(p0) - p1| < thr` under the returned H, in float64 from the pixel points; n_inliers is its size; rows
    past the count are never inliers; a count above n_max is clamped to n_max."""
    rng = np.random.default_rng(int(thr * 10))
    keys, scenes = noisy_h_batch(rng, sizes=SIZES, n_list=(200, 1500), fracs=(0.4, 0.7), thr=thr,
                                 noises=(thr / 10, thr / 6, thr / 3))
    n_max = 2048
    p0, p1, cnt = pack(rng, scenes, n_max)
    # the last pair fills all rows and claims more: clamped to n_max
    Wl, Hl = 640, 480
    Htl = motion_h("scale3", Wl, Hl)
    last = h_scene(rng, Wl, Hl, Htl, n_max, 0.5, thr, thr / 6)
    p0 = np.concatenate([p0, last[0][None]]); p1 = np.concatenate([p1, last[1][None]])
    keys.append((Wl, Hl, "scale3", n_max, 0.5, thr / 6, Htl))
    Hg, mask, n_inl = run_h(p0, p1, np.append(cnt, n_max + 100).astype(np.int32), thr, 2048, seed=1)
    for b, (W, H, kind, n, w, noise, Ht) in enumerate(keys):
        what = f"{W}x{H} {kind} n={n} w={w}"
        assert_mask_rule(ref.transfer_err(Hg[b].astype(np.float64), p0[b, :n], p1[b, :n]), mask[b, :n], thr, what)
        assert n_inl[b] == mask[b].sum() and not mask[b, n:].any(), what
    Hc, mc, nc = run_h(p0, p1, np.append(cnt, n_max).astype(np.int32), thr, 2048, seed=1)
    assert np.array_equal(Hc, Hg) and np.array_equal(mc, mask) and np.array_equal(nc, n_inl)


COST_TOL = 1.02        # homography, measured: 1.0000 at most
E_COST_TOL = 1.05      # measured: 1.022; see test_essential_msac_cost_reaches_truth


def test_homography_msac_cost_reaches_truth():
    """With enough samples for >= 10 expected all-inlier ones, the MSAC cost of the returned H (float64, pixels) is within 2 %
    of the true H's: the refit lands on the optimum the truth sits near, not on a worse local one."""
    rng = np.random.default_rng(11)
    keys, scenes = noisy_h_batch(rng, sizes=((640, 480), (3840, 2160)), n_list=(500, 2000), noises=(0.5,))
    p0, p1, cnt = pack(rng, scenes, 2048)
    Hg, _, _ = run_h(p0, p1, cnt, H_THR, 4096, seed=5)          # 0.25^4 * 4096 = 16 all-inlier samples at 25 %
    ratios = []
    for b, (W, H, kind, n, w, noise, Ht) in enumerate(keys):
        a, c = p0[b, :n], p1[b, :n]
        r = ref.msac_cost(ref.transfer_err(Hg[b].astype(np.float64), a, c), H_THR) / ref.msac_cost(ref.transfer_err(Ht, a, c), H_THR)
        ratios.append(r)
        assert r <= COST_TOL, (f"{W}x{H} {kind} n={n} w={w}", r)
    print(f"homography MSAC cost / true cost: max {max(ratios):.4f}, median {np.median(ratios):.4f}")


def h_degenerate_scenes(rng):
    """(name, p0, p1): pairs whose every 4-point sample is degenerate, with integer coordinates so the degeneracy survives the
    float32 normalisation."""
    n = 64
    ident = (np.full((n, 2), [100.0, 200.0], F32), np.full((n, 2), [300.0, 100.0], F32))
    x = rng.permutation(640)[:n].astype(F32)
    line = (np.stack([x, np.full(n, 240, F32)], 1), np.stack([x + 17, np.full(n, 240, F32)], 1))
    tri0 = np.array([[10, 20], [300, 40], [150, 400]], F32)
    tri1 = np.array([[30, 10], [320, 60], [140, 380]], F32)
    k = rng.integers(0, 3, n)
    three = (tri0[k], tri1[k])
    q0 = np.array([[100, 200], [300, 200], [500, 200], [250, 400]], F32)
    four = (q0, q0 + np.array([20, -10], F32))
    return [("identical", *ident), ("horizontal_line", *line), ("three_repeated", *three), ("four_three_collinear", *four)]


def test_homography_degenerate_inputs():
    """Pairs with no non-degenerate 4-point sample report no model, like n < 4: identity H, empty mask, n_inliers 0, and
    find_homography returns None.  A generic 4-point pair still gives its exact H; a negative count passes through."""
    rng = np.random.default_rng(13)
    degen = h_degenerate_scenes(rng)
    Ht = motion_h("perspective", 640, 480)
    g0 = np.array([[50, 60], [600, 40], [580, 430], [70, 420]], F32)
    generic = (g0, ref.apply_h(Ht, g0).astype(F32))
    good = h_scene(rng, 640, 480, Ht, 300, 0.6, H_THR)
    scenes = [(a, c) for _, a, c in degen] + [generic, good[:2], good[:2], good[:2]]
    p0, p1, cnt = pack(rng, scenes, 512)
    cnt[-2], cnt[-1] = 3, _lib.N_OVERFLOW
    Hg, mask, n_inl = run_h(p0, p1, cnt, H_THR, 1024, seed=2)
    assert np.isfinite(Hg).all()
    for b, (name, a, c) in enumerate(degen):
        assert np.array_equal(Hg[b], np.eye(3, dtype=F32)), name
        assert not mask[b].any() and n_inl[b] == 0, name
        Hs, ms = find_homography(a, c, thr=H_THR)
        assert Hs is None and not ms.any() and ms.shape == (len(a), 1), name
    b = len(degen)
    assert mask[b, :4].all() and not mask[b, 4:].any() and n_inl[b] == 4
    assert grid_dist(Hg[b].astype(np.float64), Ht, 640, 480) < 1e-5 * 800
    assert np.array_equal(mask[b + 1, :300], good[2]) and n_inl[b + 1] == good[2].sum()
    for b, want in ((len(scenes) - 2, 0), (len(scenes) - 1, _lib.N_OVERFLOW)):
        assert np.array_equal(Hg[b], np.eye(3, dtype=F32)) and not mask[b].any() and n_inl[b] == want


def test_homography_deterministic_and_isolated():
    """The same call gives the same bits; a pair's outputs do not depend on the other pairs of its batch (samples are seeded by
    batch position, so each pair keeps its position), degenerate neighbours included, nor on the padding n_max."""
    rng = np.random.default_rng(17)
    keys, scenes = noisy_h_batch(rng, n_list=(200, 900), fracs=(0.5,), noises=(0.5,), motions=("rot90", "scale3", "perspective"))
    p0, p1, cnt = pack(rng, scenes, 1024)
    out = run_h(p0, p1, cnt, H_THR, 1024, seed=4)
    again = run_h(p0, p1, cnt, H_THR, 1024, seed=4)
    for x, y in zip(out, again):
        assert np.array_equal(x, y)
    degen = h_degenerate_scenes(rng)
    _, other = noisy_h_batch(rng, n_list=(200, 900), fracs=(0.3,), noises=(1.0,), motions=("rot90", "scale3", "perspective"))
    for keep in (0, 3, len(scenes) - 1):
        mixed = [scenes[b] if b == keep else (degen[b % len(degen)][1:] if b % 2 else other[b][:2]) for b in range(len(scenes))]
        q0, q1, qc = pack(rng, mixed, 1024)
        got = run_h(q0, q1, qc, H_THR, 1024, seed=4)
        for x, y in zip(got, out):
            assert np.array_equal(x[keep], y[keep]), keep
    keep = 1
    n = int(cnt[keep])
    got = run_h(p0[:keep + 1, :n].copy(), p1[:keep + 1, :n].copy(), cnt[:keep + 1], H_THR, 1024, seed=4)
    assert np.array_equal(got[0][keep], out[0][keep]) and np.array_equal(got[1][keep], out[1][keep, :n])
    assert got[2][keep] == out[2][keep]


# ---------------------------------------------------------------------------------------------------------------------------
# essential matrix
# ---------------------------------------------------------------------------------------------------------------------------
# (focal length, image size): a 56 degree and a 120 degree horizontal field of view
CAMS = [(600.0, 640, 480), (320.0 / np.tan(np.radians(60)), 640, 480)]
E_MOTIONS = {
    "sideways": ([0.0, 0.05, 0.0], [0.5, 0.0, 0.0], (2.0, 8.0)),
    "forward": ([0.0, 0.0, 0.02], [0.0, 0.0, -0.8], (2.0, 8.0)),       # epipole at the image centre
    "small_baseline": ([0.01, -0.01, 0.0], [0.09, 0.03, 0.02], (3.0, 7.0)),   # |t| / depth ~ 0.02
    "rot30": ([0.0, np.radians(30), 0.0], [-0.8, 0.1, 0.2], (2.0, 8.0)),
}


def e_scene(rng, f, W, H, rvec, t, depth, n, frac, thr, noise_px=0.0):
    """n normalised correspondences of 3-D points seen by a W x H camera of focal length f at depths `depth` in view 0, in
    front of view 1 (X1 = R X0 + t); round(frac n) inliers (noise `noise_px` px on both views), the rest outliers redrawn in
    both views until their true Sampson distance is >= 20 thr.  Returns x0, x1 (float32), the true mask, R, t, E_true."""
    R, t = ref.rodrigues(rvec), np.asarray(t, np.float64)
    X0 = np.zeros((0, 3))
    while len(X0) < n:
        m = 4 * n + 16
        px = rng.uniform([0, 0], [W, H], (m, 2))
        X = np.concatenate([(px - [W / 2, H / 2]) / f, np.ones((m, 1))], 1) * rng.uniform(*depth, (m, 1))
        X0 = np.concatenate([X0, X[(X @ R.T + t)[:, 2] > 0.2]])[:n]
    X1 = X0 @ R.T + t
    x0, x1 = X0[:, :2] / X0[:, 2:], X1[:, :2] / X1[:, 2:]
    if noise_px:
        x0, x1 = x0 + rng.normal(0, noise_px / f, x0.shape), x1 + rng.normal(0, noise_px / f, x1.shape)
    x0, x1 = x0.astype(F32), x1.astype(F32)
    E = ref.essential_from_pose(R, t)
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:int(round(frac * n))]] = True
    lim = np.array([W / 2, H / 2]) / f
    bad = ~inl
    while bad.any():           # both views redrawn: near the epipole every x1 is close to the epipolar line of x0
        x0[bad] = rng.uniform(-lim, lim, (bad.sum(), 2)).astype(F32)
        x1[bad] = rng.uniform(-lim, lim, (bad.sum(), 2)).astype(F32)
        bad = ~inl & (ref.sampson(E, x0, x1) < 20 * thr)
    return x0, x1, inl, R, t, E


E_NW = [(8, 1.0), (9, 1.0)] + [(n, w) for n in (100, 2000) for w in (1.0, 0.8, 0.5)]
E_BIG = [(8192, w) for w in (1.0, 0.8, 0.5)]
E_THR_PX = 1.5
E_ITERS = 16384
E_TOL = 1e-4           # |E/|E| -+ E_true/|E_true|| elementwise; measured 7.6e-5
# pose from the GPU E on its mask: rotation and translation-direction error (degrees).  With 8 or 9 points the minimal problem
# is ill-conditioned in the float32 inputs themselves: the float64 8-point on the same float32 points is off by up to 3.7e-4
# deg in rotation and 1.6e-2 deg in translation over 160 such scenes, so those get 1e-2 / 5e-2 deg.
ROT_TOL_DEG, T_TOL_DEG = 1e-3, 1e-2              # measured: 4.5e-5, 2.5e-3
ROT_TOL_MIN_DEG, T_TOL_MIN_DEG = 1e-2, 5e-2      # measured: 2.7e-3, 5.5e-3
SV_TOL = 1e-5          # |s1 - 1|, |s2 - 1|, s3 of every returned non-zero E; measured 3.2e-8


def e_singular_dev(E):
    s = np.linalg.svd(E.astype(np.float64), compute_uv=False)
    return max(abs(s[0] - 1), abs(s[1] - 1), s[2])


def test_essential_exact_recovery():
    """Noise-free scenes over both cameras, four motions, counts and inlier fractions: the mask is the true inlier set, E is
    +-E_true up to scale, essential, and recover_pose on the GPU mask gives the true pose."""
    rng = np.random.default_rng(21)
    worst = dict(e=0.0, sv=0.0, rot=0.0, t=0.0, rot_min=0.0, t_min=0.0)
    for group, n_max in ((E_NW, 2048), (E_BIG, 8192)):
        keys, scenes = [], []
        for f, W, H in CAMS:
            for name, (rv, t, depth) in E_MOTIONS.items():
                for n, w in group:
                    keys.append((f, name, n, w))
                    scenes.append(e_scene(rng, f, W, H, rv, t, depth, n, w, E_THR_PX / f))
        # one threshold per call, 1.5 px at f = 600: every inlier is exact, every outlier of either camera is further than
        # 20 times this
        thr = E_THR_PX / CAMS[0][0]
        x0, x1, cnt = pack(rng, [s[:2] for s in scenes], n_max)
        Eg, mask, n_inl = run_e(x0, x1, cnt, thr, E_ITERS, seed=1)
        for b, ((f, name, n, w), (a, c, inl, R, t, Et)) in enumerate(zip(keys, scenes)):
            what = f"f={f:.0f} {name} n={n} w={w}"
            assert np.array_equal(mask[b, :n], inl) and not mask[b, n:].any() and n_inl[b] == inl.sum(), what
            E = Eg[b].astype(np.float64)
            En, Etn = E / np.linalg.norm(E), Et / np.linalg.norm(Et)
            de = min(np.abs(En - Etn).max(), np.abs(En + Etn).max())
            sv = e_singular_dev(Eg[b])
            Rg, tg = recover_pose(E, a[inl].astype(np.float64), c[inl].astype(np.float64))
            dr, dt = ref.rotation_angle_deg(Rg.T @ R), ref.angle_between_deg(tg, t)
            for k, v in (("e", de), ("sv", sv), ("rot" if n > 9 else "rot_min", dr), ("t" if n > 9 else "t_min", dt)):
                worst[k] = max(worst[k], v)
            assert de < E_TOL and sv < SV_TOL, (what, de, sv)
            if n <= 9:
                assert dr < ROT_TOL_MIN_DEG and dt < T_TOL_MIN_DEG, (what, dr, dt)
                continue
            assert dr < ROT_TOL_DEG and dt < T_TOL_DEG, (what, dr, dt)
    print("essential exact recovery, worst: |E - E_true| {e:.2e}, singular values {sv:.2e}, rotation {rot:.2e} deg, "
          "translation {t:.2e} deg (n <= 9: {rot_min:.2e}, {t_min:.2e} deg)".format(**worst))


def noisy_e_batch(rng, thr_px, fracs=(0.5, 0.7), n_list=(300, 2000), noise_px=0.5):
    keys, scenes = [], []
    for f, W, H in CAMS:
        for name, (rv, t, depth) in E_MOTIONS.items():
            for n in n_list:
                for w in fracs:
                    keys.append((f, name, n, w))
                    scenes.append(e_scene(rng, f, W, H, rv, t, depth, n, w, thr_px / f, noise_px))
    return keys, scenes


@pytest.mark.parametrize("thr_px", [0.5, 1.5, 5.0])
def test_essential_mask_is_sampson_below_thr(thr_px):
    """The mask is `Sampson < thr` under the returned E, in float64 from the normalised points; n_inliers is its size; rows
    past the count are never inliers; every returned E is essential.  One call per camera, thr in its normalised units."""
    rng = np.random.default_rng(int(thr_px * 10) + 30)
    keys, scenes = noisy_e_batch(rng, thr_px, n_list=(300, 1500), noise_px=thr_px / 3)
    sv_worst = 0.0
    for f, _, _ in CAMS:
        idx = [b for b, k in enumerate(keys) if k[0] == f]
        x0, x1, cnt = pack(rng, [scenes[b][:2] for b in idx], 2048)
        thr = thr_px / f
        Eg, mask, n_inl = run_e(x0, x1, cnt, thr, 4096, seed=2)
        for j, b in enumerate(idx):
            n = int(cnt[j])
            what = str(keys[b])
            assert_mask_rule(ref.sampson(Eg[j], x0[j, :n], x1[j, :n]), mask[j, :n], thr, what)
            assert n_inl[j] == mask[j].sum() and not mask[j, n:].any(), what
            sv = e_singular_dev(Eg[j])
            sv_worst = max(sv_worst, sv)
            assert sv < SV_TOL, (what, sv)
    print(f"thr {thr_px} px: worst singular-value deviation {sv_worst:.2e}")


def test_essential_msac_cost_reaches_truth():
    """0.5 px noise, 70 % and 50 % inliers: the MSAC cost of the returned E (Sampson, float64) is within 5 % of the true E's,
    i.e. the local optimisation reaches the optimum near the truth.  2 % as for the homography is not met: the 30 degree
    rotation at f = 600 (500 points, 70 % inliers) ends at 1.022 times the true cost.

    Not for the small baseline (|t| / depth ~ 0.02): there the 8-point hypotheses and the Sampson-weighted refits of
    rs_local_opt stop short of the optimum, at up to 1.20 times the true cost.  Those
    ratios are printed, not asserted; closing that gap is a change to the local optimisation, not to this test."""
    rng = np.random.default_rng(41)
    keys, scenes = noisy_e_batch(rng, E_THR_PX, fracs=(0.5, 0.7), n_list=(500, 2000))
    ratios, small = [], []
    for f, _, _ in CAMS:
        idx = [b for b, k in enumerate(keys) if k[0] == f]
        x0, x1, cnt = pack(rng, [scenes[b][:2] for b in idx], 2048)
        thr = E_THR_PX / f
        Eg, _, _ = run_e(x0, x1, cnt, thr, E_ITERS, seed=3)
        for j, b in enumerate(idx):
            n = int(cnt[j])
            Et = scenes[b][5]
            r = (ref.msac_cost(ref.sampson(Eg[j], x0[j, :n], x1[j, :n]), thr) /
                 ref.msac_cost(ref.sampson(Et, x0[j, :n], x1[j, :n]), thr))
            if keys[b][1] == "small_baseline":
                small.append(r)
                continue
            ratios.append((r, keys[b]))
    worst = max(ratios)
    print(f"essential MSAC cost / true cost: max {worst[0]:.4f} {worst[1]}, median {np.median([r for r, _ in ratios]):.4f}; "
          f"small baseline (not asserted): max {max(small):.4f}")
    assert worst[0] <= E_COST_TOL, worst


def test_essential_degenerate_inputs():
    """n < 8, a negative count, all points identical, a planar scene and pure rotation (t = 0).  The 8-point solver makes no
    rank test, so the identical and planar cases may legitimately report a model: only consistency is pinned -- finite
    outputs, the mask is `Sampson < thr` under the returned E, n_inliers is its size, and n < 8 gives zero E."""
    rng = np.random.default_rng(51)
    f = 600.0
    thr = E_THR_PX / f
    full = e_scene(rng, f, 640, 480, *E_MOTIONS["sideways"], 300, 1.0, thr)
    ident = (np.full((100, 2), [0.1, -0.2], F32), np.full((100, 2), [0.15, -0.18], F32))
    # planar: every point on the plane Z = 4 + 0.3 X
    R, t = ref.rodrigues([0.02, 0.1, 0.0]), np.array([0.4, 0.1, 0.05])
    xy = rng.uniform(-0.5, 0.5, (400, 2))
    Z = 4.0 / (1 - 0.3 * xy[:, 0])
    X0 = np.concatenate([xy, np.ones((400, 1))], 1) * Z[:, None]
    X1 = X0 @ R.T + t
    plane = ((X0[:, :2] / X0[:, 2:]).astype(F32), (X1[:, :2] / X1[:, 2:]).astype(F32))
    X1r = X0 @ ref.rodrigues([0.05, -0.1, 0.02]).T
    rotation = ((X0[:, :2] / X0[:, 2:]).astype(F32), (X1r[:, :2] / X1r[:, 2:]).astype(F32))
    scenes = [full[:2], full[:2], full[:2], full[:2], ident, plane, rotation]
    x0, x1, cnt = pack(rng, scenes, 512)
    cnt[1], cnt[2], cnt[3] = 7, 0, _lib.N_OVERFLOW
    Eg, mask, n_inl = run_e(x0, x1, cnt, thr, 4096, seed=4)
    assert np.isfinite(Eg).all()
    for b in range(len(scenes)):
        n = max(int(cnt[b]), 0)
        assert n_inl[b] == (cnt[b] if cnt[b] < 0 else mask[b].sum()) and not mask[b, n:].any(), b
        if n < 8:
            assert not Eg[b].any() and not mask[b].any(), b
        else:
            assert_mask_rule(ref.sampson(Eg[b], x0[b, :n], x1[b, :n]), mask[b, :n], thr, b)
    assert n_inl[0] == 300


def test_essential_deterministic_and_isolated():
    """As the homography: same bits twice, and a pair's outputs do not depend on the other pairs of its batch."""
    rng = np.random.default_rng(61)
    keys, scenes = noisy_e_batch(rng, E_THR_PX, fracs=(0.6,), n_list=(300,))
    scenes = [s[:2] for s in scenes]
    thr = E_THR_PX / 600.0
    x0, x1, cnt = pack(rng, scenes, 512)
    out = run_e(x0, x1, cnt, thr, 2048, seed=6)
    again = run_e(x0, x1, cnt, thr, 2048, seed=6)
    for x, y in zip(out, again):
        assert np.array_equal(x, y)
    _, other = noisy_e_batch(rng, E_THR_PX, fracs=(0.4,), n_list=(400,))
    ident = (np.full((100, 2), [0.1, -0.2], F32), np.full((100, 2), [0.15, -0.18], F32))
    for keep in (0, 5, len(scenes) - 1):
        mixed = [scenes[b] if b == keep else (ident if b % 3 == 0 else other[b][:2]) for b in range(len(scenes))]
        q0, q1, qc = pack(rng, mixed, 512)
        got = run_e(q0, q1, qc, thr, 2048, seed=6)
        for x, y in zip(got, out):
            assert np.array_equal(x[keep], y[keep]), keep
