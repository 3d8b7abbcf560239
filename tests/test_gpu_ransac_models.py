"""Homography, essential- and fundamental-matrix RANSAC on the GPU (xfeat_ransac_homography / _essential / _fundamental,
geometry.find_homography_batch / find_essential_batch / find_fundamental_batch) against the float64 references of
tests/ransac_ref.py, and the 7-point step alone through its test hook (xfeat_debug_seven_point).

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
from accelerated_features_b200.geometry import (find_essential_batch, find_fundamental_batch, find_homography,
                                                find_homography_batch, recover_pose)
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
    """Pairs with no non-degenerate 4-point sample report no model, like n < 4 and a batch with n_max = 0: identity H, empty
    mask, n_inliers 0, and find_homography returns None.  A generic 4-point pair still gives its exact H; a negative count
    passes through."""
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
    # a batch without correspondences (n_max = 0): every pair has no model
    Hg, mask, n_inl = run_h(np.zeros((3, 0, 2), F32), np.zeros((3, 0, 2), F32), None, H_THR, 1024, seed=2)
    assert np.array_equal(Hg, np.broadcast_to(np.eye(3, dtype=F32), (3, 3, 3))) and mask.shape == (3, 0) and not n_inl.any()


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


# ---------------------------------------------------------------------------------------------------------------------------
# fundamental matrix
# ---------------------------------------------------------------------------------------------------------------------------
def cam(W, H, fov_scale, pp=(0.52, 0.47)):
    """(K, (W, H)): focal length fov_scale * W, principal point off the image centre."""
    return ref.intrinsics(fov_scale * W, pp[0] * W, pp[1] * H), (W, H)


# image 0 and image 1 share K where the sizes are equal; the mixed pairs differ in size, focal length and principal point
SAME_PAIRS = [(cam(W, H, 0.9), cam(W, H, 0.9)) for W, H in SIZES]
MIXED_PAIRS = [(cam(64, 48, 0.8), cam(3840, 2160, 1.2, (0.49, 0.53))), (cam(640, 480, 0.9), cam(3840, 2160, 1.3, (0.55, 0.45))),
               (cam(3840, 2160, 0.85), cam(64, 48, 1.25, (0.45, 0.55)))]
F_MOTIONS = {
    "general": ([0.08, -0.12, 0.05], [0.5, 0.15, 0.25], (2.0, 8.0)),
    "sideways": ([0.0, 0.0, 0.04], [0.5, 0.0, 0.0], (2.0, 8.0)),          # R^T t and t have no z: both epipoles at infinity
    "forward": ([0.0, 0.0, 0.03], [0.0, 0.0, -0.8], (2.0, 8.0)),          # epipoles at the principal points
    "small_baseline": ([0.01, -0.01, 0.0], [0.06, 0.02, 0.015], (3.0, 7.0)),
}
F_THR = 1.0


def pair_name(pair):
    (_, (W0, H0)), (_, (W1, H1)) = pair
    return f"{W0}x{H0}-{W1}x{H1}"


def pair_diag(pair):
    return max(np.hypot(*pair[0][1]), np.hypot(*pair[1][1]))


def f_scene(rng, pair, motion, n, frac, thr, noise=0.0, far_mult=10.0):
    """n pixel correspondences of the two-view scene (pair, motion): exact float64 projections (plus Gaussian noise of `noise` px
    in both images) rounded to float32, round(frac n) inliers, the rest redrawn in both images until their Sampson distance under
    F_true is >= far_mult thr (at most a fifth of the smaller image's diagonal, which a 64 x 48 image can still reach).  Returns p0,
    p1, the true mask and F_true."""
    (K0, s0), (K1, s1) = pair
    rv, t, depth = F_MOTIONS[motion]
    R, t = ref.rodrigues(rv), np.asarray(t, np.float64)
    p0, p1 = ref.two_view_points(rng, K0, K1, s0, s1, R, t, n, depth)
    if noise:
        p0, p1 = p0 + rng.normal(0, noise, p0.shape), p1 + rng.normal(0, noise, p1.shape)
    p0, p1 = p0.astype(F32), p1.astype(F32)
    F = ref.fundamental_from_cameras(K0, K1, R, t)
    far = min(far_mult * thr, 0.2 * min(np.hypot(*s0), np.hypot(*s1)))
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:int(round(frac * n))]] = True
    bad = ~inl
    while bad.any():
        p0[bad] = rng.uniform([0, 0], s0, (bad.sum(), 2)).astype(F32)
        p1[bad] = rng.uniform([0, 0], s1, (bad.sum(), 2)).astype(F32)
        bad = ~inl & (ref.sampson(F, p0, p1) < far)
    return p0, p1, inl, F


def held_out(rng, pair, motion, n=1000):
    """Exact float64 correspondences of the scene spread over the images, none of them seen by the estimator."""
    (K0, s0), (K1, s1) = pair
    rv, t, depth = F_MOTIONS[motion]
    return ref.two_view_points(rng, K0, K1, s0, s1, ref.rodrigues(rv), np.asarray(t, np.float64), n, depth)


def all_inlier_samples(n, k, iters):
    """Expected number of 7-point samples (without replacement) drawn only from the k inliers of n points."""
    return iters * float(np.prod([(k - j) / (n - j) for j in range(7)]))


def run_f(p0, p1, cnt, thr, iters, seed, pair_ids=None):
    F, m, n = find_fundamental_batch(torch.from_numpy(p0).cuda(), torch.from_numpy(p1).cuda(),
                                     None if cnt is None else torch.from_numpy(cnt).cuda(), thr=thr, iters=iters, seed=seed,
                                     pair_ids=pair_ids)
    return F.cpu().numpy().reshape(-1, 3, 3), m.cpu().numpy(), n.cpu().numpy()


def rank_ratio(F):
    s = np.linalg.svd(np.asarray(F, np.float64), compute_uv=False)
    return s[2] / s[0]


def sign_dist(A, B):
    A, B = A / np.linalg.norm(A), B / np.linalg.norm(B)
    return float(min(np.abs(A - B).max(), np.abs(A + B).max()))


def run_seven_point(samples):
    """xfeat_debug_seven_point on (m, 7, 4) float32 normalised samples: candidates (m, 3, 3, 3) and counts (m)."""
    lib = _lib.load()
    s = torch.from_numpy(np.ascontiguousarray(samples, F32)).cuda()
    m = s.shape[0]
    F = torch.empty((m, 3, 9), dtype=torch.float32, device="cuda")
    cnt = torch.empty((m,), dtype=torch.int32, device="cuda")
    _lib.check(lib.xfeat_debug_seven_point(s.data_ptr(), m, F.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "xfeat_debug_seven_point")
    return F.cpu().numpy().reshape(m, 3, 3, 3), cnt.cpu().numpy()


# 7-point solver against seven_point in float64 on the same float32 inputs
SP_TOL = 1e-6          # each GPU candidate to its reference candidate, elementwise up to sign; measured: 3.4e-8
SP_RES_TOL = 1e-6      # |rows . f| / max|rows| and |det F| of every GPU candidate (unit norm); measured: 5.5e-8


def cubic_flags(c):
    """True where the cubic is close to losing a root: a tiny leading coefficient, or two roots (a near-double real root, or a
    complex pair about to become real) within 1e-3 of each other."""
    c = np.asarray(c, np.float64) / np.abs(c).max()
    if abs(c[0]) < 1e-6:
        return True
    r = np.roots(c)
    return any(abs(r[i] - r[j]) < 1e-3 * max(1.0, abs(r[i])) for i in range(3) for j in range(i + 1, 3))


def compare_seven_point(samples, what):
    """Compare the hook's candidate sets with the reference's, up to sign.  Returns (counts, worst candidate distance, worst
    residual, number of flagged samples whose counts differ)."""
    Fg, ng = run_seven_point(samples)
    assert np.isfinite(Fg).all() and ((ng >= 0) & (ng <= 3)).all(), what
    worst_d = worst_r = 0.0
    differ, counts = 0, []
    for i, smp in enumerate(samples.astype(np.float64)):
        x0, x1 = smp[:, :2], smp[:, 2:]
        cands, c = ref.seven_point(x0, x1)
        A = ref.epipolar_rows(x0, x1)
        k = int(ng[i])
        counts.append(len(cands))
        assert not Fg[i, k:].any(), (what, i)
        for F in Fg[i, :k].astype(np.float64):
            r = max(np.abs(A @ F.ravel()).max() / np.abs(A).max(), abs(np.linalg.det(F)), abs(np.linalg.norm(F) - 1))
            worst_r = max(worst_r, r)
            assert r < SP_RES_TOL, (what, i, r)
        if k != len(cands):
            assert cubic_flags(c), (what, i, k, len(cands), c)
            differ += 1
            continue
        for F in Fg[i, :k].astype(np.float64):
            d = min(sign_dist(F, G) for G in cands)
            worst_d = max(worst_d, d)
            assert d < SP_TOL, (what, i, d)
        for G in cands:
            assert min(sign_dist(F, G) for F in Fg[i, :k].astype(np.float64)) < SP_TOL, (what, i)
    return np.array(counts), worst_d, worst_r, differ


def cubic_scan(rng, m):
    """m random N(0, 1) samples and the discriminant of each one's cubic (coefficients scaled to max 1), vectorised."""
    s = rng.normal(0, 1, (m, 7, 4)).astype(F32)
    x = s.astype(np.float64)
    h0 = np.concatenate([x[..., :2], np.ones((m, 7, 1))], -1)
    h1 = np.concatenate([x[..., 2:], np.ones((m, 7, 1))], -1)
    A = (h1[..., :, None] * h0[..., None, :]).reshape(m, 7, 9)
    Vt = np.linalg.svd(A)[2]
    F1, F2 = Vt[:, -2].reshape(m, 3, 3), Vt[:, -1].reshape(m, 3, 3)
    lam = np.array([0.0, 1.0, -1.0, 2.0])
    d = np.stack([np.linalg.det(l * F1 + (1 - l) * F2) for l in lam], 1)
    c = np.linalg.solve(np.vander(lam, 4), d.T).T                           # (c3, c2, c1, c0)
    c /= np.abs(c).max(1, keepdims=True)
    a, b, cc, dd = c.T
    disc = 18 * a * b * cc * dd - 4 * b ** 3 * dd + b * b * cc * cc - 4 * a * cc ** 3 - 27 * a * a * dd * dd
    return s, disc


def test_seven_point_solver_vs_float64():
    """The 7-point step of ransac_hyp_kernel<RsFundamental> (normal matrix, Jacobi null space, cubic, roots, Newton polish) through
    xfeat_debug_seven_point, against seven_point in float64 on the same float32 samples.  The candidate set does not depend on
    the null-space basis, so sets are compared up to sign: equal counts and each candidate close to one of the other side's.
    Where the cubic is close to losing a root (cubic_flags) a count difference is allowed and reported; every GPU candidate
    must still satisfy its 7 rows and be singular."""
    rng = np.random.default_rng(71)
    # random general samples: both the one-root and the three-root branch, often
    s = rng.normal(0, 1, (4000, 7, 4)).astype(F32)
    counts, d, r, differ = compare_seven_point(s, "random")
    n1, n3 = int((counts == 1).sum()), int((counts == 3).sum())
    print(f"7-point, 4000 random samples: {n1} with 1 root, {n3} with 3; worst candidate distance {d:.2e}, residual {r:.2e}, "
          f"{differ} flagged count differences")
    assert n1 > 400 and n3 > 400              # measured: 1059 and 2941
    assert differ <= 20                      # measured: 0
    # samples of true scenes, in the pair's normalised frame: one candidate is +-Fn_true
    worst_t = worst_r = 0.0
    for pair in SAME_PAIRS + MIXED_PAIRS:
        for motion in F_MOTIONS:
            p0, p1, _, F = f_scene(rng, pair, motion, 350, 1.0, F_THR)
            nz = ref.pair_normaliser(p0, p1)
            T0, T1 = ref.pair_norm_matrices(nz)
            Fn = np.linalg.inv(T1).T @ F @ np.linalg.inv(T0)
            a, b = (ref._h(p0) @ T0.T)[:, :2], (ref._h(p1) @ T1.T)[:, :2]
            smp = np.concatenate([a, b], 1).reshape(50, 7, 4).astype(F32)
            what = f"{pair_name(pair)} {motion}"
            compare_seven_point(smp, what)
            Fg, ng = run_seven_point(smp)
            for i in range(50):
                # the float32 rounding of the inputs moves the exact solution: by up to 2.6e-3 for the small baseline seen from
                # 64 x 48, so the GPU is held to the float64 solver's distance on the same inputs
                dr = min(sign_dist(G, Fn) for G in ref.seven_point(smp[i, :, :2].astype(np.float64), smp[i, :, 2:].astype(np.float64))[0])
                dt = min(sign_dist(Fg[i, j].astype(np.float64), Fn) for j in range(ng[i])) if ng[i] else np.inf
                worst_t, worst_r = max(worst_t, dt), max(worst_r, dr)
                assert dr < SP_TRUE_TOL and dt < dr + SP_TOL, (what, i, dt, dr)
    print(f"7-point on true scenes: worst distance to +-Fn_true {worst_t:.2e} (float64 on the same inputs {worst_r:.2e})")
    # the samples with the smallest discriminant in a scan of 100 000
    s, disc = cubic_scan(rng, 100000)
    near = s[np.argsort(np.abs(disc))[:300]]
    counts, d, r, differ = compare_seven_point(near, "small discriminant")
    print(f"7-point, 300 smallest discriminants (max |disc| {np.sort(np.abs(disc))[299]:.1e}): worst distance {d:.2e}, "
          f"residual {r:.2e}, {differ} flagged count differences")


SP_TRUE_TOL = 1e-2     # float64 candidate to +-Fn_true from float32 scene samples; measured: 2.6e-3 (small baseline, 64 x 48)


def test_seven_point_rank_deficient_samples():
    """Seven identical points, and points collinear in both images: the null space is wider than 2 and the kernel's basis is
    whatever Jacobi returns.  Pinned: three candidates each, finite, unit-norm, singular and satisfying the 7 rows."""
    ident = np.tile(np.array([0.3, -0.2, 0.5, 0.1], F32), (7, 1))
    t = np.linspace(-1, 1, 7)
    collinear = np.stack([t, 0.5 * t + 0.1, 0.8 * t - 0.3, -0.2 * t + 0.4], 1).astype(F32)
    Fg, ng = run_seven_point(np.stack([ident, collinear]))
    print(f"rank-deficient samples: candidate counts identical {ng[0]}, collinear {ng[1]}")
    assert np.isfinite(Fg).all() and list(ng) == [3, 3]
    for i, smp in enumerate((ident, collinear)):
        A = ref.epipolar_rows(smp[:, :2].astype(np.float64), smp[:, 2:].astype(np.float64))
        assert not Fg[i, ng[i]:].any()
        for F in Fg[i, :ng[i]].astype(np.float64):
            assert abs(np.linalg.norm(F) - 1) < 1e-6 and abs(np.linalg.det(F)) < SP_RES_TOL
            assert np.abs(A @ F.ravel()).max() < SP_RES_TOL


F_NW = [(8, 1.0), (9, 1.0)] + [(n, w) for n in (64, 1000) for w in (1.0, 0.7, 0.5)]
F_BIG = [(8192, w) for w in (1.0, 0.7, 0.5)]
F_ITERS = 8192
# Exact recovery classifies at 0.1 px with outliers >= 10 px away (100 thr).  At 1 px with outliers >= 10 px, 45 exact inliers of
# a 64 x 48 image do not pin F down: an F within 0.11 px of every inlier also takes in an outlier, and its MSAC cost is lower
# than the truth's.
F_EXACT_THR = 0.1
# worst Sampson distance of 1000 held-out exact correspondences under F_gpu, over the larger image diagonal.  n = 8 and 9 need
# no looser limit than the rest: measured 2.3e-6 there.
F_HELD_TOL = 1e-5      # measured: 3.4e-6 (one K per pair), 4.3e-7 (mixed sizes)
F_RANK_TOL = 1e-8      # sigma3 / sigma1 of F_gpu; measured: 7.2e-10


def f_exact_recovery(pairs, seed):
    rng = np.random.default_rng(seed)
    worst = dict(held=0.0, held_min=0.0, rank=0.0)
    expect = []
    for group, n_max in ((F_NW, 1024), (F_BIG, 8192)):
        keys, scenes = [], []
        for pair in pairs:
            for motion in F_MOTIONS:
                for n, w in group:
                    keys.append((pair, motion, n, w))
                    scenes.append(f_scene(rng, pair, motion, n, w, F_EXACT_THR, far_mult=100.0))
                    expect.append(all_inlier_samples(n, int(round(w * n)), F_ITERS))
        p0, p1, cnt = pack(rng, [s[:2] for s in scenes], n_max)
        Fg, mask, n_inl = run_f(p0, p1, cnt, F_EXACT_THR, F_ITERS, seed=1)
        for b, ((pair, motion, n, w), (a, c, inl, Ft)) in enumerate(zip(keys, scenes)):
            what = f"{pair_name(pair)} {motion} n={n} w={w}"
            assert np.array_equal(mask[b, :n], inl) and not mask[b, n:].any() and n_inl[b] == inl.sum(), what
            F = Fg[b].astype(np.float64)
            assert abs(np.linalg.norm(F) - 1) < 1e-6, what
            h0, h1 = held_out(rng, pair, motion)
            d = ref.sampson(F, h0, h1).max() / pair_diag(pair)
            rr = rank_ratio(F)
            key = "held" if n > 9 else "held_min"
            worst[key] = max(worst[key], d)
            worst["rank"] = max(worst["rank"], rr)
            assert d < F_HELD_TOL, (what, d)
            assert rr < F_RANK_TOL, (what, rr)
    print(f"{F_ITERS} samples, at least {min(expect):.0f} all-inlier ones expected per pair; worst held-out Sampson / diagonal "
          f"{worst['held']:.2e} (n <= 9: {worst['held_min']:.2e}), sigma3 / sigma1 {worst['rank']:.2e}")


def test_fundamental_exact_recovery():
    """Noise-free scenes, one K for both images, three image sizes, four motions (general, epipoles at infinity, epipole in the
    image, small baseline), n from 8 to 8192 at w = 1, 0.7 and 0.5: the mask is the true inlier set, and F is +-F_true --
    1000 held-out exact correspondences lie on its epipolar geometry -- unit norm and rank 2."""
    f_exact_recovery(SAME_PAIRS, 81)


def test_fundamental_exact_recovery_mixed_sizes():
    """As test_fundamental_exact_recovery for two cameras that differ in focal length, principal point and image size, down to
    64 x 48 against 3840 x 2160: the pairs the single shared normalisation scale conditions worst."""
    f_exact_recovery(MIXED_PAIRS, 82)


def crop_pair(offset=(6700.0, 4800.0)):
    """A 640 x 480 camera pair whose pixel coordinates sit near (7000, 5000), like a crop of a large panorama."""
    (K0, _), (K1, _) = cam(640, 480, 0.9), cam(640, 480, 1.0, (0.5, 0.5))
    return K0, K1, offset


def f_crop_scene(rng, motion, n, frac, thr, noise):
    K0, K1, off = crop_pair()
    shift = np.array([[1, 0, off[0]], [0, 1, off[1]], [0, 0, 1.0]])
    pair = ((shift @ K0, (640 + off[0], 480 + off[1])), (shift @ K1, (640 + off[0], 480 + off[1])))
    rv, t, depth = F_MOTIONS[motion]
    R, t = ref.rodrigues(rv), np.asarray(t, np.float64)
    p0, p1 = ref.two_view_points(rng, K0, K1, (640, 480), (640, 480), R, t, n, depth)
    p0, p1 = p0 + off + rng.normal(0, noise, p0.shape), p1 + off + rng.normal(0, noise, p1.shape)
    F = ref.fundamental_from_cameras(pair[0][0], pair[1][0], R, t)
    p0, p1 = p0.astype(F32), p1.astype(F32)
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:int(round(frac * n))]] = True
    bad = ~inl
    while bad.any():
        p0[bad] = (rng.uniform([0, 0], [640, 480], (bad.sum(), 2)) + off).astype(F32)
        p1[bad] = (rng.uniform([0, 0], [640, 480], (bad.sum(), 2)) + off).astype(F32)
        bad = ~inl & (ref.sampson(F, p0, p1) < 10 * thr)
    return p0, p1, inl, F


@pytest.mark.parametrize("thr", [0.5, 1.5, 5.0])
def test_fundamental_mask_is_sampson_below_thr(thr):
    """The mask is `Sampson < thr` under the returned F, in float64 from the pixel points, on the three sizes, the mixed pairs
    and a pair near (7000, 5000); n_inliers is its size, nothing is set past the count, F is unit norm and rank 2.  Near
    (7000, 5000) a float32 evaluation of the pixel Sampson distance is off by up to 0.17 px, which fails this at 0.5 px: the
    classification is made in fp64 (ransac_final_kernel<RsFundamental>)."""
    rng = np.random.default_rng(int(thr * 10) + 90)
    keys, scenes = [], []
    for pair in SAME_PAIRS + MIXED_PAIRS:
        for motion in ("general", "sideways", "forward"):
            for n, w in ((300, 0.5), (1500, 0.7)):
                keys.append(f"{pair_name(pair)} {motion} n={n} w={w}")
                scenes.append(f_scene(rng, pair, motion, n, w, thr, thr / 3))
    for motion in ("general", "forward"):
        for n, w in ((300, 0.5), (1500, 0.7)):
            keys.append(f"crop near (7000, 5000) {motion} n={n} w={w}")
            scenes.append(f_crop_scene(rng, motion, n, w, thr, thr / 3))
    p0, p1, cnt = pack(rng, [s[:2] for s in scenes], 2048)
    Fg, mask, n_inl = run_f(p0, p1, cnt, thr, 4096, seed=2)
    worst_rank = 0.0
    for b, what in enumerate(keys):
        n = int(cnt[b])
        assert_mask_rule(ref.sampson(Fg[b], p0[b, :n], p1[b, :n]), mask[b, :n], thr, what)
        assert n_inl[b] == mask[b].sum() and not mask[b, n:].any(), what
        assert abs(np.linalg.norm(Fg[b].astype(np.float64)) - 1) < 1e-6, what
        worst_rank = max(worst_rank, rank_ratio(Fg[b]))
        assert rank_ratio(Fg[b]) < F_RANK_TOL, what
        assert mask[b, :n][scenes[b][2]].mean() > 0.9, what              # the estimate is the scene's, not a stray one
    print(f"thr {thr}: worst sigma3 / sigma1 {worst_rank:.2e}")


# cost(F_gpu) / min(cost(F_true), cost(refit of the true inliers)); measured: 1.032 (64x48-3840x2160, general, n = 300, w = 0.5)
F_COST_TOL = 1.05
F_FIXED_TOL = 0.02     # 1 - cost(f_lo_refit(F_gpu)) / cost(F_gpu); measured: 0.0078


def test_fundamental_msac_cost_and_refit():
    """Noisy scenes (0.3-1 px), w in {0.3, 0.5, 0.7}, n in {300, 2000}, same and mixed sizes, with at least 30 all-inlier
    samples expected per pair: the float64 pixel MSAC cost of F_gpu is at most F_COST_TOL times the lower of the true F's and
    the float64 refit of the true inliers', and one more refit (f_lo_refit) lowers it by at most F_FIXED_TOL: the local
    optimisation has converged.  Small-baseline ratios are printed, not asserted, as for E."""
    rng = np.random.default_rng(95)
    thr = 1.5
    ratios, fixed, small = [], [], []
    expect = []
    for w, iters in ((0.7, 2048), (0.5, 8192), (0.3, 163840)):
        keys, scenes = [], []
        for pair in SAME_PAIRS + MIXED_PAIRS:
            for motion in F_MOTIONS:
                for n in (300, 2000):
                    noise = (0.3, 0.6, 1.0)[len(scenes) % 3]
                    keys.append((pair_name(pair), motion, n, w, noise))
                    scenes.append(f_scene(rng, pair, motion, n, w, thr, noise))
                    expect.append(all_inlier_samples(n, int(round(w * n)), iters))
        p0, p1, cnt = pack(rng, [s[:2] for s in scenes], 2048)
        Fg, _, _ = run_f(p0, p1, cnt, thr, iters, seed=3)
        for b, (key, (a, c, inl, Ft)) in enumerate(zip(keys, scenes)):
            F = Fg[b].astype(np.float64)
            cost = ref.msac_cost(ref.sampson(F, a, c), thr)
            Fr = ref.f_lo_refit(Ft, a[inl], c[inl], 1e9)
            best = min(ref.msac_cost(ref.sampson(Ft, a, c), thr), ref.msac_cost(ref.sampson(Fr, a, c), thr))
            again = ref.msac_cost(ref.sampson(ref.f_lo_refit(F, a, c, thr), a, c), thr)
            if key[1] == "small_baseline":
                small.append((cost / best, 1 - again / cost, key))
                continue
            ratios.append((cost / best, key))
            fixed.append((1 - again / cost, key))
    print(f"at least {min(expect):.0f} all-inlier samples expected per pair")
    print(f"F MSAC cost / best reference cost: max {max(ratios)[0]:.4f} {max(ratios)[1]}, median {np.median([r for r, _ in ratios]):.4f}")
    print(f"one more refit lowers the cost by at most {max(fixed)[0]:.4f} {max(fixed)[1]}")
    print(f"small baseline (not asserted): cost ratio max {max(s[0] for s in small):.4f}, refit gain max {max(s[1] for s in small):.4f}")
    assert max(ratios)[0] <= F_COST_TOL, max(ratios)
    assert max(fixed)[0] <= F_FIXED_TOL, max(fixed)


def f_degenerate_scenes(rng):
    """(name, p0, p1) of pairs whose F the points do not determine, with integer coordinates where the degeneracy must survive
    float32."""
    n = 64
    ident = (np.full((n, 2), [100.0, 200.0], F32), np.full((n, 2), [300.0, 100.0], F32))
    tri0 = np.array([[10, 20], [300, 40], [150, 400]], F32)
    tri1 = np.array([[30, 10], [320, 60], [140, 380]], F32)
    k = rng.integers(0, 3, n)
    x = rng.permutation(640)[:n].astype(F32)
    line = (np.stack([x, np.full(n, 240, F32)], 1), np.stack([np.round(0.75 * x) + 17, np.full(n, 100, F32)], 1))
    # a plane seen by the two mixed-size cameras, and a pure rotation (t = 0) of the VGA camera
    (K0, s0), (K1, s1) = MIXED_PAIRS[1]
    R = ref.rodrigues([0.02, 0.1, 0.0])
    px = rng.uniform([0, 0], s0, (300, 2))
    rays = ref._h(px) @ np.linalg.inv(K0).T
    Z = 4.0 / (1 - 0.3 * rays[:, 0])                            # the plane Z = 4 + 0.3 X
    X1 = (rays * Z[:, None]) @ R.T + [0.4, 0.1, 0.05]
    q = X1 @ K1.T
    plane = (px.astype(F32), (q[:, :2] / q[:, 2:]).astype(F32))
    (Kr, sr), _ = SAME_PAIRS[1]
    pr = rng.uniform([0, 0], sr, (300, 2))
    qr = ref._h(pr) @ (Kr @ ref.rodrigues([0.05, -0.1, 0.02]) @ np.linalg.inv(Kr)).T
    rotation = (pr.astype(F32), (qr[:, :2] / qr[:, 2:]).astype(F32))
    return [("identical", *ident), ("three_repeated", tri0[k], tri1[k]), ("collinear", *line), ("plane", *plane),
            ("rotation", *rotation)]


def test_fundamental_degenerate_inputs():
    """n in {0, 7, 8}, a negative count, identical points, 3 correspondences repeated, points collinear in both images, a plane
    and a pure rotation.  The 7-point solver makes no rank test, so only consistency is pinned: finite outputs, n_inliers the
    mask size (a negative count passes through), n < 8 gives zero F and no mask, otherwise the mask rule holds and a non-zero F
    is unit norm and rank 2.  On the plane and the rotation every F of the family agrees with every point: all are inliers.
    Identical points centre to (0, 0, 0, 0): every sample's null space is spanned by unit matrices, the cubic vanishes, no
    candidate is found, and the pair gets a zero F and no inliers, as below 8 points.  The collinear pair ends the same way."""
    rng = np.random.default_rng(97)
    thr = 1.5
    full = f_scene(rng, SAME_PAIRS[1], "general", 300, 1.0, thr)
    degen = f_degenerate_scenes(rng)
    scenes = [full[:2]] * 4 + [(a, c) for _, a, c in degen]
    p0, p1, cnt = pack(rng, scenes, 512)
    cnt[1], cnt[2], cnt[3] = 7, 0, _lib.N_OVERFLOW
    cnt = np.append(cnt, 8)
    p0, p1 = np.concatenate([p0, p0[:1]]), np.concatenate([p1, p1[:1]])
    names = ["full", "n=7", "n=0", "overflow"] + [d[0] for d in degen] + ["n=8"]
    Fg, mask, n_inl = run_f(p0, p1, cnt, thr, 4096, seed=4)
    assert np.isfinite(Fg).all()
    for b, name in enumerate(names):
        n = max(int(cnt[b]), 0)
        assert n_inl[b] == (cnt[b] if cnt[b] < 0 else mask[b].sum()) and not mask[b, n:].any(), name
        if n < 8:
            assert not Fg[b].any() and not mask[b].any(), name
            continue
        assert_mask_rule(ref.sampson(Fg[b], p0[b, :n], p1[b, :n]), mask[b, :n], thr, name)
        if Fg[b].any():
            assert abs(np.linalg.norm(Fg[b].astype(np.float64)) - 1) < 1e-6 and rank_ratio(Fg[b]) < F_RANK_TOL, name
        print(f"{name}: {n_inl[b]} of {n} inliers, F {'non-zero' if Fg[b].any() else 'zero'}")
    assert n_inl[0] == 300 and n_inl[-1] == 8
    for name in ("plane", "rotation", "three_repeated"):
        b = names.index(name)
        assert n_inl[b] == cnt[b], name
    for name in ("identical", "collinear"):
        b = names.index(name)
        assert not Fg[b].any() and n_inl[b] == 0, name


def test_fundamental_deterministic_and_isolated():
    """Same bits twice; a pair's outputs are the same under zero and under garbage padding, and next to degenerate or other pairs
    at another batch position, with its pair id fixed."""
    rng = np.random.default_rng(99)
    scenes = [f_scene(rng, pair, motion, 400, 0.6, 1.5, 0.5)[:2] for pair in SAME_PAIRS + MIXED_PAIRS
              for motion in ("general", "forward")]
    B = len(scenes)
    p0, p1, cnt = pack(rng, scenes, 512)
    out = run_f(p0, p1, cnt, 1.5, 2048, seed=6)
    again = run_f(p0, p1, cnt, 1.5, 2048, seed=6)
    for x, y in zip(out, again):
        assert np.array_equal(x, y)
    z0, z1 = np.zeros_like(p0), np.zeros_like(p1)
    for b, (a, c) in enumerate(scenes):
        z0[b, :len(a)], z1[b, :len(c)] = a, c
    zero = run_f(z0, z1, cnt, 1.5, 2048, seed=6)
    for x, y in zip(zero, out):
        assert np.array_equal(x, y)
    degen = [(a, c) for _, a, c in f_degenerate_scenes(rng)]
    other = [f_scene(rng, MIXED_PAIRS[0], "sideways", 300, 0.4, 1.5, 1.0)[:2] for _ in range(B)]
    for keep, at in ((0, 5), (3, 0), (B - 1, 2)):
        mixed = [degen[j % len(degen)] if j % 2 else other[j] for j in range(B)]
        mixed[at] = scenes[keep]
        ids = [100 + j for j in range(B)]
        ids[at] = keep
        q0, q1, qc = pack(rng, mixed, 512)
        got = run_f(q0, q1, qc, 1.5, 2048, seed=6, pair_ids=ids)
        for x, y in zip(got, out):
            assert np.array_equal(x[at], y[keep]), (keep, at)
