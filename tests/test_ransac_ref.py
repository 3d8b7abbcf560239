"""CPU checks of tests/ransac_ref.py, the float64 references test_gpu_ransac_models.py compares the RANSAC kernels with, and of
geometry.recover_pose, the host pose recovery behind evalharness.estimate_pose_gpu."""
import cv2
import numpy as np
import pytest
from scipy.optimize import minimize

from accelerated_features_b200.geometry import recover_pose
from tests import ransac_ref as ref


def random_h(rng):
    A = np.eye(3) + rng.normal(0, 0.2, (3, 3))
    A[2, :2] = rng.uniform(-5e-4, 5e-4, 2)
    A[:2, 2] = rng.uniform(-50, 50, 2)
    return A / A[2, 2]


@pytest.mark.parametrize("seed", range(5))
def test_dlt_refit_exact(seed):
    """On exact data the refit is the true H, whatever the outliers it is told to ignore."""
    rng = np.random.default_rng(seed)
    H = random_h(rng)
    p0 = rng.uniform(0, [640, 480], (200, 2))
    p1 = ref.apply_h(H, p0)
    mask = rng.uniform(size=200) < 0.6
    p1[~mask] = rng.uniform(0, [640, 480], ((~mask).sum(), 2))
    Hr = ref.dlt_refit(p0, p1, mask, ref.hartley(p0), ref.hartley(p1))
    assert Hr[2, 2] == 1.0
    g = np.stack(np.meshgrid(np.linspace(0, 640, 9), np.linspace(0, 480, 9)), -1).reshape(-1, 2)
    assert np.abs(ref.apply_h(Hr, g) - ref.apply_h(H, g)).max() < 1e-10 * 800
    assert ref.transfer_err(Hr, p0[mask], p1[mask]).max() < 1e-9
    # the result does not depend on which similarity normalises the points (only on its conditioning)
    Hs = ref.dlt_refit(p0, p1, mask, (0.0, 0.0, 1.0 / 400), (0.0, 0.0, 1.0 / 400))
    assert np.abs(ref.apply_h(Hs, g) - ref.apply_h(H, g)).max() < 1e-8 * 800


def test_hartley():
    rng = np.random.default_rng(1)
    p = rng.uniform(0, [3840, 2160], (500, 2))
    cx, cy, s = ref.hartley(p)
    q = (p - [cx, cy]) * s
    assert np.abs(q.mean(0)).max() < 1e-12
    assert abs(np.linalg.norm(q, axis=1).mean() - np.sqrt(2)) < 1e-12
    assert ref.hartley(np.full((7, 2), 240.0)) == (240.0, 240.0, 1.0)        # all points identical: scale 1


def test_sampson_exact_and_first_order():
    """Zero on exact correspondences; on perturbed ones it approaches the geometric error (the smallest 4-D move onto
    x1^T E x0 = 0) to first order: the relative difference shrinks with the perturbation."""
    rng = np.random.default_rng(2)
    R, t = ref.rodrigues([0.1, -0.2, 0.05]), np.array([0.6, 0.1, 0.3])
    E = ref.essential_from_pose(R, t)
    X0 = np.stack([rng.uniform(-2, 2, 20), rng.uniform(-1.5, 1.5, 20), rng.uniform(3, 8, 20)], 1)
    X1 = X0 @ R.T + t
    x0, x1 = X0[:, :2] / X0[:, 2:], X1[:, :2] / X1[:, 2:]
    assert ref.sampson(E, x0, x1).max() < 1e-14
    rel = []
    for eps in (1e-2, 1e-3):
        d = rng.normal(0, 1, (20, 4))
        d *= eps / np.linalg.norm(d, axis=1, keepdims=True)
        y0, y1 = x0 + d[:, :2], x1 + d[:, 2:]
        s = ref.sampson(E, y0, y1)
        geo = []
        for i in range(20):
            z = np.concatenate([y0[i], y1[i]])
            con = {"type": "eq", "fun": lambda w: np.array([w[2], w[3], 1.0]) @ E @ np.array([w[0], w[1], 1.0])}
            r = minimize(lambda w: ((w - z) ** 2).sum(), z, constraints=[con], method="SLSQP",
                         options={"ftol": 1e-24, "maxiter": 200})
            geo.append(np.sqrt(((r.x - z) ** 2).sum()))
        geo = np.array(geo)
        assert np.all(s <= eps * (1 + 1e-6))                     # never more than the distance to the exact point
        rel.append(np.abs(s / geo - 1).max())
    assert rel[0] < 0.05 and rel[1] < 0.005 and rel[1] < rel[0] / 5, rel


def test_msac_cost():
    assert ref.msac_cost([0.0, 1.0, 2.0, 10.0], 3.0) == 0 + 1 + 4 + 9


def test_project_essential():
    rng = np.random.default_rng(3)
    for _ in range(10):
        M = rng.normal(size=(3, 3))
        P = ref.project_essential(M)
        assert np.allclose(np.linalg.svd(P, compute_uv=False), [1, 1, 0], atol=1e-12)
        assert np.abs(ref.project_essential(P) - P).max() < 1e-12          # idempotent
        R, t = ref.rodrigues(rng.normal(0, 0.5, 3)), rng.normal(size=3)
        E = ref.essential_from_pose(R, t / np.linalg.norm(t))               # already essential: a fixed point
        assert np.abs(ref.project_essential(E) - E).max() < 1e-12


def test_eight_point_exact():
    rng = np.random.default_rng(4)
    for n in (8, 50):
        R, t = ref.rodrigues(rng.normal(0, 0.3, 3)), rng.normal(size=3)
        X0 = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 8, n)], 1)
        X1 = X0 @ R.T + t
        E = ref.eight_point(X0[:, :2] / X0[:, 2:], X1[:, :2] / X1[:, 2:])
        Et = ref.essential_from_pose(R, t)
        Et /= np.linalg.norm(Et)
        E /= np.linalg.norm(E)
        assert min(np.abs(E - Et).max(), np.abs(E + Et).max()) < 1e-9


def _pose_scene(rng, R, t, n=60):
    """Exact normalised correspondences of n random 3-D points in front of both cameras (X1 = R X0 + t)."""
    X0 = np.zeros((0, 3))
    while len(X0) < n:
        X = np.stack([rng.uniform(-3, 3, 4 * n), rng.uniform(-2, 2, 4 * n), rng.uniform(2, 8, 4 * n)], 1)
        Z1 = (X @ R.T + t)[:, 2]
        X0 = np.concatenate([X0, X[Z1 > 0.5]])[:n]
    X1 = X0 @ R.T + t
    return X0[:, :2] / X0[:, 2:], X1[:, :2] / X1[:, 2:]


POSES = [("sideways", [0.0, 0.05, 0.0], [1.0, 0.0, 0.0]), ("sideways_neg", [0.0, -0.05, 0.0], [-1.0, 0.0, 0.0]),
         ("vertical", [0.03, 0.0, 0.0], [0.0, 1.0, 0.0]), ("forward", [0.0, 0.0, 0.1], [0.0, 0.0, -1.0]),
         ("backward", [0.0, 0.0, -0.1], [0.0, 0.0, 1.0]), ("rot30", [0.0, np.radians(30), 0.0], [-0.8, 0.1, 0.2]),
         ("rot30_oblique", [np.radians(30) / np.sqrt(3)] * 3, [0.5, -0.6, 0.4])]


def test_recover_pose_exact_all_chirality_configurations():
    """recover_pose returns the true (R, t) on exact data, agrees with cv2.recoverPose, and the truth sits in each of the four
    decomposition candidates (R in {U W V^T, U W^T V^T}, t in {+u3, -u3}) for at least one of the scenes: every branch of the
    cheirality vote is exercised."""
    rng = np.random.default_rng(5)
    Wm = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
    slots = set()
    for name, rv, t in POSES:
        R, t = ref.rodrigues(rv), np.asarray(t, np.float64) / np.linalg.norm(t)
        x0, x1 = _pose_scene(rng, R, t)
        for sign in (1.0, -1.0):
            E = sign * ref.essential_from_pose(R, t)
            Rg, tg = recover_pose(E, x0, x1)
            assert np.abs(Rg - R).max() < 1e-9 and np.abs(tg / np.linalg.norm(tg) - t).max() < 1e-9, (name, sign)
            _, Rc, tc, _ = cv2.recoverPose(E, x0, x1, np.eye(3))
            assert np.abs(Rc - R).max() < 1e-6 and np.abs(tc.ravel() - t).max() < 1e-6, (name, sign)
            # which candidate slot the truth occupies, with the same SVD sign convention recover_pose uses
            U, _, Vt = np.linalg.svd(E)
            U = -U if np.linalg.det(U) < 0 else U
            Vt = -Vt if np.linalg.det(Vt) < 0 else Vt
            ri = 0 if np.abs(U @ Wm @ Vt - R).max() < 1e-9 else 1
            ti = 0 if np.abs(U[:, 2] - t).max() < 1e-9 else 1
            slots.add((ri, ti))
    assert slots == {(0, 0), (0, 1), (1, 0), (1, 1)}, slots


# ---------------------------------------------------------------------------------------------------------------------------
# fundamental matrix
# ---------------------------------------------------------------------------------------------------------------------------
# (K0, size0, K1, size1): two cameras with different intrinsics and image sizes, and one shared
F_CAMS = [(ref.intrinsics(700, 330, 235), (640, 480), ref.intrinsics(3000, 1900, 1100), (3840, 2160)),
          (ref.intrinsics(60, 31, 25), (64, 48), ref.intrinsics(2500, 1950, 1070), (3840, 2160)),
          (ref.intrinsics(560, 320, 240), (640, 480), ref.intrinsics(560, 320, 240), (640, 480))]


def f_scene(rng, cam, n):
    K0, s0, K1, s1 = cam
    R, t = ref.rodrigues(rng.normal(0, 0.1, 3)), rng.normal(0, 0.5, 3)
    p0, p1 = ref.two_view_points(rng, K0, K1, s0, s1, R, t, n)
    return p0, p1, ref.fundamental_from_cameras(K0, K1, R, t)


def sign_dist(A, B):
    A, B = A / np.linalg.norm(A), B / np.linalg.norm(B)
    return min(np.abs(A - B).max(), np.abs(A + B).max())


def test_pair_normaliser_and_sampson_scale():
    """The DESIGN claim behind the pixel threshold: with one scale s for both images, the Sampson distance of the normalised
    points under Fn = T1^-T F T0^-1 is exactly s times the pixel one (to float64 rounding), however different the images."""
    rng = np.random.default_rng(6)
    for cam in F_CAMS:
        p0, p1, F = f_scene(rng, cam, 300)
        p1 = p1 + rng.normal(0, 2.0, p1.shape)                   # non-zero distances
        cx0, cy0, cx1, cy1, s = nz = ref.pair_normaliser(p0, p1)
        a, b = (p0 - [cx0, cy0]) * s, (p1 - [cx1, cy1]) * s
        assert np.abs(a.mean(0)).max() < 1e-12 and np.abs(b.mean(0)).max() < 1e-12
        md = np.concatenate([np.linalg.norm(a, axis=1), np.linalg.norm(b, axis=1)]).mean()
        assert abs(md - np.sqrt(2)) < 1e-12
        T0, T1 = ref.pair_norm_matrices(nz)
        Fn = np.linalg.inv(T1).T @ F @ np.linalg.inv(T0)
        d_px, d_n = ref.sampson(F, p0, p1), ref.sampson(Fn, a, b)
        assert np.abs(d_n / (s * d_px) - 1).max() < 1e-9
        assert np.allclose(T1.T @ Fn @ T0, F, rtol=0, atol=1e-12)
    assert ref.pair_normaliser(np.full((9, 2), 5.0), np.full((9, 2), 7.0)) == (5.0, 5.0, 7.0, 7.0, 1.0)


def test_det_cubic_matches_determinant():
    rng = np.random.default_rng(8)
    for _ in range(20):
        A, B = rng.normal(size=(3, 3)), rng.normal(size=(3, 3))
        c = ref.det_cubic(A, B)
        for lam in (-2.0, -0.3, 0.0, 0.7, 3.0):
            assert abs(np.polyval(c, lam) - np.linalg.det(A + lam * B)) < 1e-12 * (1 + abs(lam)) ** 3 * 30


def test_seven_point_exact():
    """On 7 exact correspondences of a non-planar scene, +-F_true is among the candidates; every candidate satisfies the 7
    epipolar constraints, has unit norm and det = 0.  Both the one-root and the three-root case occur."""
    rng = np.random.default_rng(9)
    counts = set()
    for k in range(60):
        p0, p1, F = f_scene(rng, F_CAMS[k % len(F_CAMS)], 7)
        T0, T1 = ref.pair_norm_matrices(ref.pair_normaliser(p0, p1))
        a, b = (ref._h(p0) @ T0.T)[:, :2], (ref._h(p1) @ T1.T)[:, :2]
        Fn_true = np.linalg.inv(T1).T @ F @ np.linalg.inv(T0)
        cands, _ = ref.seven_point(a, b)
        counts.add(len(cands))
        assert 1 <= len(cands) <= 3
        assert min(sign_dist(c, Fn_true) for c in cands) < 1e-8, k
        for c in cands:
            assert abs(np.linalg.norm(c) - 1) < 1e-12
            assert np.abs(ref.epipolar_rows(a, b) @ c.ravel()).max() < 1e-12
            assert abs(np.linalg.det(c)) < 1e-12
    assert counts >= {1, 3}, counts


def test_seven_point_root_at_infinity():
    """When the basis makes det(F1 - F2) = 0, the cubic loses its leading term and F1 - F2 is itself a solution: it is returned
    beside the roots of the remaining quadratic, each singular and in the span."""
    rng = np.random.default_rng(10)
    for _ in range(10):
        Fa = ref.project_rank2(rng.normal(size=(3, 3)))
        F2 = rng.normal(size=(3, 3))
        cands, c = ref.seven_point_from_basis(F2 + Fa, F2)
        assert abs(c[0]) < 1e-12 * np.abs(c).max()
        assert sign_dist(cands[-1], Fa) < 1e-12
        for G in cands:
            assert abs(np.linalg.det(G)) < 1e-10
            r = np.linalg.lstsq(np.stack([Fa.ravel(), F2.ravel()], 1), G.ravel(), rcond=None)[1]
            assert r.size == 0 or r[0] < 1e-20


def test_project_rank2_is_nearest():
    rng = np.random.default_rng(11)
    for _ in range(20):
        M = rng.normal(size=(3, 3))
        P = ref.project_rank2(M)
        s = np.linalg.svd(M, compute_uv=False)
        assert np.linalg.matrix_rank(P, tol=1e-10) == 2 and np.abs(ref.project_rank2(P) - P).max() < 1e-12
        assert abs(np.linalg.norm(M - P) - s[2]) < 1e-12            # Eckart-Young: the distance is the dropped value
        for _ in range(50):                                          # no random rank-2 matrix near M is nearer
            Q = ref.project_rank2(P + rng.normal(0, 0.05, (3, 3)))
            assert np.linalg.norm(M - Q) >= s[2] - 1e-12


def test_f_lo_refit_exact():
    """On exact inliers among far outliers, one refit from a slightly wrong F returns F_true (up to sign), whichever cameras."""
    rng = np.random.default_rng(12)
    for cam in F_CAMS:
        p0, p1, F = f_scene(rng, cam, 400)
        out = rng.uniform(size=400) < 0.4
        W1, H1 = cam[3]
        while True:
            bad = out & (ref.sampson(F, p0, p1) < 30)
            if not bad.any():
                break
            p1[bad] = rng.uniform([0, 0], [W1, H1], (bad.sum(), 2))
        Fp = F + rng.normal(0, 1e-6, (3, 3)) * np.abs(F)
        assert ref.sampson(Fp, p0[~out], p1[~out]).max() < 1.0
        Fr = ref.f_lo_refit(Fp, p0, p1, 3.0)
        assert sign_dist(Fr, F) < 1e-9 and abs(np.linalg.det(Fr)) < 1e-12
        assert ref.sampson(Fr, p0[~out], p1[~out]).max() < 1e-8
