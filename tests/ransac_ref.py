"""Float64 host references of the RANSAC models in csrc/ransac.cu (numpy only; imports neither torch, OpenCV nor the product).

The estimators are stochastic only in which minimal sample wins.  What follows the winner is deterministic, and is restated
here from its formulas so the GPU tests can check it exactly or to float32 rounding:
  * `hartley`: rs_normaliser, the Hartley normalisation of one image's first n points (centroid to the origin, mean distance
    sqrt(2); scale 1 when the mean distance is <= 1e-12).
  * `dlt_refit`: the least-squares refit of ransac_h_final_kernel: the normal equations A^T A of the two DLT rows of every
    inlier in the normalised frames, the eigenvector of the smallest eigenvalue divided by its last entry, de-normalised to
    T1^-1 Hn T0 with H[2,2] = 1.
  * `transfer_err`, `sampson`, `msac_cost`: the errors the kernels classify and score with.
  * `essential_from_pose`, `project_essential`, `eight_point`: the essential-matrix model and its plain 8-point estimate.
  * `pair_normaliser`, `seven_point`, `fundamental_from_cameras`, `project_rank2`, `f_lo_refit`: the fundamental-matrix path
    (rs_pair_normalise, rs_seven_point, one step of rs_local_opt<true>).
"""
from __future__ import annotations

import numpy as np

SQRT2 = np.sqrt(2.0)


def _h(p: np.ndarray) -> np.ndarray:
    p = np.asarray(p, np.float64)
    return np.concatenate([p, np.ones((len(p), 1))], 1)


def hartley(p: np.ndarray):
    """(cx, cy, s) of the (n, 2) points p: centroid, and the scale that makes the mean distance to it sqrt(2)."""
    p = np.asarray(p, np.float64)
    c = p.mean(0)
    md = np.linalg.norm(p - c, axis=1).mean()
    s = SQRT2 / md if md > 1e-12 else 1.0
    return float(c[0]), float(c[1]), float(s)


def norm_matrix(nz) -> np.ndarray:
    """T = [s 0 -s cx; 0 s -s cy; 0 0 1] of a normaliser (cx, cy, s)."""
    cx, cy, s = nz
    return np.array([[s, 0, -s * cx], [0, s, -s * cy], [0, 0, 1.0]])


def dlt_rows(x, y, u, v) -> np.ndarray:
    """The two DLT rows per correspondence (x, y) -> (u, v), laid out as in ransac_h_final_kernel: (2n, 9)."""
    z, o = np.zeros_like(x), np.ones_like(x)
    r0 = np.stack([x, y, o, z, z, z, -u * x, -u * y, -u], 1)
    r1 = np.stack([z, z, z, x, y, o, -v * x, -v * y, -v], 1)
    return np.concatenate([r0, r1], 0)


def dlt_refit(p0: np.ndarray, p1: np.ndarray, mask: np.ndarray, n0, n1) -> np.ndarray:
    """The homography refit of the correspondences p0[mask] -> p1[mask] (pixels) in the frames of the normalisers n0, n1:
    smallest eigenvector of A^T A, divided by h[8], de-normalised to T1^-1 Hn T0 and scaled to H[2,2] = 1."""
    m = np.asarray(mask, bool)
    T0, T1 = norm_matrix(n0), norm_matrix(n1)
    a = _h(np.asarray(p0, np.float64)[m]) @ T0.T
    b = _h(np.asarray(p1, np.float64)[m]) @ T1.T
    A = dlt_rows(a[:, 0], a[:, 1], b[:, 0], b[:, 1])
    w, V = np.linalg.eigh(A.T @ A)
    h = V[:, 0] / V[8, 0]
    H = np.linalg.inv(T1) @ h.reshape(3, 3) @ T0
    return H / H[2, 2]


def apply_h(H: np.ndarray, p: np.ndarray) -> np.ndarray:
    q = _h(p) @ np.asarray(H, np.float64).T
    return q[:, :2] / q[:, 2:]


def transfer_err(H: np.ndarray, p0: np.ndarray, p1: np.ndarray) -> np.ndarray:
    """Forward transfer error |H(p0) - p1| per correspondence."""
    return np.linalg.norm(apply_h(H, p0) - np.asarray(p1, np.float64), axis=1)


def sampson(E: np.ndarray, x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """Sampson distance of each correspondence under x1^T E x0 = 0 (first-order geometric error, in the points' units).  A
    correspondence whose gradient vanishes (denominator <= 1e-20, rs_sampson2's guard) is at infinite distance."""
    E = np.asarray(E, np.float64)
    h0, h1 = _h(x0), _h(x1)
    a, b = h0 @ E.T, h1 @ E                                     # E x0, E^T x1
    e = (h1 * a).sum(1)
    den = a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 1e-20, np.abs(e) / np.sqrt(np.maximum(den, 1e-300)), np.inf)


def msac_cost(err: np.ndarray, thr: float) -> float:
    """MSAC cost: sum of min(err^2, thr^2)."""
    err = np.asarray(err, np.float64)
    return float(np.minimum(err * err, thr * thr).sum())


def skew(t) -> np.ndarray:
    t = np.asarray(t, np.float64)
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def essential_from_pose(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """E = [t]x R, with x1^T E x0 = 0 for X1 = R X0 + t."""
    return skew(t) @ np.asarray(R, np.float64)


def project_essential(E: np.ndarray) -> np.ndarray:
    """The nearest matrix with singular values (1, 1, 0): U diag(1, 1, 0) V^T."""
    U, _, Vt = np.linalg.svd(np.asarray(E, np.float64))
    return U @ np.diag([1.0, 1.0, 0.0]) @ Vt


def eight_point(x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """Plain 8-point estimate from normalised coordinates: the right singular vector of the smallest singular value of the
    epipolar rows (u x, u y, u, v x, v y, v, x, y, 1), projected onto the essential manifold."""
    h0, h1 = _h(x0), _h(x1)
    A = (h1[:, :, None] * h0[:, None, :]).reshape(len(h0), 9)
    _, _, Vt = np.linalg.svd(A)
    return project_essential(Vt[-1].reshape(3, 3))


def rotation_angle_deg(R: np.ndarray) -> float:
    """Angle of a rotation matrix, in degrees."""
    c = (np.trace(np.asarray(R, np.float64)) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))


def angle_between_deg(a: np.ndarray, b: np.ndarray) -> float:
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    c = a @ b / (np.linalg.norm(a) * np.linalg.norm(b))
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))


def rodrigues(rvec) -> np.ndarray:
    """Rotation matrix of an axis-angle vector."""
    r = np.asarray(rvec, np.float64)
    th = np.linalg.norm(r)
    if th < 1e-300:
        return np.eye(3)
    K = skew(r / th)
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


# ---------------------------------------------------------------------------------------------------------------------------
# fundamental matrix
# ---------------------------------------------------------------------------------------------------------------------------
def pair_normaliser(p0: np.ndarray, p1: np.ndarray):
    """rs_pair_normalise: (cx0, cy0, cx1, cy1, s), each image's centroid and ONE scale s that makes the mean distance to the
    centroids sqrt(2) over all 2n points (scale 1 when that distance is <= 1e-12)."""
    p0, p1 = np.asarray(p0, np.float64), np.asarray(p1, np.float64)
    c0, c1 = p0.mean(0), p1.mean(0)
    md = np.concatenate([np.linalg.norm(p0 - c0, axis=1), np.linalg.norm(p1 - c1, axis=1)]).mean()
    s = SQRT2 / md if md > 1e-12 else 1.0
    return float(c0[0]), float(c0[1]), float(c1[0]), float(c1[1]), float(s)


def pair_norm_matrices(nz):
    """(T0, T1) of a pair normaliser: T_i = [s 0 -s cx_i; 0 s -s cy_i; 0 0 1]; F = T1^T Fn T0."""
    cx0, cy0, cx1, cy1, s = nz
    return norm_matrix((cx0, cy0, s)), norm_matrix((cx1, cy1, s))


def epipolar_rows(x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """The rows (u x, u y, u, v x, v y, v, x, y, 1) of x1^T F x0 = 0 (rs_epi_row): (n, 9)."""
    h0, h1 = _h(x0), _h(x1)
    return (h1[:, :, None] * h0[:, None, :]).reshape(len(h0), 9)


def det_cubic(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """Coefficients (c3, c2, c1, c0) of det(A + l B) = c3 l^3 + c2 l^2 + c1 l + c0, exactly from the adjugates:
    c0 = det A, c1 = tr(adj(A) B), c2 = tr(adj(B) A), c3 = det B."""
    def adj(M):
        return np.array([[M[1, 1] * M[2, 2] - M[1, 2] * M[2, 1], M[0, 2] * M[2, 1] - M[0, 1] * M[2, 2], M[0, 1] * M[1, 2] - M[0, 2] * M[1, 1]],
                         [M[1, 2] * M[2, 0] - M[1, 0] * M[2, 2], M[0, 0] * M[2, 2] - M[0, 2] * M[2, 0], M[0, 2] * M[1, 0] - M[0, 0] * M[1, 2]],
                         [M[1, 0] * M[2, 1] - M[1, 1] * M[2, 0], M[0, 1] * M[2, 0] - M[0, 0] * M[2, 1], M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]]])
    return np.array([np.linalg.det(B), np.trace(adj(B) @ A), np.trace(adj(A) @ B), np.linalg.det(A)])


def seven_point(x0: np.ndarray, x1: np.ndarray, lead_tol: float = 1e-12, imag_tol: float = 1e-9):
    """Every fundamental matrix of 7 correspondences, at unit Frobenius norm.  (F1, F2) are the last two right singular vectors
    of the 7 x 9 epipolar rows; det(l F1 + (1 - l) F2) = det(F2 + l (F1 - F2)) is a cubic with exact coefficients (det_cubic),
    and each real root (imaginary part <= imag_tol of its modulus, Newton-polished) gives one candidate.  When the leading
    coefficient vanishes (|c3| <= lead_tol max|c|) the root at infinity, F1 - F2, is a candidate too.
    Returns (candidates (k, 3, 3), cubic coefficients (c3, c2, c1, c0))."""
    _, _, Vt = np.linalg.svd(epipolar_rows(x0, x1))
    return seven_point_from_basis(Vt[-2].reshape(3, 3), Vt[-1].reshape(3, 3), lead_tol, imag_tol)


def seven_point_from_basis(F1: np.ndarray, F2: np.ndarray, lead_tol: float = 1e-12, imag_tol: float = 1e-9):
    """seven_point's candidates l F1 + (1 - l) F2 (and F1 - F2) from a given null-space basis."""
    c = det_cubic(F2, F1 - F2)
    cm = np.abs(c).max()
    out = []
    lead = abs(c[0]) <= lead_tol * cm
    roots = np.roots(c[1:] if lead else c)
    for r in roots:
        if abs(r.imag) > imag_tol * max(1.0, abs(r)):
            continue
        lam = r.real
        for _ in range(3):
            f, df = np.polyval(c, lam), np.polyval(np.polyder(c), lam)
            if df != 0:
                lam -= f / df
        out.append(lam * F1 + (1 - lam) * F2)
    if lead:
        out.append(F1 - F2)
    out = [F / np.linalg.norm(F) for F in out]
    return np.array(out).reshape(-1, 3, 3), c


def fundamental_from_cameras(K0: np.ndarray, K1: np.ndarray, R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """F = K1^-T [t]x R K0^-1 (unit Frobenius norm), x1^T F x0 = 0 in pixels for X1 = R X0 + t."""
    F = np.linalg.inv(K1).T @ essential_from_pose(R, t) @ np.linalg.inv(K0)
    return F / np.linalg.norm(F)


def project_rank2(F: np.ndarray) -> np.ndarray:
    """The nearest rank-2 matrix in the Frobenius norm: the SVD without its smallest singular value."""
    U, s, Vt = np.linalg.svd(np.asarray(F, np.float64))
    return U @ np.diag([s[0], s[1], 0.0]) @ Vt


def f_lo_refit(F: np.ndarray, p0: np.ndarray, p1: np.ndarray, thr: float) -> np.ndarray:
    """One refit of rs_local_opt<true>, in the pair's normalised frame (pair_normaliser of all the points): the points whose
    Sampson distance under Fn = T1^-T F T0^-1 is below thr * s, each epipolar row weighted by 1 / (its Sampson denominator
    under Fn), the smallest eigenvector of the weighted normal matrix, projected to rank 2, de-normalised to T1^T Fn T0 and
    scaled to unit Frobenius norm."""
    p0, p1 = np.asarray(p0, np.float64), np.asarray(p1, np.float64)
    nz = pair_normaliser(p0, p1)
    T0, T1 = pair_norm_matrices(nz)
    Fn = np.linalg.inv(T1).T @ np.asarray(F, np.float64) @ np.linalg.inv(T0)
    a, b = (_h(p0) @ T0.T)[:, :2], (_h(p1) @ T1.T)[:, :2]
    ga, gb = _h(a) @ Fn.T, _h(b) @ Fn
    den = ga[:, 0] ** 2 + ga[:, 1] ** 2 + gb[:, 0] ** 2 + gb[:, 1] ** 2
    keep = sampson(Fn, a, b) < thr * nz[4]
    A = epipolar_rows(a[keep], b[keep])
    w, V = np.linalg.eigh((A / den[keep, None]).T @ A)
    Fr = T1.T @ project_rank2(V[:, 0].reshape(3, 3)) @ T0
    return Fr / np.linalg.norm(Fr)


def intrinsics(f: float, cx: float, cy: float) -> np.ndarray:
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1.0]])


def two_view_points(rng, K0, K1, size0, size1, R, t, n, depth=(2.0, 8.0)):
    """n exact (float64) pixel correspondences of random 3-D points: uniform pixels of the W0 x H0 image 0 at depths `depth`,
    kept where they lie in front of camera 1 (X1 = R X0 + t) and inside its W1 x H1 image."""
    K0i = np.linalg.inv(K0)
    p0, p1 = np.zeros((0, 2)), np.zeros((0, 2))
    while len(p0) < n:
        m = 8 * n + 64
        px = rng.uniform([0, 0], size0, (m, 2))
        X = (_h(px) @ K0i.T) * rng.uniform(*depth, (m, 1))
        X1 = X @ np.asarray(R, np.float64).T + t
        q = X1 @ np.asarray(K1, np.float64).T
        with np.errstate(divide="ignore", invalid="ignore"):
            q = q[:, :2] / q[:, 2:]
        ok = (X1[:, 2] > 0.1) & np.all((q >= 0) & (q <= size1), axis=1)
        p0, p1 = np.concatenate([p0, px[ok]])[:n], np.concatenate([p1, q[ok]])[:n]
    return p0, p1
