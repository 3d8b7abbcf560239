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
