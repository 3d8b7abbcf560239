"""Float64 references for the calibrated relative pose (geometry.estimate_relative_pose_batch, csrc/ransac.cu RsEssential5 and
ransac_pose_kernel), formulated independently of the device:

- the five-point problem by the action matrix (Stewenius, Engels, Nister 2006, "Recent developments on direct relative
  orientation"): the ten cubic constraints over a graded monomial order, the 10 x 10 matrix of multiplication by x on the
  quotient basis, and numpy.linalg.eig -- where the device eliminates towards Nister's degree-10 polynomial and isolates its
  real roots with a Sturm sequence;
- cheirality by linear (DLT) triangulation of each point, a depth > 0 test in both cameras -- where the device (and
  geometry.recover_pose) solve a 2 x 2 least-squares system for the two depths.
"""
from __future__ import annotations

import itertools

import numpy as np

from tests.ransac_ref import angle_between_deg, essential_from_pose, rodrigues, rotation_angle_deg, skew  # noqa: F401

# the ten cubic monomials, then the quotient basis (exponents of x, y, z; w = 1)
CUBICS = [(3, 0, 0), (2, 1, 0), (2, 0, 1), (1, 2, 0), (1, 1, 1), (1, 0, 2), (0, 3, 0), (0, 2, 1), (0, 1, 2), (0, 0, 3)]
BASIS = [(2, 0, 0), (1, 1, 0), (1, 0, 1), (0, 2, 0), (0, 1, 1), (0, 0, 2), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
MONOS = CUBICS + BASIS
_COL = {m: i for i, m in enumerate(MONOS)}


def epipolar_rows(x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """Rows of x1^T E x0 = 0 over E's entries (row-major)."""
    h0 = np.concatenate([x0, np.ones((len(x0), 1))], 1)
    h1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    return np.einsum("ni,nj->nij", h1, h0).reshape(len(x0), 9)


def null_basis(x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """(4, 9): an orthonormal basis of the null space of the five epipolar rows (SVD)."""
    _, _, vt = np.linalg.svd(epipolar_rows(x0, x1), full_matrices=True)
    return vt[5:]


def _pmul(a: dict, b: dict) -> dict:
    out: dict = {}
    for (ea, ca), (eb, cb) in itertools.product(a.items(), b.items()):
        e = (ea[0] + eb[0], ea[1] + eb[1], ea[2] + eb[2])
        out[e] = out.get(e, 0.0) + ca * cb
    return out


def _padd(*ps, scale=None) -> dict:
    out: dict = {}
    for i, p in enumerate(ps):
        s = 1.0 if scale is None else scale[i]
        for e, c in p.items():
            out[e] = out.get(e, 0.0) + s * c
    return out


def constraint_matrix(N: np.ndarray) -> np.ndarray:
    """(10, 20): det(E) = 0 and 2 E E^T E - tr(E E^T) E = 0 for E = x N0 + y N1 + z N2 + N3, over MONOS."""
    E = [[{(1, 0, 0): N[0, 3 * i + j], (0, 1, 0): N[1, 3 * i + j], (0, 0, 1): N[2, 3 * i + j], (0, 0, 0): N[3, 3 * i + j]}
          for j in range(3)] for i in range(3)]
    rows = []
    det = {}
    for p in itertools.permutations(range(3)):       # Leibniz
        sign = np.linalg.det(np.eye(3)[list(p)])
        det = _padd(det, _pmul(_pmul(E[0][p[0]], E[1][p[1]]), E[2][p[2]]), scale=[1.0, sign])
    rows.append(det)
    EEt = [[_padd(*[_pmul(E[i][k], E[j][k]) for k in range(3)]) for j in range(3)] for i in range(3)]
    tr = _padd(EEt[0][0], EEt[1][1], EEt[2][2])
    for i in range(3):
        for j in range(3):
            rows.append(_padd(*[_pmul(EEt[i][k], E[k][j]) for k in range(3)], _pmul(tr, E[i][j]), scale=[2.0, 2.0, 2.0, -1.0]))
    A = np.zeros((10, 20))
    for r, p in enumerate(rows):
        for e, c in p.items():
            A[r, _COL[e]] += c
    return A


def five_point_roots(N: np.ndarray):
    """Every solution (x, y, z) of the constraints of N, complex: (eigenvalues, (10, 3) complex solutions)."""
    A = constraint_matrix(N)
    G = np.linalg.solve(A[:, :10], A[:, 10:])        # cubic_i = -G[i] . BASIS
    M = np.zeros((10, 10))
    for i, b in enumerate(BASIS):
        xb = (b[0] + 1, b[1], b[2])
        if xb in _COL and _COL[xb] < 10:
            M[i] = -G[_COL[xb]]
        else:
            M[i, BASIS.index(xb)] = 1.0
    w, V = np.linalg.eig(M)
    sol = V[6:9].T / V[9][:, None]
    return w, sol


def five_point(x0: np.ndarray, x1: np.ndarray, imag_tol: float = 1e-8):
    """Candidates E (k, 3, 3), unit Frobenius norm, of a 5-point sample: the solutions whose |imaginary part| is below
    imag_tol, relative to 1 + |root|.  Also returns the eigenvalues (the x of every solution, complex)."""
    N = null_basis(x0, x1)
    w, sol = five_point_roots(N)
    out = []
    for k in range(10):
        if np.all(np.abs(sol[k].imag) <= imag_tol * (1.0 + np.abs(sol[k]))):
            x, y, z = sol[k].real
            E = (x * N[0] + y * N[1] + z * N[2] + N[3]).reshape(3, 3)
            out.append(E / np.linalg.norm(E))
    return np.array(out).reshape(-1, 3, 3), w


def essential_residuals(E: np.ndarray):
    """(|det E|, max |2 E E^T E - tr(E E^T) E|) of a unit-norm E."""
    return abs(np.linalg.det(E)), np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max()


def sampson(E: np.ndarray, x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """Sampson distance (not squared) of normalised correspondences under x1^T E x0 = 0."""
    h0 = np.concatenate([x0, np.ones((len(x0), 1))], 1)
    h1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    Ex0 = h0 @ E.T
    Etx1 = h1 @ E
    e = np.sum(h1 * Ex0, 1)
    return np.abs(e) / np.sqrt(Ex0[:, 0] ** 2 + Ex0[:, 1] ** 2 + Etx1[:, 0] ** 2 + Etx1[:, 1] ** 2)


def decompositions(E: np.ndarray):
    """The four (R, t) with [t]x R ~ E: R in {U W V^T, U W^T V^T} with det U = det V = +1, t = +-U[:, 2] (unit)."""
    U, _, Vt = np.linalg.svd(E)
    U = U * np.sign(np.linalg.det(U))
    Vt = Vt * np.sign(np.linalg.det(Vt))
    W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    return [(R, s * U[:, 2]) for R in (U @ W @ Vt, U @ W.T @ Vt) for s in (1.0, -1.0)]


def triangulate_depths(R: np.ndarray, t: np.ndarray, x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """(n, 2) depths of each point in camera 0 (P0 = [I | 0]) and camera 1 (P1 = [R | t]) by linear DLT triangulation."""
    P0 = np.hstack([np.eye(3), np.zeros((3, 1))])
    P1 = np.hstack([R, t.reshape(3, 1)])
    out = np.empty((len(x0), 2))
    for i, (a, b) in enumerate(zip(x0, x1)):
        A = np.stack([a[0] * P0[2] - P0[0], a[1] * P0[2] - P0[1], b[0] * P1[2] - P1[0], b[1] * P1[2] - P1[1]])
        X = np.linalg.svd(A)[2][-1]
        X = X[:3] / X[3] if abs(X[3]) > 1e-300 else X[:3] * 1e300
        out[i] = X[2], (R @ X + t)[2]
    return out


def cheirality(E: np.ndarray, x0: np.ndarray, x1: np.ndarray):
    """(R, t, counts): the decomposition with the most points in front of both cameras (the first on a tie) and the four
    counts, in decompositions()' order."""
    cands = decompositions(E)
    counts = [int(np.sum(np.all(triangulate_depths(R, t, x0, x1) > 0, 1))) for R, t in cands]
    b = int(np.argmax(counts))
    return cands[b][0], cands[b][1], counts


def pose_clean(x0: np.ndarray, x1: np.ndarray, rng, samples: int = 8):
    """Relative pose of a scene without outliers: the five-point candidate of a few random samples with the smallest
    largest Sampson error over all points, then cheirality.  (E, R, t)."""
    best, bestE = np.inf, None
    for _ in range(samples):
        idx = rng.choice(len(x0), 5, replace=False)
        for E in five_point(x0[idx], x1[idx])[0]:
            err = sampson(E, x0, x1).max()
            if err < best:
                best, bestE = err, E
    R, t, _ = cheirality(bestE, x0, x1)
    return bestE, R, t


def rotation_error_deg(Ra: np.ndarray, Rb: np.ndarray) -> float:
    """Angle between two rotations from the chord |Ra - Rb|_F = 2 sqrt(2) sin(angle / 2): unlike arccos((tr - 1) / 2), it
    resolves small angles of fp32 matrices (arccos reads 6e-8 of trace rounding as ~0.02 degrees)."""
    d = np.linalg.norm(np.asarray(Ra, np.float64) - np.asarray(Rb, np.float64))
    return float(np.degrees(2.0 * np.arcsin(min(1.0, d / (2.0 * np.sqrt(2.0))))))


def intrinsics4(K: np.ndarray) -> np.ndarray:
    return np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])


def normalise(p: np.ndarray, K: np.ndarray) -> np.ndarray:
    """Pixels -> K^-1 coordinates (skew-free K)."""
    return (p - K[[0, 1], [2, 2]][None]) / K[[0, 1], [0, 1]][None]


def random_pose(rng, rot_deg=(5.0, 30.0), baseline=1.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    R = rodrigues(axis * np.deg2rad(rng.uniform(*rot_deg)))
    t = rng.normal(size=3)
    return R, baseline * t / np.linalg.norm(t)


def calibrated_scene(rng, n: int, K0: np.ndarray, K1: np.ndarray, R: np.ndarray, t: np.ndarray, size=(1024, 768),
                     inlier_frac: float = 1.0, noise_px: float = 0.0, depth=(4.0, 12.0), planar: bool = False):
    """Pixel correspondences of n points: the first round(inlier_frac * n) are projections of random points in front of both
    cameras (a plane when `planar`), with Gaussian noise of noise_px; the rest are uniform in the images.  The inliers are then
    shuffled among the outliers.  Returns (p0, p1, is_inlier)."""
    n_in = int(round(inlier_frac * n))
    pts = []
    while len(pts) < n_in:
        m = 4 * n_in + 16
        u = rng.uniform(0, size[0], m)
        v = rng.uniform(0, size[1], m)
        z = rng.uniform(*depth, m)
        X = np.linalg.solve(K0, np.stack([u * z, v * z, z]))
        if planar:
            nrm = np.array([0.1, 0.2, 1.0]) / np.linalg.norm([0.1, 0.2, 1.0])
            d0 = 0.5 * (depth[0] + depth[1])
            X = X * (d0 / (nrm @ X))[None]
        Y = R @ X + t[:, None]
        uv1 = K1 @ Y
        uv1 = uv1[:2] / uv1[2]
        ok = (X[2] > 0) & (Y[2] > 0.1) & (uv1[0] >= 0) & (uv1[0] < size[0]) & (uv1[1] >= 0) & (uv1[1] < size[1])
        pts += list(zip(np.stack([u, v], 1)[ok] if not planar else (K0 @ X)[:2, ok].T / (K0 @ X)[2, ok, None], uv1.T[ok]))
    pts = pts[:n_in]
    p0 = np.array([a for a, _ in pts]).reshape(-1, 2) + rng.normal(scale=noise_px, size=(n_in, 2)) * (noise_px > 0)
    p1 = np.array([b for _, b in pts]).reshape(-1, 2) + rng.normal(scale=noise_px, size=(n_in, 2)) * (noise_px > 0)
    o0 = np.stack([rng.uniform(0, size[0], n - n_in), rng.uniform(0, size[1], n - n_in)], 1)
    o1 = np.stack([rng.uniform(0, size[0], n - n_in), rng.uniform(0, size[1], n - n_in)], 1)
    p0, p1 = np.concatenate([p0, o0]), np.concatenate([p1, o1])
    inl = np.arange(n) < n_in
    perm = rng.permutation(n)
    return p0[perm], p1[perm], inl[perm]
