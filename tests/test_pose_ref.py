"""The float64 relative-pose reference (tests/pose_ref.py) on its own, without a GPU: the five-point action-matrix solver
recovers E exactly from noise-free minimal samples, and the reference pipeline agrees with cv2.findEssentialMat +
cv2.recoverPose on clean scenes.  Every bound is at least 5x the reference's own error on the case."""
import numpy as np
import pytest

from tests import pose_ref as P

K0 = np.array([[980.0, 0.0, 500.0], [0.0, 1010.0, 370.0], [0.0, 0.0, 1.0]])
K1 = np.array([[720.0, 0.0, 330.0], [0.0, 700.0, 250.0], [0.0, 0.0, 1.0]])


def _unit(E):
    return E / np.linalg.norm(E)


def _dist_up_to_sign(A, B):
    return min(np.abs(A - B).max(), np.abs(A + B).max())


@pytest.mark.parametrize("planar", [False, True])
def test_five_point_recovers_exact_e(planar):
    """Noise-free minimal samples of known (R, t): one candidate is the true E to rounding, every real candidate satisfies
    the essential constraints, and the candidate count is at most 10."""
    rng = np.random.default_rng(11 + planar)
    errs, res = [], []
    for _ in range(200):
        R, t = P.random_pose(rng)
        p0, p1, _ = P.calibrated_scene(rng, 5, K0, K1, R, t, planar=planar)
        Es, w = P.five_point(P.normalise(p0, K0), P.normalise(p1, K1))
        assert 1 <= len(Es) <= 10 and len(w) == 10
        true = _unit(P.essential_from_pose(R, t))
        errs.append(min(_dist_up_to_sign(E, true) for E in Es))
        res += [max(P.essential_residuals(E)) for E in Es]
    # measured: worst error 3.8e-7 and worst residual 5.7e-8 (clustered roots); the bounds are > 10x those
    print(f"five-point exact recovery: worst |E - E_true| {max(errs):.2e}, worst residual {max(res):.2e}")
    assert max(errs) < 5e-6
    assert max(res) < 1e-5


def test_decompositions_and_cheirality_pick_the_true_pose():
    rng = np.random.default_rng(5)
    for _ in range(50):
        R, t = P.random_pose(rng)
        p0, p1, _ = P.calibrated_scene(rng, 64, K0, K1, R, t)
        x0, x1 = P.normalise(p0, K0), P.normalise(p1, K1)
        Rb, tb, counts = P.cheirality(P.essential_from_pose(R, t), x0, x1)
        assert max(counts) == 64 and sorted(counts)[-2] < 64
        assert np.abs(Rb - R).max() < 1e-9
        assert np.abs(tb - t).max() < 1e-9


def test_reference_agrees_with_opencv_on_clean_scenes():
    """Noise-free scenes without outliers, K0 != K1: the reference's pose and cv2's both match the ground truth, and each
    other, within 5x the larger of their measured errors.  The floor, 1e-5 degrees, is 5x the resolution of an angle read
    through arccos in float64 (~2e-6 degrees near 0)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(8)
    ours, theirs = [], []
    for _ in range(40):
        R, t = P.random_pose(rng)
        p0, p1, _ = P.calibrated_scene(rng, 200, K0, K1, R, t)
        x0, x1 = P.normalise(p0, K0), P.normalise(p1, K1)
        _, Rr, tr = P.pose_clean(x0, x1, rng)
        E, mask = cv2.findEssentialMat(x0, x1, np.eye(3), method=cv2.RANSAC, prob=0.999999, threshold=1e-6)
        _, Rc, tc, _ = cv2.recoverPose(E[:3], x0, x1, np.eye(3), mask=mask)
        ours.append((P.rotation_angle_deg(Rr.T @ R), P.angle_between_deg(tr, t)))
        theirs.append((P.rotation_angle_deg(Rc.T @ R), P.angle_between_deg(tc.ravel(), t)))
    ours, theirs = np.array(ours), np.array(theirs)
    print(f"reference worst (R, t) error {ours.max(0)} deg, cv2 worst {theirs.max(0)} deg")
    bound = 5 * max(ours.max(), theirs.max(), 2e-6)
    assert ours.max() < bound and theirs.max() < bound
    assert ours.max() < 1e-5          # the reference alone: its measured worst is the arccos resolution
