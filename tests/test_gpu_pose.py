"""The calibrated relative pose on the GPU (geometry.estimate_relative_pose_batch, csrc/ransac.cu RsEssential5 +
ransac_pose_kernel) against the float64 reference of tests/pose_ref.py, ground truth and cv2: the five-point hook, exact
recovery, noisy scenes, the on-device cheirality, edge cases, and the pair-list and eval-harness entry points."""
import numpy as np
import pytest
import torch

from accelerated_features_b200 import _lib
from accelerated_features_b200.geometry import estimate_relative_pose, estimate_relative_pose_batch, recover_pose
from tests import pose_ref as P

pytestmark = pytest.mark.gpu

KA = np.array([[1000.0, 0.0, 512.0], [0.0, 1000.0, 384.0], [0.0, 0.0, 1.0]])
KB = np.array([[820.0, 0.0, 300.0], [0.0, 790.0, 260.0], [0.0, 0.0, 1.0]])


def run_five_point(samples: np.ndarray):
    """xfeat_debug_five_point on (S, 5, 4) float32 rows -> (candidates (S, 10, 3, 3), counts (S))."""
    lib = _lib.load()
    s = torch.from_numpy(np.ascontiguousarray(samples, np.float32)).cuda()
    E = torch.empty((len(samples), 10, 9), dtype=torch.float32, device="cuda")
    c = torch.empty((len(samples),), dtype=torch.int32, device="cuda")
    _lib.check(lib.xfeat_debug_five_point(s.data_ptr(), len(samples), E.data_ptr(), c.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), "xfeat_debug_five_point")
    return E.cpu().numpy().reshape(-1, 10, 3, 3), c.cpu().numpy()


def _up_to_sign(A, B):
    return min(np.abs(A - B).max(), np.abs(A + B).max())


def _minimal_samples(rng, kind, count):
    out, truth = [], []
    for _ in range(count):
        R, t = P.random_pose(rng, baseline=0.1 if kind == "small_baseline" else 1.0)
        p0, p1, _ = P.calibrated_scene(rng, 5, KA, KB, R, t, planar=kind == "planar")
        x0, x1 = P.normalise(p0, KA), P.normalise(p1, KB)
        out.append(np.concatenate([x0, x1], 1).astype(np.float32))
        truth.append(P.essential_from_pose(R, t) / np.linalg.norm(P.essential_from_pose(R, t)))
    return np.array(out), truth


@pytest.mark.parametrize("kind", ["general", "planar", "small_baseline"])
def test_five_point_hook_against_reference(kind):
    """Every real root of the action-matrix reference (|Im| <= 1e-8 (1 + |root|); the reference's residuals on its real roots
    are ~1e-8, so complex pairs it calls real are at least that well resolved) is a device candidate up to sign, within 1e-3
    (fp32 output of unit-norm E, plus the conditioning of the degree-10 polynomial), and every device candidate satisfies the
    essential constraints within 1e-3 (measured 3e-6).  Planar and small-baseline samples put roots close together on the z axis, where the Sturm
    isolation on the expanded polynomial loses roots the eigen-solver keeps: there the share of reference roots found and of
    samples whose true E is found are bounded from below instead (measured on the H100: 97 % and 97 % of 400 samples)."""
    rng = np.random.default_rng({"general": 1, "planar": 2, "small_baseline": 3}[kind])
    samples, truth = _minimal_samples(rng, kind, 400)
    Ed, cnt = run_five_point(samples)
    assert np.all(np.isfinite(Ed)) and cnt.min() >= 0 and cnt.max() <= 10
    assert np.all(Ed[np.arange(10)[None, :] >= cnt[:, None]] == 0)
    n_ref = n_found = true_found = 0
    worst_match = worst_res = 0.0
    for s in range(len(samples)):
        x = samples[s].astype(np.float64)
        Er, _ = P.five_point(x[:, :2], x[:, 2:])
        D = Ed[s, :cnt[s]].astype(np.float64)
        for E in Er:
            d = min([_up_to_sign(E, c) for c in D] or [np.inf])
            n_ref += 1
            if d < 1e-3:
                n_found += 1
                worst_match = max(worst_match, d)
        true_found += min([_up_to_sign(truth[s], c) for c in D] or [np.inf]) < 1e-3
        worst_res = max([worst_res] + [max(P.essential_residuals(c / np.linalg.norm(c))) for c in D])
    print(f"five-point {kind}: {n_found}/{n_ref} reference roots found (worst {worst_match:.1e}), true E in "
          f"{true_found}/{len(samples)}, worst device residual {worst_res:.1e}, mean count {cnt.mean():.2f}")
    if kind == "general":
        assert n_found == n_ref and true_found == len(samples)
        assert worst_res < 1e-3
    else:
        assert n_found >= 0.95 * n_ref and true_found >= 0.95 * len(samples)


def test_five_point_degenerate_samples():
    rng = np.random.default_rng(4)
    good, _ = _minimal_samples(rng, "general", 3)
    same = np.repeat(good[0, :1], 5, 0)                       # five identical points
    rep = good[1].copy()
    rep[3] = rep[1]                                           # one repeated point
    zero = np.zeros((5, 4), np.float32)
    Ed, cnt = run_five_point(np.stack([same, rep, zero]))
    assert cnt.tolist() == [0, 0, 0]
    assert np.all(Ed == 0)


def _batch(scenes, counts_as=None):
    n_max = max(len(s[0]) for s in scenes)
    B = len(scenes)
    p0 = np.zeros((B, n_max, 2), np.float32)
    p1 = np.zeros((B, n_max, 2), np.float32)
    for b, (a, c, *_) in enumerate(scenes):
        p0[b, :len(a)], p1[b, :len(a)] = a, c
    cnt = np.array([len(s[0]) for s in scenes], np.int32) if counts_as is None else np.asarray(counts_as, np.int32)
    return torch.from_numpy(p0).cuda(), torch.from_numpy(p1).cuda(), torch.from_numpy(cnt).cuda()


def _scene(rng, n, frac, noise, K0=KA, K1=KB, **kw):
    R, t = P.random_pose(rng)
    p0, p1, inl = P.calibrated_scene(rng, n, K0, K1, R, t, inlier_frac=frac, noise_px=noise, **kw)
    return p0, p1, R, t, inl


@pytest.mark.parametrize("frac", [1.0, 0.5])
def test_exact_recovery(frac):
    """Noise-free scenes, K0 != K1, at thr 0.05 px (noise-free inliers sit at the fp32 rounding of their pixels, ~1e-4 px; a
    wider band would let outliers near their epipolar lines bias the refit).  Bounds, 2e-4 degrees for R and 5e-4 degrees for t
    up to sign: fp32 pixels carry ~6e-5 px, 6e-8 rad at f ~ 900; E, R and t are stored in fp32 (6e-8 relative); the direction
    of t, a null vector of E, amplifies E's error by the inverse gap of its singular values; together ~1e-5 degrees."""
    rng = np.random.default_rng(21 + int(frac * 10))
    scenes = [_scene(rng, 400, frac, 0.0) for _ in range(32)]
    p0, p1, cnt = _batch(scenes)
    K0 = np.repeat(KA[None], 32, 0)
    K1 = np.repeat(KB[None], 32, 0)
    E, R, t, mask, n_inl, n_front = estimate_relative_pose_batch(p0, p1, K0, K1, cnt, thr=0.05)
    R, t, mask, n_inl = R.cpu().numpy(), t.cpu().numpy(), mask.cpu().numpy(), n_inl.cpu().numpy()
    er = [P.rotation_error_deg(R[b], s[2]) for b, s in enumerate(scenes)]
    et = [P.angle_between_deg(t[b], s[3]) for b, s in enumerate(scenes)]
    print(f"exact recovery, {frac:.0%} inliers: worst rotation {max(er):.2e} deg, worst translation {max(et):.2e} deg")
    assert max(er) < 2e-4 and max(et) < 5e-4
    for b, s in enumerate(scenes):
        assert mask[b, :400][s[4]].all()                    # every true inlier (an outlier may fall near its epipolar line)
        assert n_inl[b] >= s[4].sum()


def test_noisy_scenes_against_ground_truth_and_opencv():
    """sigma = 0.5 px at f ~ 1000, 256-4096 correspondences, 30-80 % inliers.  The device and cv2's 5-point RANSAC
    (estimate_pose_opencv's call) on the same points: the device's median and 90th-percentile errors may exceed cv2's by at
    most 1.5x + 0.05 degrees, and its worst stays below 2 degrees."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(31)
    scenes, Ks0, Ks1 = [], [], []
    for b in range(48):
        n = int(rng.integers(256, 4097))
        K0 = KA if b % 2 else KB
        scenes.append(_scene(rng, n, rng.uniform(0.3, 0.8), 0.5, K0=K0, K1=KA))
        Ks0.append(K0)
        Ks1.append(KA)
    p0, p1, cnt = _batch(scenes)
    _, R, t, _, n_inl, _ = estimate_relative_pose_batch(p0, p1, np.array(Ks0), np.array(Ks1), cnt, thr=1.0)
    R, t = R.cpu().numpy().astype(np.float64), t.cpu().numpy().astype(np.float64)
    dev, ocv = [], []
    for b, s in enumerate(scenes):
        dev.append(max(P.rotation_angle_deg(R[b].T @ s[2]), min(P.angle_between_deg(t[b], s[3]), 180 - P.angle_between_deg(t[b], s[3]))))
        x0, x1 = P.normalise(s[0], Ks0[b]), P.normalise(s[1], Ks1[b])
        f = 0.25 * (Ks0[b][0, 0] + Ks0[b][1, 1] + Ks1[b][0, 0] + Ks1[b][1, 1])
        E, m = cv2.findEssentialMat(x0, x1, np.eye(3), threshold=1.0 / f, prob=0.99999, method=cv2.RANSAC)
        _, Rc, tc, _ = cv2.recoverPose(E[:3], x0, x1, np.eye(3), mask=m)
        ocv.append(max(P.rotation_angle_deg(Rc.T @ s[2]), min(P.angle_between_deg(tc.ravel(), s[3]),
                                                            180 - P.angle_between_deg(tc.ravel(), s[3]))))
    dev, ocv = np.array(dev), np.array(ocv)
    q = [50, 90, 100]
    print(f"noisy scenes: device max(R, t) error percentiles {q}: {np.percentile(dev, q)} deg; cv2: {np.percentile(ocv, q)} deg")
    for a, b in zip(np.percentile(dev, [50, 90]), np.percentile(ocv, [50, 90])):
        assert a <= 1.5 * b + 0.05
    assert dev.max() < 2.0


def test_cheirality_matches_recover_pose():
    """The device's own E and inliers through geometry.recover_pose: the same (R, t) within fp32 rounding, except where the
    best two candidates' counts differ by no more than the points whose depth is within eps of zero."""
    rng = np.random.default_rng(41)
    scenes = [_scene(rng, int(rng.integers(200, 1500)), 0.6, 0.5) for _ in range(40)]
    p0, p1, cnt = _batch(scenes)
    K0, K1 = np.repeat(KA[None], 40, 0), np.repeat(KB[None], 40, 0)
    E, R, t, mask, n_inl, n_front = (x.cpu().numpy() for x in estimate_relative_pose_batch(p0, p1, K0, K1, cnt, thr=1.0))
    exceptions = 0
    for b, s in enumerate(scenes):
        m = mask[b, :len(s[0])]
        x0 = P.normalise(s[0].astype(np.float32).astype(np.float64), KA)[m]
        x1 = P.normalise(s[1].astype(np.float32).astype(np.float64), KB)[m]
        Rh, th = recover_pose(E[b].astype(np.float64), x0, x1)
        if np.abs(Rh - R[b]).max() < 1e-5 and np.abs(th - t[b]).max() < 1e-5:
            continue
        counts, near = [], 0
        for Rc, tc in P.decompositions(E[b].astype(np.float64)):
            z = P.triangulate_depths(Rc, tc, x0, x1)
            counts.append(int(np.all(z > 0, 1).sum()))
            near = max(near, int((np.abs(z) < 1e-6).any(1).sum()))
        top = sorted(counts)[-2:]
        assert top[1] - top[0] <= near, (b, counts, near)
        exceptions += 1
    print(f"cheirality: {exceptions} of {len(scenes)} pairs differ from recover_pose (near-ties)")
    assert np.all(n_front <= n_inl) and np.all(n_front[n_inl > 0] > 0)


def test_edge_counts_overflow_and_mixed_cameras():
    rng = np.random.default_rng(51)
    base = _scene(rng, 8192, 0.6, 0.5)                        # cameras KA -> KB
    other = _scene(rng, 300, 0.6, 0.5, K0=KB, K1=KA)          # the last pair: cameras KB -> KA
    counts = [0, 4, 5, 8192, _lib.N_OVERFLOW, 300]
    p0, p1, cnt = _batch([base[:2]] * 5 + [other[:2]], counts_as=counts)
    K0 = np.array([P.intrinsics4(KA)] * 5 + [P.intrinsics4(KB)])
    K1 = np.array([P.intrinsics4(KB)] * 5 + [P.intrinsics4(KA)])
    E, R, t, mask, n_inl, n_front = (x.cpu().numpy() for x in estimate_relative_pose_batch(p0, p1, K0, K1, cnt, thr=1.0))
    for b in (0, 1, 4):                                       # no model: zero E, R = I, t = 0, counts passed through
        assert np.all(E[b] == 0) and np.array_equal(R[b], np.eye(3, dtype=np.float32)) and np.all(t[b] == 0)
        assert not mask[b].any() and n_front[b] == 0
    assert n_inl[0] == 0 and n_inl[1] == 0 and n_inl[4] == _lib.N_OVERFLOW
    assert np.all(np.isfinite(E[2])) and np.all(np.isfinite(R[2])) and not mask[2, 5:].any()
    assert n_inl[3] > 0.5 * 8192 and P.rotation_error_deg(R[3], base[2]) < 1.0
    assert not mask[5, 300:].any() and P.rotation_error_deg(R[5], other[2]) < 1.0
    assert abs(np.linalg.norm(t[3]) - 1) < 1e-6
    with pytest.raises(_lib.XFeatLibraryError):               # n_max above 8192 is refused
        z = torch.zeros((1, 8193, 2), device="cuda")
        estimate_relative_pose_batch(z, z, K0[:1], K1[:1])


def test_batch_invariance_and_determinism():
    rng = np.random.default_rng(61)
    scenes = [_scene(rng, int(rng.integers(100, 900)), 0.5, 0.5) for _ in range(12)]
    p0, p1, cnt = _batch(scenes)
    n = cnt.cpu().numpy()
    K0, K1 = np.repeat(KA[None], 12, 0), np.repeat(KB[None], 12, 0)
    ids = np.arange(100, 112, dtype=np.int32)
    a = [x.cpu().numpy() for x in estimate_relative_pose_batch(p0, p1, K0, K1, cnt, pair_ids=ids, seed=7)]
    b = [x.cpu().numpy() for x in estimate_relative_pose_batch(p0, p1, K0, K1, cnt, pair_ids=ids, seed=7)]
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for k in (0, 5, 11):                                      # alone, with its id: the same result bit for bit
        one = [x.cpu().numpy() for x in estimate_relative_pose_batch(p0[k:k + 1, :n[k]], p1[k:k + 1, :n[k]], K0[k:k + 1],
                                                                      K1[k:k + 1], None, pair_ids=ids[k:k + 1], seed=7)]
        for x, y in zip(a, one):
            xs = x[k]
            if x.ndim == 2 and x.shape[1] == p0.shape[1]:
                xs = x[k, :n[k]]
            assert np.array_equal(xs, y[0])


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat(device=0)


def test_pose_pairs_equal_pairs_then_batch(xf, assets_vga, monkeypatch):
    """match_xfeat_pose_pairs equals match_xfeat_pairs followed by estimate_relative_pose_batch(..., pair_ids=[p]) per pair,
    bit for bit, over several chunks."""
    from accelerated_features_b200 import xfeat as xfm
    monkeypatch.setattr(xfm, "PAIRS_MATCH_CHUNK", 3)
    ref, tgt = assets_vga
    images = [ref, tgt, np.ascontiguousarray(ref[::-1]), np.ascontiguousarray(tgt[:, ::-1])]
    K = np.array([[[600.0 + 10 * i, 0, 320], [0, 610.0, 240], [0, 0, 1]] for i in range(4)])
    pairs = np.array([[0, 1], [1, 0], [0, 2], [2, 3], [3, 1], [1, 2], [0, 3]])
    got = xf.match_xfeat_pose_pairs(images, pairs, K, top_k=1024, iters=512, seed=3)
    matched = xf.match_xfeat_pairs(images, pairs, top_k=1024)
    for p, (i, j) in enumerate(pairs):
        a, b = matched[p]
        assert np.array_equal(got[p]["mkpts0"], a) and np.array_equal(got[p]["mkpts1"], b)
        E, R, t, m, n, nf = (x.cpu().numpy() for x in estimate_relative_pose_batch(
            torch.from_numpy(a)[None].cuda(), torch.from_numpy(b)[None].cuda(), K[i:i + 1], K[j:j + 1], None, 1.0, 512, 3,
            pair_ids=[p]))
        assert got[p]["n_inliers"] == n[0] and got[p]["n_front"] == nf[0]
        assert np.array_equal(got[p]["inliers"], m[0])
        if n[0] >= 5:
            for k, v in (("E", E), ("R", R), ("t", t)):
                assert np.array_equal(got[p][k], v[0].astype(np.float64))
        else:
            assert got[p]["E"] is None and got[p]["R"] is None and got[p]["t"] is None
    with pytest.raises(ValueError):
        xf.match_xfeat_pose_pairs(images, pairs, K, top_k=8193)


def test_run_pose_benchmark_batched_equals_per_pair():
    from accelerated_features_b200 import evalharness as eh
    rng = np.random.default_rng(71)
    samples = []
    for b in range(10):
        R, t = P.random_pose(rng)
        K0, K1 = (KA, KB) if b % 2 else (KB, KA)
        n = 3 if b == 4 else int(rng.integers(50, 600))
        p0, p1, _ = P.calibrated_scene(rng, n, K0, K1, R, t, inlier_frac=0.6, noise_px=0.5)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, t
        samples.append({"image0": p0, "image1": p1, "scale0": np.ones(2), "scale1": np.ones(2), "K0": K0, "K1": K1,
                        "T_0to1": T})

    def match_pairs(pairs):
        return [(a.astype(np.float32), b.astype(np.float32)) for a, b in pairs]

    batched = eh.run_pose_benchmark(match_pairs, samples, ransac_thr=1.0, batch_size=4, pose_batch_fn=eh.estimate_poses_gpu)
    single = eh.run_pose_benchmark(match_pairs, samples, ransac_thr=1.0, batch_size=4,
                                   pose_fn=lambda a, b, k0, k1, thr: estimate_relative_pose(a, b, k0, k1, thr))
    assert batched["pairs"] == single["pairs"]
    assert np.isinf(batched["pairs"][4]["R_err"])
