"""XFeat.tracker against the public calls it composes: match_xfeat(reference, frame, top_k, min_cossim=0.82) for the matches and
geometry.find_homography_batch on those matches for H / inliers, bit for bit -- on the eager first call, the capturing second
call and the replays, across reference switches, frame-shape changes, batches and workspace growth of the XFeat instance."""
import cv2
import numpy as np
import pytest
import torch

from accelerated_features_b200 import _lib
from accelerated_features_b200.geometry import find_homography_batch
from tests.test_gpu_mnn_tc import mnn_impl

pytestmark = pytest.mark.gpu

TOPK = 4096
THR, ITERS, SEED, MIN_INL = 4.0, 700, 0, 50


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat(device=0)


def warp_frames(img, n, seed):
    """n seeded perspective warps of img (corners moved by up to 60 px): [(frame, true 3x3 homography img -> frame)]."""
    rng = np.random.default_rng(seed)
    h, w = img.shape[:2]
    src = np.float32([[0, 0], [w, 0], [w, h], [0, h]])
    out = []
    for _ in range(n):
        Hm = cv2.getPerspectiveTransform(src, (src + rng.uniform(-60, 60, src.shape)).astype(np.float32))
        out.append((cv2.warpPerspective(img, Hm, (w, h), flags=cv2.INTER_LINEAR), Hm))
    return out


@pytest.fixture(scope="module")
def frames(assets_vga):
    ref, tgt = assets_vga
    warps = warp_frames(ref, 6, seed=5)
    return ref, [tgt] + [f for f, _ in warps], [None] + [Hm for _, Hm in warps]


def oracle(xf, ref, frames, top_k=TOPK, min_inliers=MIN_INL):
    """What the tracker must return for one batch of frames, from match_xfeat and one batched find_homography_batch call."""
    ms = [xf.match_xfeat(ref, f[:, :, None] if isinstance(f, np.ndarray) and f.ndim == 2 else f, top_k=top_k, min_cossim=0.82)
          for f in frames]
    B = len(frames)
    p0, p1 = torch.zeros((B, top_k, 2)), torch.zeros((B, top_k, 2))
    cnt = torch.tensor([len(a) for a, _ in ms], dtype=torch.int32)
    for b, (a, c) in enumerate(ms):
        p0[b, :len(a)], p1[b, :len(c)] = torch.from_numpy(a), torch.from_numpy(c)
    H, mask, n_inl = find_homography_batch(p0.cuda(), p1.cuda(), cnt.cuda(), THR, ITERS, SEED)
    H, mask, n_inl = H.cpu().double().numpy(), mask.cpu().numpy(), n_inl.cpu().numpy()
    return [{"mkpts0": a, "mkpts1": c, "inliers": mask[b, :len(a)], "n_inliers": int(n_inl[b]),
             "H": H[b] if n_inl[b] >= max(min_inliers, 4) else None} for b, (a, c) in enumerate(ms)]


def assert_same(got, want, what):
    assert set(got) == {"mkpts0", "mkpts1", "inliers", "n_inliers", "H"}, what
    assert got["mkpts0"].dtype == np.float32 and got["inliers"].dtype == np.bool_, what
    for k in ("mkpts0", "mkpts1", "inliers"):
        assert np.array_equal(got[k], want[k]), f"{what}: {k} differs ({len(got[k])} vs {len(want[k])} rows)"
    assert got["n_inliers"] == want["n_inliers"], what
    if want["H"] is None:
        assert got["H"] is None, what
    else:
        assert got["H"].dtype == np.float64 and got["H"].shape == (3, 3), what
        assert np.array_equal(got["H"], want["H"]), f"{what}: H differs"


@pytest.mark.parametrize("impl", [1, 0])
def test_frames_and_batches_equal_public_calls(xf, frames, impl):
    """Implementation 1 (default) works on the matcher's operand rows, implementation 0 on fp32 descriptors.  Each frame key
    runs eagerly, then captures, then replays."""
    ref, fs, _ = frames
    with mnn_impl(xf, impl):
        tr = xf.tracker(ref)
        want = [oracle(xf, ref, [f])[0] for f in fs]
        for i, f in enumerate(fs):
            assert_same(tr(f), want[i], f"impl {impl} frame {i}")
        assert tr.capture_count == 1
        batch = np.stack(fs[1:4])
        want3 = oracle(xf, ref, list(batch))            # RANSAC pair b = frame b of the batch
        for rep in range(3):
            got = tr(batch)
            assert isinstance(got, list) and len(got) == 3
            for b in range(3):
                assert_same(got[b], want3[b], f"impl {impl} batch call {rep} frame {b}")
        assert tr.capture_count == 2


def test_sixty_frame_sequence_one_capture(xf, frames):
    ref, fs, _ = frames
    want = [oracle(xf, ref, [f])[0] for f in fs]
    tr = xf.tracker(ref)
    for i in range(60):
        assert_same(tr(fs[i % len(fs)]), want[i % len(fs)], f"sequence frame {i}")
    assert tr.capture_count == 1


def test_reference_switch_and_frame_shapes(xf, frames, assets_vga):
    ref, fs, _ = frames
    tr = xf.tracker(ref)
    for f in fs[:3]:
        tr(f)
    assert tr.capture_count == 1
    ref2 = np.ascontiguousarray(assets_vga[1][40:424, 32:608])          # another shape: 384 x 576
    tr.set_reference(ref2)
    for i, f in enumerate(fs[:4]):
        assert_same(tr(f), oracle(xf, ref2, [f])[0], f"new reference, frame {i}")
    assert tr.capture_count == 1
    small = [np.ascontiguousarray(f[16:464, 48:592]) for f in fs[:3]]    # a second frame shape: 448 x 544
    for rep in range(2):
        for i, f in enumerate(small):
            assert_same(tr(f), oracle(xf, ref2, [f])[0], f"second shape, round {rep}, frame {i}")
    assert tr.capture_count == 2
    for i, f in enumerate(fs[:3]):
        assert_same(tr(f), oracle(xf, ref2, [f])[0], f"first shape again, frame {i}")
    assert tr.capture_count == 2


def test_instance_workspace_growth_does_not_disturb_graphs(xf, frames):
    ref, fs, _ = frames
    tr = xf.tracker(ref, top_k=2048)
    want = [oracle(xf, ref, [f], top_k=2048)[0] for f in fs[:3]]
    for i, f in enumerate(fs[:3]):
        assert_same(tr(f), want[i], f"before growth, frame {i}")
    big = [cv2.resize(f, (1920, 1440), interpolation=cv2.INTER_LINEAR) for f in fs[:3]]
    before = {k: v.numel() for k, v in xf._ws.items()}
    xf.match_xfeat_pairs(big, [(0, 1), (1, 2)], top_k=8192)                   # the caller's stream
    with torch.cuda.stream(tr._stream):                                        # and the tracker's own stream
        xf.match_xfeat_pairs(big, [(2, 0)], top_k=8192)
    torch.cuda.synchronize()
    assert any(xf._ws[k].numel() > before.get(k, 0) for k in xf._ws), "the instance workspace did not grow"
    for i in range(6):
        assert_same(tr(fs[i % 3]), want[i % 3], f"after growth, frame {i}")
    assert tr.capture_count == 1


def test_constant_frame_and_inlier_gate(xf, frames):
    ref, fs, _ = frames
    tr = xf.tracker(ref)
    flat = np.full((480, 640, 3), 128, np.uint8)
    for _ in range(3):
        r = tr(flat)
        assert len(r["mkpts0"]) == 0 and r["n_inliers"] == 0 and r["H"] is None
    w = oracle(xf, ref, [fs[0]])[0]
    assert w["n_inliers"] >= 4
    strict = xf.tracker(ref, min_inliers=w["n_inliers"] + 1)
    for _ in range(3):
        r = strict(fs[0])
        assert r["n_inliers"] == w["n_inliers"] and r["H"] is None
        assert np.array_equal(r["mkpts0"], w["mkpts0"]) and np.array_equal(r["inliers"], w["inliers"])


def test_overflow_names_the_frame_and_tracker_recovers(xf, frames):
    """The NMS overflow of a real image cannot be provoked reliably, so the host step that unpacks a replay is given counts
    holding XF_N_OVERFLOW for frame 1."""
    ref, fs, _ = frames
    tr = xf.tracker(ref)
    for f in fs[:2]:
        tr(f)
    B = 3
    cnt = np.array([7, _lib.N_OVERFLOW, 3], np.int32)
    args = (np.zeros((B, TOPK, 2), np.float32), np.zeros((B, TOPK, 2), np.float32), cnt, np.zeros((B, 3, 3), np.float32),
            np.zeros((B, TOPK), bool), np.zeros(B, np.int32))
    with pytest.raises(_lib.XFeatLibraryError, match=r"frame 1\b"):
        tr._results(*args)
    assert_same(tr(fs[2]), oracle(xf, ref, [fs[2]])[0], "frame after the overflow")


def test_rejects_top_k_above_ransac_cache(xf, frames):
    with pytest.raises(ValueError, match="8192"):
        xf.tracker(frames[0], top_k=8193)


def test_input_forms(xf, frames):
    ref, fs, _ = frames
    tr = xf.tracker(ref)
    gray = cv2.cvtColor(fs[1], cv2.COLOR_RGB2GRAY)
    dev = torch.from_numpy(fs[2]).permute(2, 0, 1).float().cuda() / 255
    flt = fs[3].astype(np.float32)
    for rep in range(3):
        assert_same(tr(gray), oracle(xf, ref, [gray])[0], f"numpy gray, call {rep}")
        assert_same(tr(fs[1]), oracle(xf, ref, [fs[1]])[0], f"numpy uint8 HWC, call {rep}")
        assert_same(tr(dev), oracle(xf, ref, [dev])[0], f"device float tensor, call {rep}")
        assert_same(tr(flt), oracle(xf, ref, [flt])[0], f"numpy float HWC, call {rep}")
    got = tr([fs[1], fs[4]])
    want = oracle(xf, ref, [fs[1], fs[4]])
    assert len(got) == 2
    for b, (g, w) in enumerate(zip(got, want)):
        assert_same(g, w, f"list item {b}")
    one = tr(dev[None])
    assert isinstance(one, list) and len(one) == 1


def test_homography_matches_true_warp(xf, frames):
    ref, fs, Hs = frames
    tr = xf.tracker(ref)
    for i in range(1, len(fs)):
        r = tr(fs[i])
        assert r["H"] is not None, f"warp {i}: {r['n_inliers']} inliers"
        p = np.concatenate([r["mkpts0"][r["inliers"]].astype(np.float64), np.ones((r["n_inliers"], 1))], 1)
        a, b = p @ r["H"].T, p @ Hs[i].T
        err = np.linalg.norm(a[:, :2] / a[:, 2:] - b[:, :2] / b[:, 2:], axis=1)
        assert err.mean() < 1.0, f"warp {i}: mean transfer error {err.mean():.3f} px over {len(err)} inliers"
