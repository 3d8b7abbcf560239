"""Batched form of the reference's evaluation callers (SURVEY 8f-2).

`modules/eval/megadepth1500.py:200-237` (run_pose_benchmark) and `modules/eval/scannet1500.py:207-230` call
`matcher_fn(bgr0, bgr1)` one pair at a time, 1500 times.  Here the same protocol runs the matcher over the whole list of pairs
(sparse: XFeat.match_xfeat_pairs, semi-dense: XFeat.match_xfeat_star_pairs; each distinct image extracted once) and returns
the matches in the callers' order, so the pose / AUC stage downstream is unchanged.  The metric functions are
restated from the reference (citations on each) because its module imports poselib at import time, which is not installed
here; the pose estimator is pluggable (default: OpenCV's 5-point RANSAC as a stand-in for poselib)."""
from __future__ import annotations

from typing import Callable, Dict, Iterable, List, Sequence, Tuple

import numpy as np


def batched_matcher(xf, mode: str = "sparse", top_k=None, batch_size: int = 64) -> Callable[[Sequence[Tuple[np.ndarray, np.ndarray]]], List[Tuple[np.ndarray, np.ndarray]]]:
    """-> match_pairs(pairs): pairs = [(img0, img1)] numpy (H,W,3) uint8 images (any mix of shapes) -> [(mkpts0, mkpts1)] in the
    same order; what [matcher_fn(a, b) for a, b in pairs] returns with matcher_fn = xfeat.match_xfeat / match_xfeat_star.
    One call over the whole list -- sparse: match_xfeat_pairs, star: match_xfeat_star_pairs -- in which an image object that
    appears in several pairs is extracted once (images are told apart by identity).  `batch_size` is not used any more (both
    modes size their launches themselves); it stays for the callers that pass it."""
    if mode not in ("sparse", "star"):
        raise ValueError("mode must be 'sparse' or 'star'")
    match_list = xf.match_xfeat_pairs if mode == "sparse" else xf.match_xfeat_star_pairs

    def match_pairs(pairs):
        images: List[np.ndarray] = []
        slot: Dict[int, int] = {}
        idx = []
        for pair in pairs:
            for im in pair:
                if id(im) not in slot:
                    slot[id(im)] = len(images)
                    images.append(im)
            idx.append([slot[id(pair[0])], slot[id(pair[1])]])
        return match_list(images, np.asarray(idx, np.int64).reshape(-1, 2), top_k=top_k)

    return match_pairs


# ---- metrics: restated from modules/eval/megadepth1500.py ------------------------------------------------------------
def relative_pose_error(T_0to1, R, t, ignore_gt_t_thr=0.0):
    """megadepth1500.py:69-85: angular errors (degrees) of the translation direction (up to sign) and of the rotation."""
    t_gt = T_0to1[:3, 3]
    n = np.linalg.norm(t) * np.linalg.norm(t_gt)
    t_err = np.rad2deg(np.arccos(np.clip(np.dot(t, t_gt) / n, -1.0, 1.0)))
    t_err = np.minimum(t_err, 180 - t_err)
    if np.linalg.norm(t_gt) < ignore_gt_t_thr:
        t_err = 0
    R_gt = T_0to1[:3, :3]
    cos = np.clip((np.trace(np.dot(R.T, R_gt)) - 1) / 2, -1.0, 1.0)
    return t_err, np.rad2deg(np.abs(np.arccos(cos)))


def error_auc(errors, thresholds=(5, 10, 20)):
    """megadepth1500.py:159-176: area under the recall-vs-error curve up to each threshold."""
    errors = [0] + sorted(list(errors))
    recall = list(np.linspace(0, 1, len(errors)))
    aucs = []
    for thr in thresholds:
        last_index = int(np.searchsorted(errors, thr))
        y = recall[:last_index] + [recall[last_index - 1]]
        x = errors[:last_index] + [thr]
        aucs.append(float(np.trapezoid(y, x) / thr) if hasattr(np, "trapezoid") else float(np.trapz(y, x) / thr))
    return {f"auc@{t}": a for t, a in zip(thresholds, aucs)}


def compute_maa(pairs, thresholds=(5, 10, 20)):
    """megadepth1500.py:178-197, returning the numbers it prints."""
    errors = np.array([max(p["t_err"], p["R_err"]) for p in pairs])
    out = error_auc(errors, thresholds)
    for t in thresholds:
        out[f"mAcc@{t}"] = float((errors <= t).sum() / len(errors))
    return out


def estimate_pose_opencv(kpts0, kpts1, K0, K1, thresh, conf=0.99999):
    """Stand-in for estimate_pose_poselib (megadepth1500.py:98-113): 5-point RANSAC on normalised coordinates + cheirality."""
    import cv2
    if len(kpts0) < 5:
        return None
    f = 0.25 * (K0[0, 0] + K0[1, 1] + K1[0, 0] + K1[1, 1])
    n0 = (kpts0 - K0[[0, 1], [2, 2]][None]) / K0[[0, 1], [0, 1]][None]
    n1 = (kpts1 - K1[[0, 1], [2, 2]][None]) / K1[[0, 1], [0, 1]][None]
    E, mask = cv2.findEssentialMat(n0, n1, np.eye(3), threshold=thresh / f, prob=conf, method=cv2.RANSAC)
    if E is None:
        return None
    best, ret = 0, None
    for _E in np.split(E, len(E) // 3):
        n, R, t, _ = cv2.recoverPose(_E, n0, n1, np.eye(3), 1e9, mask=mask.copy())
        if n > best:
            best, ret = n, (R, t[:, 0], mask.ravel() > 0)
    return ret


def estimate_pose_gpu(kpts0, kpts1, K0, K1, thresh, iters: int = 8192, seed: int = 0):
    """estimate_pose_poselib's role (megadepth1500.py:98-113) on the GPU: essential-matrix RANSAC (geometry.find_essential_batch,
    8-point + Sampson + re-fit) and the cheirality test.  Same signature / return as estimate_pose_opencv.  An 8-point sample is
    all-inlier with probability w^8 (0.4 % at w = 0.5, against 3 % for a 5-point solver): hence the default of 8192 hypotheses."""
    import torch
    from .geometry import find_essential_batch, recover_pose
    if len(kpts0) < 8:
        return None
    f = 0.25 * (K0[0, 0] + K0[1, 1] + K1[0, 0] + K1[1, 1])
    n0 = ((kpts0 - K0[[0, 1], [2, 2]][None]) / K0[[0, 1], [0, 1]][None]).astype(np.float32)
    n1 = ((kpts1 - K1[[0, 1], [2, 2]][None]) / K1[[0, 1], [0, 1]][None]).astype(np.float32)
    E, mask, n_inl = find_essential_batch(torch.from_numpy(n0)[None].cuda(), torch.from_numpy(n1)[None].cuda(), None,
                                          thr=thresh / f, iters=iters, seed=seed)
    if int(n_inl.item()) < 8:
        return None
    m = mask[0].cpu().numpy()
    R, t = recover_pose(E[0].double().cpu().numpy(), n0[m].astype(np.float64), n1[m].astype(np.float64))
    return R, t, m


def estimate_poses_gpu(kpts0: Sequence[np.ndarray], kpts1: Sequence[np.ndarray], K0: Sequence[np.ndarray],
                       K1: Sequence[np.ndarray], thresh, iters: int = 1024, seed: int = 0) -> List:
    """estimate_pose_opencv over a chunk of pairs in ONE batched call of geometry.estimate_relative_pose_batch (five-point
    RANSAC + cheirality on the GPU, per-pair intrinsics): lists of (N_i,2) pixel keypoints and (3,3) intrinsics -> per pair
    (R, t, mask) or None, as estimate_pose_opencv returns.  Every pair is seeded as pair 0, so pair i's result is what
    geometry.estimate_relative_pose(kpts0[i], kpts1[i], K0[i], K1[i], thresh, iters, seed) returns.  At most 8192 keypoints
    per pair."""
    import torch
    from .geometry import estimate_relative_pose_batch
    B = len(kpts0)
    if B == 0:
        return []
    n = np.array([len(k) for k in kpts0], np.int32)
    p0 = np.zeros((B, max(int(n.max()), 1), 2), np.float32)
    p1 = np.zeros_like(p0)
    for b in range(B):
        p0[b, :n[b]], p1[b, :n[b]] = kpts0[b], kpts1[b]
    dev = torch.device("cuda", torch.cuda.current_device())
    E, R, t, mask, n_inl, _ = estimate_relative_pose_batch(
        torch.from_numpy(p0).to(dev), torch.from_numpy(p1).to(dev), np.asarray(K0, np.float32), np.asarray(K1, np.float32),
        torch.from_numpy(n).to(dev), thresh, iters, seed, pair_ids=np.zeros(B, np.int32))
    R, t, mask, n_inl = R.double().cpu().numpy(), t.double().cpu().numpy(), mask.cpu().numpy(), n_inl.cpu().numpy()
    return [(R[b], t[b], mask[b, :n[b]].copy()) if n[b] >= 5 and n_inl[b] >= 5 else None for b in range(B)]


def run_pose_benchmark(match_pairs, samples: Iterable[dict], ransac_thr: float = 2.5, batch_size: int = 64,
                       pose_fn=estimate_pose_opencv, pose_batch_fn=None) -> dict:
    """run_pose_benchmark (megadepth1500.py:200-237) over batches.  `samples`: dicts with 'image0', 'image1' (H,W,3) uint8 BGR
    (what tensor2bgr produces there), 'scale0', 'scale1', 'K0', 'K1', 'T_0to1' as numpy arrays.  Returns compute_maa's numbers
    plus the per-pair records.  `pose_batch_fn` (e.g. estimate_poses_gpu), when given, is called once per chunk with the lists
    of the chunk's (kpts0, kpts1, K0, K1) and the threshold, instead of pose_fn once per pair."""
    samples = list(samples)
    records = []
    for o in range(0, len(samples), batch_size):
        chunk = samples[o:o + batch_size]
        matches = match_pairs([(d["image0"], d["image1"]) for d in chunk])
        scaled = [(src * np.asarray(d["scale0"], np.float32), dst * np.asarray(d["scale1"], np.float32))   # rescale kpts
                  for d, (src, dst) in zip(chunk, matches)]                                             # (megadepth1500.py:230-231)
        Ks = [(np.asarray(d["K0"], np.float64), np.asarray(d["K1"], np.float64)) for d in chunk]
        if pose_batch_fn is not None:
            rets = pose_batch_fn([s for s, _ in scaled], [s for _, s in scaled], [k for k, _ in Ks], [k for _, k in Ks],
                                 ransac_thr)
        else:
            rets = [pose_fn(src, dst, k0, k1, ransac_thr) for (src, dst), (k0, k1) in zip(scaled, Ks)]
        for d, (src, _), ret in zip(chunk, scaled, rets):
            rec = {"R_err": np.inf, "t_err": np.inf, "n_matches": len(src)}
            if ret is not None:
                R, t, _ = ret
                rec["t_err"], rec["R_err"] = relative_pose_error(np.asarray(d["T_0to1"], np.float64), R, t)
            records.append(rec)
    out = compute_maa(records)
    out["pairs"] = records
    return out
