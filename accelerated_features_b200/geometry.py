"""Geometric verification of matches on the GPU (SURVEY 8f-3): the step every caller of the reference runs right after
matching -- `cv2.findHomography(points1, points2, cv2.USAC_MAGSAC, thr, maxIters=700, confidence=0.995)` in
realtime_demo.py:225 and the notebooks -- the essential- and fundamental-matrix estimators, and the calibrated relative pose
(five-point RANSAC + cheirality), for a whole batch of pairs in two kernel launches (homography), three (essential and
fundamental matrix) or four (relative pose; csrc/ransac.cu), without the matches leaving the device."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib


def _intrinsics4(K, B: int, dev) -> torch.Tensor:
    """(B, 3, 3) or (B, 4) intrinsics -> (B, 4) float32 (fx, fy, cx, cy) on `dev`."""
    k = torch.as_tensor(K).to(device=dev, dtype=torch.float32)
    if k.shape == (B, 3, 3):
        k = torch.stack([k[:, 0, 0], k[:, 1, 1], k[:, 0, 2], k[:, 1, 2]], 1)
    if k.shape != (B, 4):
        raise RuntimeError(f"intrinsics must be (B, 3, 3) or (B, 4) with B = {B}, got {tuple(k.shape)}")
    return k.contiguous()


def _ransac_batch(entry: str, diag: float, pts0: torch.Tensor, pts1: torch.Tensor, counts: Optional[torch.Tensor], thr: float,
                  iters: int, seed: int, workspace: Optional[torch.Tensor] = None, pair_ids=None, cams=None) -> Tuple:
    """The one path of the estimators into the C ABI (`entry`): validation, outputs, workspace and the call.  A batch
    without correspondences gets what the kernels report for a pair without a model: `diag` on the model's diagonal (1:
    identity H, 0: zero E / F), an empty mask and a count of 0.  With `cams` = (K0, K1) (the relative pose), the call also
    returns R (B,3,3) (identity without a model), t (B,3) and n_front (B), as (E, R, t, mask, n_inliers, n_front)."""
    lib = _lib.load()
    name = "estimate_relative_pose_batch" if cams is not None else entry.replace("xfeat_ransac_", "find_") + "_batch"
    if not (pts0.is_cuda and pts1.is_cuda):
        raise RuntimeError(f"{name} runs on the GPU only (no CPU fallback)")
    p0 = pts0.float().contiguous()
    p1 = pts1.float().contiguous()
    if p0.ndim != 3 or p0.shape != p1.shape or p0.shape[-1] != 2:
        raise RuntimeError("points must be two (B, n, 2) tensors of the same shape")
    B, n_max, _ = p0.shape
    dev = p0.device
    pose = ()
    if cams is not None:
        k0, k1 = _intrinsics4(cams[0], B, dev), _intrinsics4(cams[1], B, dev)
        pose = (torch.eye(3, device=dev).expand(B, 3, 3).contiguous(), torch.zeros((B, 3), device=dev),
                torch.zeros((B,), dtype=torch.int32, device=dev))
    if B == 0 or n_max == 0:
        model = (diag * torch.eye(3, device=dev)).expand(B, 3, 3).clone()
        empty = (torch.zeros((B, n_max), dtype=torch.bool, device=dev), torch.zeros((B,), dtype=torch.int32, device=dev))
        return (model, *pose[:2], *empty, *pose[2:]) if pose else (model, *empty)
    model = torch.empty((B, 3, 3), dtype=torch.float32, device=dev)
    mask = torch.empty((B, n_max), dtype=torch.uint8, device=dev)
    n_inl = torch.empty((B,), dtype=torch.int32, device=dev)
    cnt = None if counts is None else counts.to(dev).to(torch.int32).contiguous()
    ids = ()
    if entry in ("xfeat_ransac_fundamental", "xfeat_relative_pose"):
        ids = (None,)
        if pair_ids is not None:
            t = torch.as_tensor(pair_ids).to(device=dev, dtype=torch.int32).reshape(-1).contiguous()
            if t.numel() != B:
                raise RuntimeError(f"pair_ids must hold one id per pair ({B}), got {t.numel()}")
            ids = (t.data_ptr(),)
    ws = workspace
    if ws is None:
        ws = torch.empty(max(256, lib.xfeat_ransac_workspace_bytes(B, iters)), dtype=torch.uint8, device=dev)
    K = (k0.data_ptr(), k1.data_ptr()) if pose else ()
    outs = (model.data_ptr(), pose[0].data_ptr(), pose[1].data_ptr()) if pose else (model.data_ptr(),)
    front = (pose[2].data_ptr(),) if pose else ()
    with torch.cuda.device(dev):
        _lib.check(getattr(lib, entry)(p0.data_ptr(), p1.data_ptr(), None if cnt is None else cnt.data_ptr(), *K, *ids, n_max, B,
                                       float(thr), int(iters), int(seed) & 0xffffffff, *outs, mask.data_ptr(), n_inl.data_ptr(),
                                       *front, ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream),
                   entry)
    if pose:
        return model, pose[0], pose[1], mask.bool(), n_inl, pose[2]
    return model, mask.bool(), n_inl


def _one_pair(points1, points2, device: Optional[torch.device]):
    """The input handling of the cv2-shaped single-pair calls: two (N,2) arrays -> two (1, N, 2) float32 device tensors."""
    dev = device or torch.device("cuda", torch.cuda.current_device())
    p0 = torch.as_tensor(np.asarray(points1, dtype=np.float32)).reshape(1, -1, 2).to(dev)
    p1 = torch.as_tensor(np.asarray(points2, dtype=np.float32)).reshape(1, -1, 2).to(dev)
    return p0, p1


def _ransac_one(batch_fn, p_min: int, points1, points2, thr: float, iters: int, seed: int, device: Optional[torch.device]):
    """The cv2-shaped single-pair call: (model (3,3) float64 or None, mask (N,1) uint8); None (and an empty mask) below p_min
    correspondences or p_min inliers."""
    p0, p1 = _one_pair(points1, points2, device)
    n = p0.shape[1]
    if n < p_min:
        return None, np.zeros((n, 1), np.uint8)
    model, mask, n_inl = batch_fn(p0, p1, None, thr, iters, seed)
    if int(n_inl.item()) < p_min:
        return None, np.zeros((n, 1), np.uint8)
    return model[0].double().cpu().numpy(), mask[0].to(torch.uint8).cpu().numpy().reshape(-1, 1)


def find_homography_batch(pts0: torch.Tensor, pts1: torch.Tensor, counts: Optional[torch.Tensor] = None, thr: float = 3.0,
                          iters: int = 1024, seed: int = 0,
                          workspace: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """pts0, pts1: (B, n_max, 2) float32 CUDA tensors of matched coordinates (pair b uses the first counts[b] rows; None: all).
    Returns H (B,3,3) float32 with H[2,2] = 1 mapping image-0 to image-1 pixels, inliers (B, n_max) bool, n_inliers (B) int32.
    A pair with fewer than 4 correspondences, or whose every 4-point sample is degenerate (all points identical, all exactly
    on one line, fewer than 4 distinct points), has no model: identity H, no inliers, n_inliers 0 (a negative count passes
    through).
    `thr`: forward transfer error in pixels of image 1 (cv2's ransacReprojThreshold).  `workspace`: a uint8 CUDA tensor of at
    least xfeat_ransac_workspace_bytes(B, iters) bytes to use as scratch (default: a fresh one), for callers that capture the
    call into a CUDA graph and keep the scratch alive with it."""
    return _ransac_batch("xfeat_ransac_homography", 1.0, pts0, pts1, counts, thr, iters, seed, workspace)


def find_homography(points1, points2, thr: float = 3.0, iters: int = 1024, seed: int = 0, device: Optional[torch.device] = None):
    """cv2.findHomography-shaped call for ONE pair: (N,2) arrays -> (H (3,3) float64 or None, mask (N,1) uint8)."""
    return _ransac_one(find_homography_batch, 4, points1, points2, thr, iters, seed, device)


def find_essential_batch(x0: torch.Tensor, x1: torch.Tensor, counts: Optional[torch.Tensor] = None, thr: float = 1e-3,
                         iters: int = 1024, seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Essential-matrix RANSAC for a batch of pairs (the relative-pose step of the 1500-pair benchmarks,
    modules/eval/megadepth1500.py:98-113).  x0, x1: (B, n_max, 2) NORMALISED image coordinates (K^-1 applied) on the GPU;
    `thr`: Sampson distance threshold in the same units (pixels / focal length).  Returns E (B,3,3) with x1^T E x0 = 0,
    inliers (B, n_max) bool, n_inliers (B)."""
    return _ransac_batch("xfeat_ransac_essential", 0.0, x0, x1, counts, thr, iters, seed)


def find_fundamental_batch(pts0: torch.Tensor, pts1: torch.Tensor, counts: Optional[torch.Tensor] = None, thr: float = 3.0,
                           iters: int = 2048, seed: int = 0, pair_ids=None,
                           workspace: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Fundamental-matrix RANSAC for a batch of pairs: what cv2.findFundamentalMat(p0, p1, cv2.USAC_MAGSAC, thr) computes per
    pair, for uncalibrated, non-planar pairs (photo collections, the 1500-pair benchmarks).  pts0, pts1: (B, n_max, 2) float32
    CUDA tensors of matched PIXEL coordinates (pair b uses the first counts[b] rows; None: all; n_max <= 8192).
    Returns F (B,3,3) float32 with x1^T F x0 = 0 in homogeneous pixels (unit Frobenius norm), inliers (B, n_max) bool and
    n_inliers (B) int32 (a negative count passes through; fewer than 8 correspondences: zero F, no inliers).

    `thr`: Sampson distance in pixels, the USAC meaning of cv2's ransacReprojThreshold (3.0 is cv2's default).  `iters`: 7-point
    samples per pair; 2048 because an all-inlier sample has probability w^7, 6.4e-4 at w = 0.35, so 2048 samples draw about
    1.3 of them, and the local optimisation recovers the full consensus set from a near-all-inlier one.  `pair_ids` (B ints,
    default 0..B-1) seed each pair's samples: with its id fixed, a pair's result does not depend on its batch.  `workspace`: as
    find_homography_batch.  A planar scene has no unique F: no degeneracy test is made."""
    return _ransac_batch("xfeat_ransac_fundamental", 0.0, pts0, pts1, counts, thr, iters, seed, workspace,
                         pair_ids)


def find_fundamental(points1, points2, thr: float = 3.0, iters: int = 2048, seed: int = 0,
                     device: Optional[torch.device] = None):
    """cv2.findFundamentalMat-shaped call for ONE pair: (N,2) pixel arrays -> (F (3,3) float64 or None, mask (N,1) uint8).
    None (and an empty mask) below 8 correspondences or 8 inliers.  Arguments as find_fundamental_batch."""
    return _ransac_one(find_fundamental_batch, 8, points1, points2, thr, iters, seed, device)


def estimate_relative_pose_batch(pts0: torch.Tensor, pts1: torch.Tensor, K0, K1, counts: Optional[torch.Tensor] = None,
                                 thr: float = 1.0, iters: int = 1024, seed: int = 0, pair_ids=None,
                                 workspace: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, ...]:
    """Calibrated relative pose for a batch of pairs, on the GPU: the estimate_pose_poselib step of the 1500-pair benchmarks
    (modules/eval/megadepth1500.py:98-113; poselib's non-linear refinement is not done).  pts0, pts1: (B, n_max, 2) float32
    CUDA tensors of matched PIXEL coordinates (pair b uses the first counts[b] rows; None: all; n_max <= 8192); K0, K1: each
    pair's intrinsics, (B, 3, 3) or (B, 4) as (fx, fy, cx, cy), any mix of cameras.

    Five-point RANSAC on K^-1-normalised coordinates (MSAC on the Sampson distance, locally optimised winners), then the
    cheirality test on the inliers.  `thr`: pixels, as estimate_pose_opencv's `thresh`: the Sampson threshold is thr / f with
    f = (fx0 + fy0 + fx1 + fy1) / 4.  `iters`: 5-point samples per pair; 1024 because an all-inlier sample has probability
    w^5, 0.53 % at an inlier ratio w = 0.35, so 1024 samples draw about 5 of them, and the local optimisation recovers the full
    consensus set from a near-all-inlier one.  `pair_ids` (B ints, default 0..B-1) seed each pair's samples: with its id fixed,
    a pair's result does not depend on its batch.  `workspace`: as find_homography_batch.

    Returns device tensors, without a host synchronisation: E (B,3,3) float32 with x1^T E x0 = 0 in normalised coordinates,
    R (B,3,3) and unit t (B,3) float32 with X1 = R X0 + t, inliers (B, n_max) bool, n_inliers (B) int32 (a negative count
    passes through) and n_front (B) int32, the inliers in front of both cameras under (R, t).  A pair with fewer than 5
    correspondences, or without a model, gets zero E, R = I, t = 0, no inliers, n_inliers and n_front 0."""
    return _ransac_batch("xfeat_relative_pose", 0.0, pts0, pts1, counts, thr, iters, seed, workspace, pair_ids, (K0, K1))


def estimate_relative_pose(points1, points2, K0, K1, thr: float = 1.0, iters: int = 1024, seed: int = 0,
                           device: Optional[torch.device] = None):
    """The single-pair call, shaped as evalharness.estimate_pose_opencv's result: (N,2) pixel arrays and (3,3) or (4,)
    intrinsics -> (R (3,3) float64, t (3,) float64 unit, mask (N,) bool) or None below 5 correspondences or 5 inliers.
    Arguments as estimate_relative_pose_batch (the pair is seeded as pair 0)."""
    p0, p1 = _one_pair(points1, points2, device)
    if p0.shape[1] < 5:
        return None
    k0 = torch.as_tensor(np.asarray(K0, np.float32)).reshape(1, *np.shape(K0))
    k1 = torch.as_tensor(np.asarray(K1, np.float32)).reshape(1, *np.shape(K1))
    _, R, t, mask, n_inl, _ = estimate_relative_pose_batch(p0, p1, k0, k1, None, thr, iters, seed)
    if int(n_inl.item()) < 5:
        return None
    return R[0].double().cpu().numpy(), t[0].double().cpu().numpy(), mask[0].cpu().numpy()


def recover_pose(E: np.ndarray, x0: np.ndarray, x1: np.ndarray):
    """(R, t) with X1 = R X0 + t from an essential matrix and normalised inlier correspondences: the candidate (of the four
    decompositions) that puts the most triangulated points in front of both cameras (what cv2.recoverPose does)."""
    U, _, Vt = np.linalg.svd(E)
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    Wm = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
    best, ret = -1, None
    h0 = np.concatenate([x0, np.ones((len(x0), 1))], 1)
    h1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    for R in (U @ Wm @ Vt, U @ Wm.T @ Vt):
        for t in (U[:, 2], -U[:, 2]):
            # depth of X0 along ray h0: solve z0 (R h0) - z1 h1 = -t in the least-squares sense, per point
            a = (R @ h0.T).T
            A = np.stack([a, -h1], 2)                                    # (n, 3, 2)
            AtA = np.einsum("nij,nik->njk", A, A)
            Atb = np.einsum("nij,i->nj", A, -t)
            z = np.linalg.solve(AtA + 1e-12 * np.eye(2), Atb[..., None])[..., 0]
            good = int(((z[:, 0] > 0) & (z[:, 1] > 0)).sum())
            if good > best:
                best, ret = good, (R, t)
    return ret
