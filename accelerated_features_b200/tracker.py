"""Tracking of one reference frame through a video stream (the per-frame step of the reference's realtime_demo.py): sparse
extraction of the frame, mutual-nearest-neighbour matching against the cached reference at min_cossim 0.82, and homography
RANSAC, replayed as one CUDA graph per frame shape.  `XFeat.tracker(reference, ...)` builds a Tracker.

Per frame shape (the key (B, C, H, W, dtype, "/255", channels-last, on the device)) the first call runs eagerly, which settles
what the library decides on first use (include/xfeat_b200.h, "CUDA-graph capture"); the second call captures the whole step --
the upload out of a pinned staging buffer, every kernel, the download of the results into pinned buffers -- and later calls
replay it, then wait once for the tracker's stream.  Every buffer a graph reads or writes belongs to the tracker: its image
table (slot 0 the reference, slots 1..B the frames), its workspace, its staging and result buffers, and the graph's own memory
pool.  Eager calls on the XFeat instance therefore cannot move memory under a graph, and set_reference rewrites slot 0 in place
without a new capture.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib
from .geometry import find_homography_batch

MAX_TOP_K = 8192        # RS_MAX_PTS of csrc/ransac.cu: the RANSAC kernels cache at most this many correspondences per pair


class _Route:
    """Buffers and graph of one frame key."""

    def __init__(self, B: int, shape, dtype, on_device: bool, channels_last: bool, div255: bool, table, pairs, ws, top_k: int,
                 dev):
        self.B = B
        self.table, self.pairs, self.ws = table, pairs, ws
        self.stage = None if on_device else torch.empty(shape, dtype=dtype, pin_memory=True)
        self.dev_in = torch.empty(shape, dtype=dtype, device=dev)
        self.x = self.dev_in.permute(0, 3, 1, 2) if channels_last else self.dev_in
        self.div255 = div255
        self.out = (torch.empty((B, top_k, 2), dtype=torch.float32, pin_memory=True),      # mkpts0
                    torch.empty((B, top_k, 2), dtype=torch.float32, pin_memory=True),      # mkpts1
                    torch.empty((B,), dtype=torch.int32, pin_memory=True),                 # matches per frame
                    torch.empty((B, 3, 3), dtype=torch.float32, pin_memory=True),          # H
                    torch.empty((B, top_k), dtype=torch.bool, pin_memory=True),            # inlier mask
                    torch.empty((B,), dtype=torch.int32, pin_memory=True))                 # inliers per frame
        self.calls = 0
        self.graph: Optional[torch.cuda.CUDAGraph] = None


class Tracker:
    """Matches frames against one reference image and fits the homography reference -> frame, on the GPU.

        tr = xf.tracker(reference, top_k=None, min_cossim=0.82, ransac_thr=4.0, iters=700, min_inliers=50, seed=0)
        res = tr(frame)              # one frame -> dict
        ress = tr(frames)            # (B,H,W,C) numpy / (B,C,H,W) tensor / list of same-shape frames -> list of B dicts
        tr.set_reference(img)        # new reference, any shape

    Each result holds 'mkpts0' (N,2) reference pixels, 'mkpts1' (N,2) frame pixels, 'inliers' (N,) bool, 'n_inliers' int and
    'H' (3,3) float64, or None when fewer than max(min_inliers, 4) matches support it (realtime_demo.py drops homographies with
    fewer than 50 inliers).  The defaults are realtime_demo.py's: top_k = the XFeat's top_k, cosine similarity above 0.82,
    cv2.findHomography(..., USAC_MAGSAC, 4.0, maxIters=700).  mkpts0 / mkpts1 are what match_xfeat(reference, frame, top_k,
    min_cossim) returns, and H / inliers what geometry.find_homography_batch returns on them (frame b of a batch is RANSAC
    pair b), bit for bit.

    Frames follow match_xfeat_stream's image rules: numpy uint8 or float (H,W) / (H,W,C) / (B,H,W,C), with "/255" for numpy
    (on the device for uint8, on the host for float), or torch (C,H,W) / (B,C,H,W) on the host or the device, taken as they are.
    A 2-D or 3-D input is one frame and gives one dict; a 4-D input or a list gives a list.

    The matcher and convolution implementations and the XFeat's detection threshold in effect when the tracker is built are
    the ones it uses (captured graphs keep them); changing an implementation afterwards makes the next call raise.
    """

    def __init__(self, xf, reference, top_k: Optional[int] = None, min_cossim: float = 0.82, ransac_thr: float = 4.0,
                 iters: int = 700, min_inliers: int = 50, seed: int = 0):
        top_k = xf.top_k if top_k is None else int(top_k)
        if not 1 <= top_k <= MAX_TOP_K:
            raise ValueError(f"tracker: top_k must be in [1, {MAX_TOP_K}] (the RANSAC caches {MAX_TOP_K} matches per frame), "
                             f"got {top_k}")
        if not iters >= 1 or not ransac_thr > 0:
            raise ValueError("tracker: iters must be >= 1 and ransac_thr > 0")
        self.xf = xf
        self.top_k = top_k
        self.min_cossim = float(min_cossim)
        self.ransac_thr = float(ransac_thr)
        self.iters = int(iters)
        self.min_inliers = int(min_inliers)
        self.seed = int(seed)
        self.detection_threshold = xf.detection_threshold
        self._impls = (xf._lib.xfeat_get_mnn_impl(), xf._lib.xfeat_get_conv_impl())
        # the layout match_xfeat_pairs picks: the matcher's operand rows for the presplit implementations, else fp32 descriptors
        self._presplit = self._impls[0] in (1, 2, 3)
        self._desc_key = "desc_split" if self._presplit else "descriptors"
        self._stream = torch.cuda.Stream(xf.dev)
        self._done = torch.cuda.Event()
        self._ref: Optional[Dict[str, torch.Tensor]] = None
        self._tables: Dict[int, Dict[str, torch.Tensor]] = {}      # B -> image table of 1 + B slots
        self._pairs: Dict[int, torch.Tensor] = {}                  # B -> (B, 2) int32 pair table [(0, 1), ..., (0, B)]
        self._routes: Dict[tuple, _Route] = {}
        self.capture_count = 0                                     # graphs captured so far (one per frame key)
        self.set_reference(reference)

    # ------------------------------------------------------------------------------------------------------------------------
    def _frames(self, x):
        """-> (tensor in its natural layout: (B,H,W,C) for numpy, (B,C,H,W) for torch; div255; channels_last; one frame)."""
        if isinstance(x, (list, tuple)):
            if len(x) == 0:
                raise ValueError("tracker: empty list of frames")
            if all(isinstance(f, np.ndarray) for f in x):
                fs = [f[:, :, None] if f.ndim == 2 else f for f in x]
                if any(f.ndim != 3 or f.shape != fs[0].shape or f.dtype != fs[0].dtype for f in fs):
                    raise ValueError("tracker: a list of frames must hold (H,W) or (H,W,C) arrays of one shape and dtype")
                t, div255, cl = self.xf._host_batch(np.stack(fs))
                return t, div255, cl, False
            if all(isinstance(f, torch.Tensor) for f in x):
                fs = [f[0] if f.ndim == 4 and f.shape[0] == 1 else f for f in x]
                if any(f.ndim != 3 or f.shape != fs[0].shape or f.dtype != fs[0].dtype or f.device != fs[0].device for f in fs):
                    raise ValueError("tracker: a list of frames must hold (C,H,W) tensors of one shape, dtype and device")
                return torch.stack(fs), False, False, False
            raise TypeError("tracker: a list of frames must hold numpy arrays or torch tensors, not a mix")
        if isinstance(x, np.ndarray):
            if x.ndim not in (2, 3, 4):
                raise ValueError("tracker: numpy frames must be (H,W), (H,W,C) or (B,H,W,C)")
            single = x.ndim < 4
            t, div255, cl = self.xf._host_batch(x[:, :, None] if x.ndim == 2 else x)
            return t, div255, cl, single
        if isinstance(x, torch.Tensor):
            if x.ndim not in (3, 4):
                raise ValueError("tracker: tensor frames must be (C,H,W) or (B,C,H,W)")
            return (x[None] if x.ndim == 3 else x), False, False, x.ndim == 3
        raise TypeError(f"tracker: unsupported frame type {type(x).__name__}")

    def _check_impls(self):
        now = (self.xf._lib.xfeat_get_mnn_impl(), self.xf._lib.xfeat_get_conv_impl())
        if now != self._impls:
            raise RuntimeError(f"tracker: built under (matcher, convolution) implementations {self._impls}, now {now}; "
                               "build a new tracker")

    def _extract(self, x, div255: bool, out=None, ws=None):
        return self.xf._detect_sparse_device([x], self.top_k, self.detection_threshold, [div255], want_split=self._presplit,
                                             want_desc=not self._presplit, out=out, ws=ws)

    @torch.inference_mode()
    def set_reference(self, img):
        """Extract a new reference (any shape, same input rules as a frame) into slot 0 of every image table.  Runs eagerly on the
        tracker's stream with one host synchronisation; the captured graphs read slot 0 in place, so nothing is re-captured.
        Raises XFeatLibraryError, keeping the previous reference, if the reference's NMS candidate buffer overflows."""
        t, div255, cl, single = self._frames(img)
        if not single:
            raise ValueError("tracker: the reference is one image")
        self._check_impls()
        main = torch.cuda.current_stream(self.xf.dev)
        self._stream.wait_stream(main)
        with torch.cuda.stream(self._stream):
            x = t.to(self.xf.dev)
            o = self._extract(x.permute(0, 3, 1, 2) if cl else x, div255)
            n = int(o["n_valid"].item())
            self.xf._check_counts([n], "tracker.set_reference", ["the reference"])
            self._ref = {k: o[k] for k in ("keypoints", "n_valid", self._desc_key)}
            for tab in self._tables.values():
                for k, v in self._ref.items():
                    tab[k][0].copy_(v[0])
        main.wait_stream(self._stream)

    def _table(self, B: int):
        """Image table of 1 + B slots for batches of B frames, slot 0 filled from the reference."""
        tab = self._tables.get(B)
        if tab is None:
            e = self.xf._empty
            tab = {"keypoints": e((1 + B, self.top_k, 2)), "n_valid": e((1 + B,), torch.int32)}
            if self._presplit:
                tab["desc_split"] = e((1 + B, self.xf._split_rows(self.top_k), 128), torch.float16)
            else:
                tab["descriptors"] = e((1 + B, self.top_k, 64))
            for k, v in self._ref.items():
                tab[k][0].copy_(v[0])
            self._tables[B] = tab
            self._pairs[B] = torch.tensor([[0, b] for b in range(1, B + 1)], dtype=torch.int32, device=self.xf.dev)
        return tab, self._pairs[B]

    def _route(self, key, t: torch.Tensor, div255: bool, cl: bool) -> _Route:
        B = t.shape[0]
        Hi, Wi = (t.shape[1], t.shape[2]) if cl else (t.shape[2], t.shape[3])
        H, W = (Hi // 32) * 32, (Wi // 32) * 32
        if H == 0 or W == 0:
            raise RuntimeError("tracker: frame smaller than 32 pixels")
        lib = self.xf._lib
        match_bytes = (lib.xfeat_mnn_pairs_workspace_bytes(B, self.top_k) if self._presplit
                       else lib.xfeat_mnn_workspace_bytes(B, self.top_k, self.top_k))
        sparse_bytes = lib.xfeat_sparse_workspace_bytes(B, H, W, self.top_k)
        if sparse_bytes == 0:
            raise _lib.XFeatLibraryError("xfeat_sparse_workspace_bytes failed: " + lib.xfeat_last_error().decode())
        nbytes = max(256, lib.xfeat_net_workspace_bytes(B, H, W), sparse_bytes, match_bytes,
                     lib.xfeat_ransac_workspace_bytes(B, self.iters))
        tab, pairs = self._table(B)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.xf.dev)
        r = _Route(B, t.shape, t.dtype, t.is_cuda, cl, div255, tab, pairs, ws, self.top_k, self.xf.dev)
        self._routes[key] = r
        return r

    def _step(self, r: _Route):
        """The whole per-frame step on the current stream: no host synchronisation, no allocation outside the current memory pool,
        every scratch byte from r.ws."""
        if r.stage is not None:
            r.dev_in.copy_(r.stage, non_blocking=True)
        out = {k: v[1:] for k, v in r.table.items()}
        self._extract(r.x, r.div255, out=out, ws=r.ws)
        mk0, mk1, cnt = self.xf._match_table_pairs(r.table, r.pairs, self.top_k, self.min_cossim, self._presplit, ws=r.ws)
        H, mask, n_inl = find_homography_batch(mk0, mk1, cnt, self.ransac_thr, self.iters, self.seed, workspace=r.ws)
        for h, d in zip(r.out, (mk0, mk1, cnt, H, mask, n_inl)):
            h.copy_(d, non_blocking=True)

    def _results(self, mk0: np.ndarray, mk1: np.ndarray, cnt: np.ndarray, H: np.ndarray, mask: np.ndarray,
                 n_inl: np.ndarray) -> List[dict]:
        """Per-frame result dicts from the downloaded buffers of one step.  Raises XFeatLibraryError naming the frames whose NMS
        candidate buffer overflowed (count XF_N_OVERFLOW)."""
        c = [int(v) for v in cnt]
        self.xf._check_counts(c, "tracker", [f"frame {b}" for b in range(len(c))])
        res = []
        for b, n in enumerate(c):
            ni = int(n_inl[b])
            res.append({"mkpts0": mk0[b, :n].copy(), "mkpts1": mk1[b, :n].copy(), "inliers": mask[b, :n].copy(), "n_inliers": ni,
                        "H": H[b].astype(np.float64) if ni >= max(self.min_inliers, 4) else None})
        return res

    @torch.inference_mode()
    def __call__(self, frames):
        self._check_impls()
        t, div255, cl, single = self._frames(frames)
        key = (*t.shape, str(t.dtype).replace("torch.", ""), bool(div255), cl, t.is_cuda)
        main = torch.cuda.current_stream(self.xf.dev)
        with torch.cuda.stream(self._stream):
            r = self._routes.get(key) or self._route(key, t, div255, cl)
            if t.is_cuda:
                self._stream.wait_stream(main)          # the frames come from the caller's stream
                r.dev_in.copy_(t, non_blocking=True)
            else:
                r.stage.copy_(t)                         # host copy; the previous step's upload has finished
            if r.graph is None and r.calls >= 1:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self._stream):
                    self._step(r)
                r.graph = g
                self.capture_count += 1
            if r.graph is not None:
                r.graph.replay()
            else:
                self._step(r)
            r.calls += 1
            self._done.record(self._stream)
        self._done.synchronize()
        res = self._results(*(h.numpy() for h in r.out))
        return res[0] if single else res
