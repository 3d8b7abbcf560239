"""Drop-in replacement for `modules.xfeat.XFeat` (verlab/accelerated_features) on NVIDIA H100.

Same constructor, method names, argument meaning, return types and error behaviour as the reference class
(modules/xfeat.py), but every operation of the hot path runs in libxfeat_sm90.so (hand-written sm_90a CUDA kernels
behind the C-ABI of include/xfeat_b200.h).  PyTorch is used for device memory, streams and the final slicing only.
There is no CPU / eager fallback: without a CUDA device and the built library the constructor raises.

Beyond the reference surface: `match_xfeat_batch` (batched match_xfeat) and `match_xfeat_stream` (pinned, double-buffered
host -> device -> host pipeline over a sequence of batches; SURVEY 8f-1), `match_lighterglue_batch` and
`match_xfeat_lighterglue_batch` (LighterGlue on batches of pairs, csrc/lighterglue.cu), `match_xfeat_pairs` and
`match_xfeat_lighterglue_pairs` (a list of pairs into one set of mixed-size images, each image extracted once),
`match_xfeat_star_pairs` (the same for semi-dense matching: XFeat* over a list of pairs, each image extracted once per scale),
`tracker` (one reference tracked through a video stream, each frame's step replayed as one CUDA graph; tracker.py), and
`match_xfeat_verified_pairs` (match_xfeat_pairs followed on the device by a fundamental-matrix RANSAC per pair; geometry.py).
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Dict, Iterable, Iterator, List, Optional, Tuple

import numpy as np
import torch

from . import _lib
from . import weights as _weights

_F32 = np.float32
_D2H_ON_MAIN = bool(os.environ.get("XFEAT_STREAM_D2H_MAIN"))   # A/B switch of match_xfeat_stream: results leave on the compute stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# ----------------------------------------------------------------------------------------------------------------------
# host-side plan of match_xfeat_pairs (no device work: testable without a GPU)
# ----------------------------------------------------------------------------------------------------------------------
PAIRS_EXTRACT_CHUNK = 64      # images per extraction launch sequence
PAIRS_MATCH_CHUNK = 4096      # pairs per matcher launch (and per host synchronisation)
# device bytes per match_xfeat_star_pairs matcher chunk (split operands, matcher and refine workspaces, outputs): about 39 pairs
# at 10 000 rows per image, 96 at 4096; the image table and the extraction come on top
STAR_PAIRS_MATCH_BYTES = 2 << 30


def pair_image_key(x) -> tuple:
    """Extraction bucket of one image of match_xfeat_pairs: (C, H, W, dtype, div255), with the dtype and the "/255" flag that
    _parse_input gives it (numpy uint8: "/255" on the device; numpy float: divided on the host, float32; tensors: as they are).
    numpy (H,W) is read as (H,W,1); tensors are (C,H,W) or (1,C,H,W)."""
    if isinstance(x, np.ndarray):
        if x.ndim == 2:
            return (1, x.shape[0], x.shape[1], "uint8" if x.dtype == np.uint8 else "float32", x.dtype == np.uint8)
        if x.ndim == 3:
            return (x.shape[2], x.shape[0], x.shape[1], "uint8" if x.dtype == np.uint8 else "float32", x.dtype == np.uint8)
        raise RuntimeError("match_xfeat_pairs: numpy images must be (H,W) or (H,W,C)")
    if isinstance(x, torch.Tensor):
        if x.ndim == 4 and x.shape[0] == 1:
            x = x[0]
        if x.ndim != 3:
            raise RuntimeError("match_xfeat_pairs: tensor images must be (C,H,W) or (1,C,H,W)")
        return (x.shape[0], x.shape[1], x.shape[2], str(x.dtype).replace("torch.", ""), False)
    raise RuntimeError(f"match_xfeat_pairs: unsupported image type {type(x).__name__}")


def check_pairs(pairs, n_images: int) -> np.ndarray:
    """`pairs` as a validated (P, 2) int64 array of indices into `n_images` images (P = 0 for an empty input)."""
    a = np.asarray(pairs)
    if a.size == 0:
        return np.zeros((0, 2), np.int64)
    if a.ndim != 2 or a.shape[1] != 2:
        raise ValueError(f"pairs must be (P, 2), got shape {a.shape}")
    if not np.issubdtype(a.dtype, np.integer):
        raise TypeError(f"pairs must hold integers, got {a.dtype}")
    if a.min() < 0 or a.max() >= n_images:
        bad = np.nonzero((a < 0).any(1) | (a >= n_images).any(1))[0]
        raise ValueError(f"pairs {bad[:8].tolist()} index outside the {n_images} images")
    return a.astype(np.int64)


def _dense_cells(h: int, w: int) -> int:
    """1/8-resolution cells of an h x w image after preprocess_tensor's crop to multiples of 32 (xfeat.py:229-231)."""
    return ((h // 32) * 32 // 8) * ((w // 32) * 32 // 8)


def _dense_cap(top_k: int) -> int:
    return 100_000_000 if top_k < 1 else top_k           # extractDense: `if top_k < 1: top_k = 100_000_000` (xfeat.py:357-358)


def dense_counts(H: int, W: int, top_k: int, s1: float = 0.6, s2: float = 1.3) -> Tuple[int, int]:
    """Rows (k1, k2) that extract_dualscale gives an H x W image at its two scales (xfeat.py:379-394): the first scale keeps
    int(top_k * 0.2) cells, the second int(top_k * 0.8), each capped by the cells of the rescaled image, and a cap below 1 means
    unlimited (so top_k = 4 leaves the first scale unlimited).  A scale whose image is under 32 pixels gives 0 rows."""
    t1, t2 = _dense_cap(int(top_k * 0.20)), _dense_cap(int(top_k * 0.80))      # xfeat.py:385-386
    k1 = min(_dense_cells(int(math.floor(H * s1)), int(math.floor(W * s1))), t1)
    k2 = min(_dense_cells(int(math.floor(H * s2)), int(math.floor(W * s2))), t2)
    return k1, k2


def star_pair_rows(keys, plan: "PairPlan", top_k: int) -> np.ndarray:
    """(n_slots,) int32: dense rows k1 + k2 of each planned image of match_xfeat_star_pairs.  Raises, naming the image, for an
    image match_xfeat_star would refuse (under 32 pixels after the 0.6 rescale)."""
    rows = np.zeros(plan.n_slots, np.int32)
    for i in np.nonzero(plan.slot >= 0)[0].tolist():
        H, W = keys[i][1], keys[i][2]
        k1, k2 = dense_counts(H, W, top_k)
        if k1 == 0 or k2 == 0:
            raise RuntimeError(f"match_xfeat_star_pairs: image {i} ({H}x{W}): image smaller than 32 pixels after the 0.6 rescale")
        rows[plan.slot[i]] = k1 + k2
    return rows


# carve_refine (csrc/refine.cu) per coarse-row slot: X (128), two MLP activations (512 each), logits (64), tmp (4), keep (1)
_REFINE_ROW_BYTES = 4 * (128 + 512 + 512 + 64 + 4 + 1)


def star_pair_bytes(k_max: int) -> int:
    """Device bytes one pair of a match_xfeat_star_pairs chunk needs at k_max rows per image: [hi | lo] operand rows of both
    sides (512 B per padded row), best12 / best21, idx0 / idx1, the refine workspace and the refined matches, plus 2 KB for the
    workspaces' 256-byte alignment."""
    n_pad = (k_max + 511) // 512 * 512
    return 2 * n_pad * 256 + k_max * (2 * 8 + 2 * 8 + _REFINE_ROW_BYTES + 16) + 2048


def star_match_chunks(n_pairs: int, k_max: int, budget: Optional[int] = None) -> List[Tuple[int, int]]:
    """[start, stop) ranges of the matched pairs: as many pairs per chunk as fit in `budget` bytes (STAR_PAIRS_MATCH_BYTES), at
    least one, at most 65535 (the kernels' grid limit)."""
    budget = STAR_PAIRS_MATCH_BYTES if budget is None else budget
    step = max(1, min(65535, budget // star_pair_bytes(k_max)))
    return [(o, min(o + step, n_pairs)) for o in range(0, n_pairs, step)]


class PairPlan:
    """Which images match_xfeat_pairs extracts, where their rows go and how the pairs address them.

    chunks: lists of image indices; each list shares one bucket key and is at most `chunk` long.  Table slots are assigned in
    chunk order (chunk 0 takes slots 0..len-1, ...), so slot[image] is the image's row in the keypoint / operand tables (-1:
    no pair references it, not extracted).  table_pairs (P, 2) int32: the pairs in slot numbers."""

    def __init__(self, keys, pairs, chunk: int = PAIRS_EXTRACT_CHUNK):
        self.pairs = check_pairs(pairs, len(keys))
        used = np.zeros(len(keys), bool)
        used[self.pairs.ravel()] = True
        buckets: Dict[tuple, List[int]] = {}
        for n in np.nonzero(used)[0].tolist():
            buckets.setdefault(keys[n], []).append(n)
        self.chunks = [b[o:o + chunk] for b in buckets.values() for o in range(0, len(b), chunk)]
        self.slot = np.full(len(keys), -1, np.int64)
        order = [n for c in self.chunks for n in c]
        self.slot[order] = np.arange(len(order))
        self.n_slots = len(order)
        self.table_pairs = self.slot[self.pairs].astype(np.int32).reshape(-1, 2)

    def match_order(self) -> np.ndarray:
        """Order in which the pairs are matched: by (j, i) of the table pairs, so that the pairs running at the same time stream
        the same second image (its rows stay in L2)."""
        return np.lexsort((self.table_pairs[:, 0], self.table_pairs[:, 1]))


class InterpolateSparse2d(torch.nn.Module):
    """Mirror of modules/interpolator.py:10-33: sample a (B,C,H',W') map at sparse (x,y) positions given in an H x W frame
    (grid_sample, align_corners=False, zeros padding) -> (B,N,C).  Runs xfeat_interpolate_sparse."""

    _MODES = {"nearest": 0, "bilinear": 1, "bicubic": 2}

    def __init__(self, mode: str = "bicubic", align_corners: bool = False):
        super().__init__()
        if mode not in self._MODES:
            raise ValueError(f"unsupported interpolation mode {mode!r}")
        self.mode = mode
        self.align_corners = align_corners

    @torch.inference_mode()
    def forward(self, x: torch.Tensor, pos: torch.Tensor, H: int, W: int) -> torch.Tensor:
        lib = _lib.load()
        if not x.is_cuda:
            raise RuntimeError("InterpolateSparse2d runs on the GPU only (no CPU fallback)")
        x = x.float().contiguous()
        pos = pos.to(x.device).float().contiguous()      # int64 / float positions: true division happens in fp32 (interpolator.py:19)
        B, C, Hm, Wm = x.shape
        N = pos.shape[1]
        out = torch.empty((B, N, C), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(lib.xfeat_interpolate_sparse(x.data_ptr(), pos.data_ptr(), B, C, Hm, Wm, N, int(H), int(W),
                                                    self._MODES[self.mode], out.data_ptr(),
                                                    torch.cuda.current_stream(x.device).cuda_stream), "xfeat_interpolate_sparse")
        return out


class _FineMatcher(torch.nn.Module):
    """`XFeat.net.fine_matcher` (model.py:97-111): (N,128) -> (N,64) logits through xfeat_fine_matcher."""

    def __init__(self, owner: "XFeat"):
        super().__init__()
        object.__setattr__(self, "_o", owner)      # not a registered sub-module: no parent <-> child cycle

    @torch.inference_mode()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        o = self._o
        x = x.to(o.dev).float().contiguous()
        if x.ndim != 2 or x.shape[1] != 128:
            raise RuntimeError("fine_matcher expects (N,128)")
        n = x.shape[0]
        out = o._empty((n, 64))
        if n == 0:
            return out
        ws = o._workspace(o._lib.xfeat_fine_matcher_workspace_bytes(n))
        with torch.cuda.device(o.dev):
            _lib.check(o._lib.xfeat_fine_matcher(o._ctx, x.data_ptr(), n, out.data_ptr(), ws.data_ptr(), ws.numel(), o._stream()),
                       "xfeat_fine_matcher")
        return out


class _Net(torch.nn.Module):
    """Stands in for `XFeat.net` (XFeatModel, model.py:27): callable (B,C,H,W) -> (feats, keypoints, heatmap)."""

    def __init__(self, owner: "XFeat"):
        super().__init__()
        object.__setattr__(self, "_o", owner)
        self.fine_matcher = _FineMatcher(owner)

    @torch.inference_mode()
    def forward(self, x: torch.Tensor):
        """XFeatModel.forward (model.py:123-154).  x: (B,C,H,W) with H, W multiples of 32.
        Returns feats (B,64,H/8,W/8), keypoint logits (B,65,H/8,W/8), reliability (B,1,H/8,W/8) as NCHW *views*
        of channels-last storage."""
        o = self._o
        x = x.to(o.dev)
        B, C, H, W = x.shape
        if H % 32 or W % 32:
            raise RuntimeError("XFeatModel input must have H, W divisible by 32")
        xn = o._preprocess(x, H, W, div255=False)
        feats, heat, rel, logits = o._run_net(xn, B, H, W, want_logits=True)
        return feats.permute(0, 3, 1, 2), logits.permute(0, 3, 1, 2), rel.unsqueeze(1)


# LightGlue prunes an image only while it has more points than this; 1536 is upstream's threshold on CUDA with
# scaled-dot-product attention available (what the reference runs on an H100 with torch 2.x).  DESIGN section 7.
LG_PRUNE_MIN_POINTS = 1536


class _LighterGlue:
    """`XFeat.lighterglue`: the matcher's handle (packed weights on the device, xfeat_lg_create)."""

    def __init__(self, owner: "XFeat", weights):
        self._lib = owner._lib
        blob = _weights.pack_lighterglue(_weights.load_lighterglue_state(weights))
        handle = ctypes.c_void_p()
        _lib.check(self._lib.xfeat_lg_create(ctypes.byref(handle), owner.dev.index, blob.ctypes.data, blob.size), "xfeat_lg_create")
        self.ctx = handle

    def __del__(self):
        try:
            if getattr(self, "ctx", None):
                self._lib.xfeat_lg_destroy(self.ctx)
                self.ctx = None
        except Exception:
            pass


class XFeat(torch.nn.Module):
    """H100-native XFeat inference (sparse `detectAndCompute` / `match_xfeat`, semi-dense `match_xfeat_star`)."""

    def __init__(self, weights=_weights.DEFAULT_WEIGHTS, top_k: int = 4096, detection_threshold: float = 0.05,
                 device: Optional[int] = None, lighterglue_weights=_weights.LG_DEFAULT_WEIGHTS):
        # reference: xfeat.py:23-46.  `weights`: path (.pt/.npz), state_dict mapping, or None (random init).
        # `lighterglue_weights`: the published xfeat-lighterglue.pt (or its matcher state re-saved as .npz, or a mapping); read on
        # the first LighterGlue call
        super().__init__()
        if not torch.cuda.is_available():
            raise RuntimeError("accelerated_features_b200.XFeat needs a CUDA device (sm_90a); there is no CPU fallback")
        self._lib = _lib.load()
        dev_index = torch.cuda.current_device() if device is None else int(device)
        self.dev = torch.device("cuda", dev_index)
        self.top_k = top_k
        self.detection_threshold = detection_threshold
        sd = _weights.random_state_dict(0) if weights is None else _weights.load_state_dict(weights)
        if isinstance(weights, str):
            print("loading weights from: " + weights)
        blob = _weights.pack_weights(sd)
        handle = ctypes.c_void_p()
        _lib.check(self._lib.xfeat_create(ctypes.byref(handle), dev_index, blob.ctypes.data, blob.size), "xfeat_create")
        self._ctx = handle
        self._ws: Dict[int, torch.Tensor] = {}          # grow-only workspace per CUDA stream (kernels are stream ordered)
        self.net = _Net(self)
        self.interpolator = InterpolateSparse2d("bicubic")   # xfeat.py:37
        self.kornia_available = False
        self.lighterglue = None
        self._lighterglue_weights = lighterglue_weights
        self._pipe = None                               # lazily built copy pipeline of match_xfeat_stream

    def __del__(self):
        try:
            if getattr(self, "_ctx", None):
                self._lib.xfeat_destroy(self._ctx)
                self._ctx = None
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------------------------
    # plumbing
    # ------------------------------------------------------------------------------------------------------------
    def _stream(self) -> int:
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _workspace(self, nbytes: int) -> torch.Tensor:
        """Scratch memory for the current stream.  One buffer per stream: work queued on another stream keeps its own
        scratch, and a re-allocation only ever replaces the buffer of the stream that is asking (the caching allocator keeps
        the old block alive until that stream's queued work is done)."""
        key = self._stream()
        ws = self._ws.get(key)
        if ws is None or ws.numel() < nbytes:
            self._ws.pop(key, None)
            ws = torch.empty(int(nbytes * 1.05) + 4096, dtype=torch.uint8, device=self.dev)
            self._ws[key] = ws
        return ws

    def _empty(self, shape, dtype=torch.float32) -> torch.Tensor:
        return torch.empty(shape, dtype=dtype, device=self.dev)

    @staticmethod
    def _img_args(x: torch.Tensor):
        """(tensor, dtype code) with a layout the kernels can address in place."""
        if x.dtype == torch.uint8:
            return x, 1
        if x.dtype != torch.float32:
            x = x.float()          # same as the reference's `.float()` (xfeat.py:233)
        return x, 0

    @staticmethod
    def _check_counts(counts: List[int], what: str, labels: Optional[List[str]] = None):
        """`labels`: how to name item b in the error (default: "batch items [b, ...]")."""
        if counts and min(counts) < 0:
            bad = [i for i, c in enumerate(counts) if c < 0]
            items = f"batch items {bad}" if labels is None else ", ".join(labels[i] for i in bad)
            raise _lib.XFeatLibraryError(
                f"{what}: NMS candidate buffer overflow (more than H*W/4 maxima above the threshold) for {items}; "
                "nothing is returned for them rather than an arbitrary subset")

    def _preprocess(self, x: torch.Tensor, H: int, W: int, div255: bool, out: Optional[torch.Tensor] = None,
                    scale: Optional[float] = None) -> torch.Tensor:
        """xfeat_preprocess: resize to (H,W), channel mean, InstanceNorm -> (B,H,W) fp32 (optionally into `out`).
        `scale`: source-coordinate scale of an F.interpolate(scale_factor=1/scale) (default: in / out, F.interpolate(size=...))."""
        x, code = self._img_args(x)
        B, C, Hi, Wi = x.shape
        sb, sc, sh, sw = x.stride()
        xn = self._empty((B, H, W)) if out is None else out
        stats = self._empty((B, 2), torch.float64)
        with torch.cuda.device(self.dev):
            if scale is None:
                _lib.check(self._lib.xfeat_preprocess(x.data_ptr(), code, B, C, Hi, Wi, sb, sc, sh, sw, int(div255), H, W,
                                                      xn.data_ptr(), stats.data_ptr(), self._stream()), "xfeat_preprocess")
            else:
                sf = float(_F32(scale))
                _lib.check(self._lib.xfeat_preprocess_scaled(x.data_ptr(), code, B, C, Hi, Wi, sb, sc, sh, sw, int(div255), H, W, sf, sf,
                                                             xn.data_ptr(), stats.data_ptr(), self._stream()),
                           "xfeat_preprocess_scaled")
        return xn

    def _run_net(self, xn: torch.Tensor, B: int, H: int, W: int, want_logits: bool = False, ws: Optional[torch.Tensor] = None):
        """`ws`: scratch to use instead of the instance's per-stream workspace (a caller that captures the call into a CUDA graph
        passes one it owns, so that a later eager call growing the instance's workspace cannot free memory the graph reads)."""
        feats = self._empty((B, H // 8, W // 8, 64))
        heat = self._empty((B, H, W))
        rel = self._empty((B, H // 8, W // 8))
        logits = self._empty((B, H // 8, W // 8, 65)) if want_logits else None
        if ws is None:
            ws = self._workspace(self._lib.xfeat_net_workspace_bytes(B, H, W))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_net(self._ctx, xn.data_ptr(), B, H, W, feats.data_ptr(), heat.data_ptr(),
                                           rel.data_ptr(), _ptr(logits), ws.data_ptr(), ws.numel(), self._stream()),
                       "xfeat_net")
        return feats, heat, rel, logits

    def _to_bchw(self, x) -> torch.Tensor:
        """preprocess_tensor's input handling (xfeat.py:221-233): numpy (H,W)/(H,W,C) or tensor (B,C,H,W)."""
        if isinstance(x, np.ndarray):
            if len(x.shape) == 3:
                x = torch.from_numpy(np.ascontiguousarray(x)).permute(2, 0, 1)[None]
            elif len(x.shape) == 2:
                x = torch.from_numpy(np.ascontiguousarray(x))[None, None]
            else:
                raise RuntimeError('For numpy arrays, only (H,W) or (H,W,C) format is supported.')
        if len(x.shape) != 4:
            raise RuntimeError('Input tensor needs to be in (B,C,H,W) format')
        return x.to(self.dev, non_blocking=True)

    # ------------------------------------------------------------------------------------------------------------
    # sparse path
    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _split_rows(top_k: int) -> int:
        return (top_k + 511) // 512 * 512                       # row padding of the tensor-core matcher (mnn_tc.cu)

    def _detect_sparse_device(self, x, top_k: int, detection_threshold: float, div255=False, want_split: bool = False,
                              want_desc: bool = True, out: Optional[Dict[str, torch.Tensor]] = None,
                              ws: Optional[torch.Tensor] = None):
        """Whole sparse extraction on the device, fixed-capacity outputs, no host sync.  `x` is one image batch or a list
        of batches of identical shape (they are normalised into one activation batch without concatenating the inputs);
        `div255` is one flag or one per batch (parse_input's "/255" applies to numpy inputs only, xfeat.py:400-401).
        `want_split`: also return 'desc_split' (B, split_rows, 128) fp16, the matcher's pre-split operand rows.
        `out`: write 'keypoints', 'n_valid' and (when asked for) 'descriptors' / 'desc_split' into these (B, ...) tensors, e.g.
        slices of an image table, instead of fresh ones.
        `ws`: scratch for the network and the selection instead of the instance's workspace (see _run_net).
        Returns dict of device tensors: keypoints (B,k,2), scores (B,k), descriptors (B,k,64), n_valid (B) int32."""
        xs = [self._to_bchw(t) for t in (x if isinstance(x, (list, tuple)) else [x])]
        flags = list(div255) if isinstance(div255, (list, tuple)) else [div255] * len(xs)
        if len(flags) != len(xs):
            raise RuntimeError("one div255 flag per image batch")
        _, _, Hi, Wi = xs[0].shape
        if any(t.shape[1:] != xs[0].shape[1:] for t in xs):
            raise RuntimeError("image batches must share (C,H,W)")
        B = sum(t.shape[0] for t in xs)
        H, W = (Hi // 32) * 32, (Wi // 32) * 32
        if H == 0 or W == 0:
            raise RuntimeError("image smaller than 32 pixels")
        if top_k < 1:
            raise RuntimeError("top_k must be positive")
        rh, rw = Hi / H, Wi / W                                     # python floats, as xfeat.py:237
        xn = self._empty((B, H, W))
        o = 0
        for t, f in zip(xs, flags):
            self._preprocess(t, H, W, bool(f), out=xn[o:o + t.shape[0]])
            o += t.shape[0]
        if ws is None:
            feats, heat, rel, _ = self._run_net(xn, B, H, W)
        else:
            feats, heat, rel, _ = self._run_net(xn, B, H, W, ws=ws)
        dst = out or {}
        kpts = dst["keypoints"] if "keypoints" in dst else self._empty((B, top_k, 2))
        scores = self._empty((B, top_k))
        desc = None
        if want_desc or not want_split:                     # match-only callers take the split rows alone
            desc = dst["descriptors"] if "descriptors" in dst else self._empty((B, top_k, 64))
        n_valid = dst["n_valid"] if "n_valid" in dst else self._empty((B,), torch.int32)
        n_cand = self._empty((B,), torch.int32)
        nbytes = self._lib.xfeat_sparse_workspace_bytes(B, H, W, top_k)
        if nbytes == 0:
            raise _lib.XFeatLibraryError("xfeat_sparse_workspace_bytes failed: " + self._lib.xfeat_last_error().decode())
        if ws is None:
            ws = self._workspace(nbytes)
        split_rows = self._split_rows(top_k)
        split = None
        if want_split:
            split = dst["desc_split"] if "desc_split" in dst else self._empty((B, split_rows, 128), torch.float16)
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_detect_sparse_split(self._ctx, feats.data_ptr(), heat.data_ptr(), rel.data_ptr(), B, H, W,
                                                           top_k, float(detection_threshold), float(_F32(rw)), float(_F32(rh)),
                                                           kpts.data_ptr(), scores.data_ptr(), _ptr(desc),
                                                           n_valid.data_ptr(), n_cand.data_ptr(), None, _ptr(split),
                                                           split_rows if want_split else 0, ws.data_ptr(),
                                                           ws.numel(), self._stream()), "xfeat_detect_sparse_split")
        return {"keypoints": kpts, "scores": scores, "descriptors": desc, "n_valid": n_valid, "n_cand": n_cand,
                "feats": feats, "heat": heat, "reliability": rel, "H": H, "W": W, "desc_split": split}

    @torch.inference_mode()
    def detectAndCompute(self, x, top_k=None, detection_threshold=None) -> List[Dict[str, torch.Tensor]]:
        """Compute sparse keypoints & descriptors, batched (reference: xfeat.py:49-103).

        x -> torch.Tensor(B,C,H,W) or np.ndarray (H,W)/(H,W,C), grayscale or rgb.
        Returns List[Dict]: 'keypoints' (N,2) (x,y), 'scores' (N,), 'descriptors' (N,64); sorted by score, N <= top_k.
        """
        if top_k is None: top_k = self.top_k
        if detection_threshold is None: detection_threshold = self.detection_threshold
        out = self._detect_sparse_device(x, top_k, detection_threshold)
        n = out["n_valid"].tolist()                                   # the only host sync
        self._check_counts(n, "detectAndCompute")
        return [{"keypoints": out["keypoints"][b, :n[b]], "scores": out["scores"][b, :n[b]],
                 "descriptors": out["descriptors"][b, :n[b]]} for b in range(len(n))]

    def _mnn_device(self, f1, n1, n1_max, stride1, f2, n2, n2_max, stride2, batch, min_cossim, abs_bound=0.0, ws=None):
        """abs_bound > 0: the caller guarantees max|f| <= abs_bound (1.0 for the sparse path's unit-norm descriptors), which
        spares the tensor-core matcher its max-reduction pass over both descriptor sets.  `ws`: see _run_net."""
        idx0 = self._empty((batch, n1_max), torch.int64)
        idx1 = self._empty((batch, n1_max), torch.int64)
        cnt = self._empty((batch,), torch.int32)
        if ws is None:
            ws = self._workspace(self._lib.xfeat_mnn_workspace_bytes(batch, n1_max, n2_max))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_mnn_match_bounded(f1.data_ptr(), _ptr(n1), n1_max, stride1, f2.data_ptr(), _ptr(n2),
                                                         n2_max, stride2, batch, float(min_cossim), float(abs_bound),
                                                         idx0.data_ptr(), idx1.data_ptr(), cnt.data_ptr(), ws.data_ptr(),
                                                         ws.numel(), self._stream()),
                       "xfeat_mnn_match_bounded")
        return idx0, idx1, cnt

    @staticmethod
    def _as_desc(f: torch.Tensor, dev) -> torch.Tensor:
        f = f.to(dev)
        if f.dtype != torch.float32:
            f = f.float()
        return f.contiguous()

    @torch.inference_mode()
    def match(self, feats1, feats2, min_cossim=0.82):
        """Mutual nearest neighbours of two descriptor sets (reference: xfeat.py:327-348) -> (idx0, idx1) int64."""
        f1, f2 = self._as_desc(feats1, self.dev), self._as_desc(feats2, self.dev)
        if f1.ndim != 2 or f2.ndim != 2 or f1.shape[-1] != 64 or f2.shape[-1] != 64:
            raise RuntimeError("descriptors must be (N,64)")
        if len(f1) == 0 or len(f2) == 0:
            e = torch.empty((0,), dtype=torch.int64, device=self.dev)
            return e, e.clone()
        idx0, idx1, cnt = self._mnn_device(f1, None, len(f1), 0, f2, None, len(f2), 0, 1, min_cossim)
        n = int(cnt.item())
        return idx0[0, :n], idx1[0, :n]

    @torch.inference_mode()
    def batch_match(self, feats1, feats2, min_cossim=-1):
        """Batched MNN on raw dot products (reference: xfeat.py:265-290) -> list of B (idx0_b, idx1_b)."""
        f1, f2 = self._as_desc(feats1, self.dev), self._as_desc(feats2, self.dev)
        if f1.ndim != 3 or f2.ndim != 3 or f1.shape[-1] != 64 or f2.shape[-1] != 64 or f1.shape[0] != f2.shape[0]:
            raise RuntimeError("descriptors must be (B,N,64) with the same B")
        B, n1, _ = f1.shape
        n2 = f2.shape[1]
        if B == 0 or n1 == 0 or n2 == 0:
            e = torch.empty((0,), dtype=torch.int64, device=self.dev)
            return [(e, e.clone()) for _ in range(B)]
        idx0, idx1, cnt = self._mnn_device(f1, None, n1, n1 * 64, f2, None, n2, n2 * 64, B, min_cossim)
        c = cnt.tolist()
        return [(idx0[b, :c[b]], idx1[b, :c[b]]) for b in range(B)]

    def _match_sparse_batch_device(self, imgs1, imgs2, top_k: int, min_cossim: float, div255=False):
        """Extraction of both image sets + per-pair MNN + keypoint gather, all on the device (no host sync).
        `div255`: one flag, or (flag for imgs1, flag for imgs2).  Returns mkpts0, mkpts1 (B,top_k,2) and n_matches (B) int32
        (XF_N_OVERFLOW for a pair whose NMS candidate buffer overflowed)."""
        x1, x2 = self._to_bchw(imgs1), self._to_bchw(imgs2)
        da, db = (div255 if isinstance(div255, (list, tuple)) else (div255, div255))
        B = x1.shape[0]
        if x2.shape[0] != B:
            raise RuntimeError("the two image sets must have the same batch size")
        if x1.shape[1:] == x2.shape[1:]:
            presplit = self._lib.xfeat_get_mnn_impl() in (1, 2, 3)     # the sampler writes the matcher's operand rows itself
            o = self._detect_sparse_device([x1, x2], top_k, self.detection_threshold, [da, db], want_split=presplit,
                                           want_desc=not presplit)
            k1, k2 = o["keypoints"][:B], o["keypoints"][B:]
            n1, n2 = o["n_valid"][:B], o["n_valid"][B:]
            if not presplit:
                d1, d2 = o["descriptors"][:B], o["descriptors"][B:]
            if presplit:
                sp = o["desc_split"]
                idx0, idx1, cnt = self._mnn_presplit_device(sp[:B], n1, sp[B:], n2, top_k, sp.shape[1], B, min_cossim)
                return self._gather_matches(k1, k2, idx0, idx1, cnt, B, top_k)
        else:
            o1 = self._detect_sparse_device(x1, top_k, self.detection_threshold, da)
            o2 = self._detect_sparse_device(x2, top_k, self.detection_threshold, db)
            k1, k2, d1, d2, n1, n2 = (o1["keypoints"], o2["keypoints"], o1["descriptors"], o2["descriptors"],
                                      o1["n_valid"], o2["n_valid"])
        idx0, idx1, cnt = self._mnn_device(d1, n1, top_k, top_k * 64, d2, n2, top_k, top_k * 64, B, min_cossim,
                                           abs_bound=1.0)   # xfeat_detect_sparse writes unit-norm rows
        return self._gather_matches(k1, k2, idx0, idx1, cnt, B, top_k)

    def _gather_matches(self, k1, k2, idx0, idx1, cnt, B: int, top_k: int):
        mk0, mk1 = self._empty((B, top_k, 2)), self._empty((B, top_k, 2))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_gather_matches(k1.data_ptr(), k2.data_ptr(), top_k, top_k, idx0.data_ptr(),
                                                      idx1.data_ptr(), cnt.data_ptr(), B, mk0.data_ptr(), mk1.data_ptr(),
                                                      self._stream()), "xfeat_gather_matches")
        return mk0, mk1, cnt

    def _mnn_presplit_device(self, f1s, n1, f2s, n2, n_max: int, n_pad: int, batch: int, min_cossim: float):
        """xfeat_mnn_match_presplit on the operand rows xfeat_detect_sparse_split wrote (no max-reduction / split pass)."""
        idx0 = self._empty((batch, n_max), torch.int64)
        idx1 = self._empty((batch, n_max), torch.int64)
        cnt = self._empty((batch,), torch.int32)
        ws = self._workspace(self._lib.xfeat_mnn_presplit_workspace_bytes(batch, n_max, n_max))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_mnn_match_presplit(f1s.data_ptr(), _ptr(n1), n_max, f2s.data_ptr(), _ptr(n2), n_max, n_pad,
                                                          batch, 13, float(min_cossim), idx0.data_ptr(), idx1.data_ptr(),
                                                          cnt.data_ptr(), ws.data_ptr(), ws.numel(), self._stream()),
                       "xfeat_mnn_match_presplit")
        return idx0, idx1, cnt

    @torch.inference_mode()
    def match_xfeat(self, img1, img2, top_k=None, min_cossim=-1) -> Tuple[np.ndarray, np.ndarray]:
        """Extract + MNN match one image pair (reference: xfeat.py:165-186; only batch item 0 is used, as there).
        Returns mkpts_0, mkpts_1 -> np.ndarray (N,2)."""
        if top_k is None: top_k = self.top_k
        img1, d1 = self._parse_input(img1)
        img2, d2 = self._parse_input(img2)
        mk0, mk1, cnt = self._match_sparse_batch_device(img1[:1], img2[:1], top_k, min_cossim, div255=(d1, d2))
        n = int(cnt.item())
        self._check_counts([n], "match_xfeat")
        return mk0[0, :n].cpu().numpy(), mk1[0, :n].cpu().numpy()

    @torch.inference_mode()
    def match_xfeat_batch(self, imgs1, imgs2, top_k=None, min_cossim=-1) -> List[Tuple[np.ndarray, np.ndarray]]:
        """Batched extension of match_xfeat (the reference has none: xfeat.py:169): pair b = (imgs1[b], imgs2[b]).
        Host inputs travel through the pinned copy pipeline of match_xfeat_stream."""
        return next(self.match_xfeat_stream([(imgs1, imgs2)], top_k=top_k, min_cossim=min_cossim))

    @torch.inference_mode()
    def match_xfeat_verified_batch(self, imgs1, imgs2, top_k=None, min_cossim=-1, ransac_thr: float = 3.0, iters: int = 1024,
                                   seed: int = 0) -> List[Dict[str, np.ndarray]]:
        """match_xfeat_batch followed, still on the device, by the homography RANSAC the reference's callers run on the matches
        (cv2.findHomography(..., USAC_MAGSAC, thr) in realtime_demo.py:225): per pair {'mkpts0', 'mkpts1' (N,2), 'H' (3,3),
        'inliers' (N,) bool}.  One host synchronisation for the whole batch."""
        from .geometry import find_homography_batch
        if top_k is None: top_k = self.top_k
        x1, d1 = self._parse_input(imgs1)
        x2, d2 = self._parse_input(imgs2)
        mk0, mk1, cnt = self._match_sparse_batch_device(x1, x2, top_k, min_cossim, div255=(d1, d2))
        H, mask, _ = find_homography_batch(mk0, mk1, cnt, ransac_thr, iters, seed)
        c = cnt.tolist()
        self._check_counts(c, "match_xfeat_verified_batch")
        mk0, mk1, H, mask = mk0.cpu().numpy(), mk1.cpu().numpy(), H.cpu().numpy(), mask.cpu().numpy()
        return [{"mkpts0": mk0[b, :c[b]], "mkpts1": mk1[b, :c[b]], "H": H[b], "inliers": mask[b, :c[b]]} for b in range(len(c))]

    def tracker(self, reference, top_k=None, min_cossim: float = 0.82, ransac_thr: float = 4.0, iters: int = 700,
                min_inliers: int = 50, seed: int = 0):
        """A Tracker (tracker.py) of `reference` through a video stream: per frame, match_xfeat(reference, frame, top_k,
        min_cossim) and the homography RANSAC of match_xfeat_verified_batch, replayed as one CUDA graph per frame shape with the
        reference extracted once.  The defaults are realtime_demo.py's (min_cossim 0.82, USAC_MAGSAC at 4 px, 700 iterations,
        homographies with fewer than 50 inliers dropped).  top_k above 8192 is refused."""
        from .tracker import Tracker
        return Tracker(self, reference, top_k, min_cossim, ransac_thr, iters, min_inliers, seed)

    # ------------------------------------------------------------------------------------------------------------
    # streaming: pinned, double-buffered host -> device -> host pipeline (SURVEY 8f-1)
    # ------------------------------------------------------------------------------------------------------------
    class _Pipe:
        """Per-instance copy machinery: a copy stream, two device input slots and two pinned result slots with their events."""

        def __init__(self, dev):
            self.copy = torch.cuda.Stream(dev)
            self.dev_in = [None, None]           # [(tensor1, tensor2)] device input slots
            self.stage = [None, None]            # pinned staging for pageable host inputs
            self.ready = [torch.cuda.Event(), torch.cuda.Event()]
            self.freed = [torch.cuda.Event(), torch.cuda.Event()]
            self.res = [None, None]              # pinned (mk0, mk1, cnt)
            self.res_dev = [None, None]          # the device tensors being copied out (kept alive until the copy has finished)
            self.d2h = torch.cuda.Stream(dev)    # results leave on their own stream: the next batch's kernels do not queue behind them
            self.computed = [torch.cuda.Event(), torch.cuda.Event()]
            self.done = [torch.cuda.Event(), torch.cuda.Event()]

    def pinned_like(self, shape, dtype=torch.uint8) -> torch.Tensor:
        """A page-locked host tensor.  Fill it and hand it (a (B,C,H,W) tensor) -- or its `.numpy()` view for (B,H,W,C) uint8
        camera frames -- to match_xfeat_stream / match_xfeat_batch: pinned memory skips the staging copy pageable memory needs."""
        return torch.empty(shape, dtype=dtype, pin_memory=True)

    def _host_batch(self, x) -> Tuple[torch.Tensor, bool, bool]:
        """-> (tensor in its natural layout (B,H,W,C numpy style or B,C,H,W tensor style), div255 flag, channels_last)."""
        if isinstance(x, np.ndarray):
            if x.ndim == 3:
                x = x[None]
            if x.ndim != 4:
                raise RuntimeError("numpy image batches must be (B,H,W,C) or (H,W,C)")
            t = torch.from_numpy(np.ascontiguousarray(x))
            if t.dtype != torch.uint8:
                return t.float() / 255, False, True        # parse_input (xfeat.py:400-401) on the host for float arrays
            return t, True, True
        if x.ndim == 3:
            x = x[None]
        if x.ndim != 4:
            raise RuntimeError("Input tensor needs to be in (B,C,H,W) format")
        return x, False, False

    def _upload(self, pipe, slot: int, batches):
        """Queue the H2D copies of a list of image batches on the copy stream (into the slot's device buffers): the two image
        sets of one match_xfeat_stream batch, or the images of one match_xfeat_pairs chunk."""
        hs = [self._host_batch(b) for b in batches]
        devs, stages = [], []
        prev_dev = pipe.dev_in[slot] or []
        prev_stage = pipe.stage[slot] or []
        for j, (t, _, _) in enumerate(hs):          # device slots come from the compute stream's pool (they are read there)
            if t.is_cuda:
                devs.append(t)
                continue
            old = prev_dev[j] if j < len(prev_dev) else None
            if old is None or old.shape != t.shape or old.dtype != t.dtype or old.data_ptr() == t.data_ptr():
                old = torch.empty(t.shape, dtype=t.dtype, device=self.dev)
            devs.append(old)
        for j, (t, _, _) in enumerate(hs):
            st = None
            if not t.is_cuda and not t.is_pinned():
                st = prev_stage[j] if j < len(prev_stage) else None
                if st is None or st.shape != t.shape or st.dtype != t.dtype:
                    st = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                else:
                    pipe.ready[slot].synchronize()           # the previous H2D out of this staging buffer has finished
                st.copy_(t)                                  # host memcpy into page-locked memory
            stages.append(st)
        with torch.cuda.stream(pipe.copy):
            pipe.copy.wait_event(pipe.freed[slot])           # the kernels that read this slot two batches ago are done
            for j, (t, _, _) in enumerate(hs):
                if not t.is_cuda:
                    devs[j].copy_(stages[j] if stages[j] is not None else t, non_blocking=True)
            pipe.ready[slot].record(pipe.copy)
        pipe.dev_in[slot] = devs
        pipe.stage[slot] = stages
        return [(d.permute(0, 3, 1, 2) if cl else d, f) for d, (_, f, cl) in zip(devs, hs)]

    @torch.inference_mode()
    def match_xfeat_stream(self, batches: Iterable, top_k=None, min_cossim=-1) -> Iterator[List[Tuple[np.ndarray, np.ndarray]]]:
        """Sparse extract + match over a sequence of batches with copies overlapped with compute.

        batches: iterable of (imgs1, imgs2); each image set is a numpy (B,H,W,C) array (uint8: "/255" on the device, as
        parse_input does for numpy images, xfeat.py:396-403) or a torch (B,C,H,W) tensor, on the host (pinned or pageable)
        or already on the device.  Yields, per batch and in order, a list of B (mkpts_0, mkpts_1) numpy pairs -- what B calls
        of the reference's match_xfeat return.

        Batch i+1 is uploaded on a copy stream while batch i computes; the results of batch i come back through pinned
        buffers while batch i+1 computes (its list is yielded once batch i+1 has been queued)."""
        if top_k is None: top_k = self.top_k
        if self._pipe is None:
            self._pipe = XFeat._Pipe(self.dev)
        pipe = self._pipe
        main = torch.cuda.current_stream(self.dev)
        for ev in pipe.freed:
            ev.record(main)
        it = iter(batches)

        def finish(slot):
            pipe.done[slot].synchronize()
            pipe.res_dev[slot] = None
            r0, r1, rc = pipe.res[slot]
            c = rc.tolist()
            self._check_counts(c, "match_xfeat_stream")
            a0, a1 = r0.numpy(), r1.numpy()              # one view per buffer, one copy per pair and side
            return [(a0[b, :c[b]].copy(), a1[b, :c[b]].copy()) for b in range(len(c))]

        try:
            nxt = next(it)
        except StopIteration:
            return
        cur = self._upload(pipe, 0, nxt)
        i, pending = 0, None
        while cur is not None:
            slot = i & 1
            try:
                nxt = next(it)
                nxt_dev = self._upload(pipe, slot ^ 1, nxt)       # overlaps the kernels queued below
            except StopIteration:
                nxt_dev = None
            main.wait_event(pipe.ready[slot])
            (x1, f1), (x2, f2) = cur
            mk0, mk1, cnt = self._match_sparse_batch_device(x1, x2, top_k, min_cossim, div255=(f1, f2))
            pipe.freed[slot].record(main)
            B = mk0.shape[0]
            res = pipe.res[slot]
            if res is None or res[0].shape != mk0.shape:
                res = (torch.empty(mk0.shape, dtype=torch.float32, pin_memory=True),
                       torch.empty(mk1.shape, dtype=torch.float32, pin_memory=True),
                       torch.empty((B,), dtype=torch.int32, pin_memory=True))
                pipe.res[slot] = res
            pipe.computed[slot].record(main)
            pipe.res_dev[slot] = (mk0, mk1, cnt)
            out_stream = main if _D2H_ON_MAIN else pipe.d2h
            with torch.cuda.stream(out_stream):
                out_stream.wait_event(pipe.computed[slot])
                res[0].copy_(mk0, non_blocking=True)
                res[1].copy_(mk1, non_blocking=True)
                res[2].copy_(cnt, non_blocking=True)
                pipe.done[slot].record(out_stream)
            if pending is not None:
                yield finish(pending)
            pending = slot
            cur = nxt_dev
            i += 1
        if pending is not None:
            yield finish(pending)

    # ------------------------------------------------------------------------------------------------------------
    # pair lists over a shared set of images: every referenced image is extracted once
    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _pair_image(x):
        """One image of match_xfeat_pairs as _host_batch takes it (numpy (H,W) -> (H,W,1))."""
        return x[:, :, None] if isinstance(x, np.ndarray) and x.ndim == 2 else x

    def _extract_table(self, images, plan: PairPlan, top_k: int, want_split: bool, want_desc: bool) -> Dict[str, torch.Tensor]:
        """Sparse extraction of every planned image into one table (row = slot): keypoints (n, top_k, 2), n_valid (n) and the
        descriptors (n, top_k, 64) and / or operand rows (n, split_rows, 128).  No host sync."""
        n = plan.n_slots
        tab = {"keypoints": self._empty((n, top_k, 2)), "n_valid": self._empty((n,), torch.int32)}
        if want_desc:
            tab["descriptors"] = self._empty((n, top_k, 64))
        if want_split:
            tab["desc_split"] = self._empty((n, self._split_rows(top_k), 128), torch.float16)

        def step(cur, out):
            self._detect_sparse_device([x for x, _ in cur], top_k, self.detection_threshold, [f for _, f in cur],
                                       want_split=want_split, want_desc=want_desc, out=out)
        return self._fill_table(images, plan, tab, step)

    def _fill_table(self, images, plan: PairPlan, tab: Dict[str, torch.Tensor], step) -> Dict[str, torch.Tensor]:
        """Run `step(batches, out)` over the plan's chunks: `batches` is the chunk's images on the device, [((1,C,H,W) tensor,
        div255)] of one bucket, and `out` = {name: table[s0:s1]} the chunk's slots of every table in `tab`.  The chunks go
        through match_xfeat_stream's copy pipeline: chunk c+1 is uploaded on the copy stream while chunk c is extracted."""
        if self._pipe is None:
            self._pipe = XFeat._Pipe(self.dev)
        pipe = self._pipe
        main = torch.cuda.current_stream(self.dev)
        for ev in pipe.freed:
            ev.record(main)

        def upload(c: int, slot: int):
            return self._upload(pipe, slot, [self._pair_image(images[i]) for i in plan.chunks[c]])

        cur, s0 = upload(0, 0), 0
        for c, chunk in enumerate(plan.chunks):
            slot = c & 1
            nxt = upload(c + 1, slot ^ 1) if c + 1 < len(plan.chunks) else None     # overlaps the kernels queued below
            main.wait_event(pipe.ready[slot])
            s1 = s0 + len(chunk)
            step(cur, {k: v[s0:s1] for k, v in tab.items()})
            pipe.freed[slot].record(main)
            cur, s0 = nxt, s1
        return tab

    def _mnn_pairs_device(self, tab, tp: torch.Tensor, top_k: int, min_cossim: float, ws: Optional[torch.Tensor] = None):
        """xfeat_mnn_match_pairs on the table's operand rows for the (B, 2) int32 device pair table `tp`.  `ws`: see _run_net."""
        B = tp.shape[0]
        sp = tab["desc_split"]
        idx0 = self._empty((B, top_k), torch.int64)
        idx1 = self._empty((B, top_k), torch.int64)
        cnt = self._empty((B,), torch.int32)
        if ws is None:
            ws = self._workspace(self._lib.xfeat_mnn_pairs_workspace_bytes(B, top_k))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_mnn_match_pairs(sp.data_ptr(), tab["n_valid"].data_ptr(), sp.shape[0], top_k, sp.shape[1],
                                                       tp.data_ptr(), B, 13, float(min_cossim), idx0.data_ptr(), idx1.data_ptr(),
                                                       cnt.data_ptr(), ws.data_ptr(), ws.numel(), self._stream()),
                       "xfeat_mnn_match_pairs")
        return idx0, idx1, cnt

    def _match_table_pairs(self, tab, tp: torch.Tensor, top_k: int, min_cossim: float, presplit: bool,
                           ws: Optional[torch.Tensor] = None):
        """MNN + keypoint gather of the (B, 2) int32 device pair table `tp` over an _extract_table table: xfeat_mnn_match_pairs
        on its operand rows (`presplit`), else xfeat_mnn_match_bounded on its fp32 descriptors gathered per pair.  Returns mkpts0,
        mkpts1 (B, top_k, 2) and n_matches (B) int32 (XF_N_OVERFLOW for a pair with an overflowed image).  No host sync.
        `ws`: see _run_net."""
        B = tp.shape[0]
        if presplit:
            idx0, idx1, cnt = self._mnn_pairs_device(tab, tp, top_k, min_cossim, ws=ws)
        else:
            ti, tj = tp[:, 0].long(), tp[:, 1].long()
            d, n = tab["descriptors"], tab["n_valid"]
            idx0, idx1, cnt = self._mnn_device(d.index_select(0, ti), n.index_select(0, ti), top_k, top_k * 64,
                                               d.index_select(0, tj), n.index_select(0, tj), top_k, top_k * 64, B, min_cossim,
                                               abs_bound=1.0, ws=ws)
        mk0, mk1 = self._empty((B, top_k, 2)), self._empty((B, top_k, 2))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_gather_matches_pairs(tab["keypoints"].data_ptr(), top_k, tp.data_ptr(), idx0.data_ptr(),
                                                            idx1.data_ptr(), cnt.data_ptr(), B, mk0.data_ptr(), mk1.data_ptr(),
                                                            self._stream()), "xfeat_gather_matches_pairs")
        return mk0, mk1, cnt

    @staticmethod
    def _pair_labels(plan: PairPlan, sel: np.ndarray) -> List[str]:
        return [f"pair {p} (images {plan.pairs[p, 0]}, {plan.pairs[p, 1]})" for p in sel.tolist()]

    @torch.inference_mode()
    def match_xfeat_pairs(self, images, pairs, top_k=None, min_cossim=-1) -> List[Tuple[np.ndarray, np.ndarray]]:
        """match_xfeat over a list of pairs into one set of images: result p is what match_xfeat(images[i], images[j], top_k,
        min_cossim) returns for pairs[p] = (i, j), bit for bit -- self pairs, repeated pairs and both orders included.

        images: sequence of single images in any mix of shapes and types -- numpy (H,W) / (H,W,C), uint8 or float, or torch
        (C,H,W) / (1,C,H,W) on the host or the device (numpy (H,W) is read as (H,W,1)).  pairs: (P, 2) array-like of ints.
        Only images some pair names are extracted, each exactly once, in launch sequences of up to 64 images of one
        (C, H, W, dtype, "/255") bucket; the pairs are then matched straight from the shared table, up to 4096 per launch."""
        if top_k is None: top_k = self.top_k
        plan = PairPlan([pair_image_key(x) for x in images], pairs)
        if len(plan.pairs) == 0:
            return []
        return self._pairs_matched(images, plan, top_k, min_cossim, "match_xfeat_pairs")

    @torch.inference_mode()
    def match_xfeat_verified_pairs(self, images, pairs, top_k=None, min_cossim=-1, ransac_thr: float = 3.0, iters: int = 2048,
                                   seed: int = 0) -> List[Dict[str, np.ndarray]]:
        """match_xfeat_pairs (same inputs, same extraction, same matches bit for bit) followed, still on the device, by the
        fundamental-matrix RANSAC of geometry.find_fundamental_batch on every pair: the cv2.findFundamentalMat(mkpts0, mkpts1,
        cv2.USAC_MAGSAC, ransac_thr) step that pair lists from photo collections run next.  Result p: {'mkpts0', 'mkpts1' (N,2),
        'inliers' (N,) bool, 'n_inliers' int, 'F' (3,3) float64 with x1^T F x0 = 0 in pixels, or None when fewer than 8 inliers
        support it}.  Pair p's samples are seeded by (seed, p), so its result is what find_fundamental_batch gives its matches
        alone with pair_ids=[p].  One host synchronisation per chunk of pairs.  top_k above 8192 is refused."""
        if top_k is None: top_k = self.top_k
        if top_k > 8192:
            raise ValueError(f"match_xfeat_verified_pairs: top_k {top_k} > 8192 (the RANSAC caches at most 8192 matches per pair)")
        plan = PairPlan([pair_image_key(x) for x in images], pairs)
        if len(plan.pairs) == 0:
            return []
        return self._pairs_matched(images, plan, top_k, min_cossim, "match_xfeat_verified_pairs", (ransac_thr, iters, seed))

    def _pairs_matched(self, images, plan: PairPlan, top_k: int, min_cossim: float, what: str, ransac=None) -> List:
        """The body of match_xfeat_pairs over a non-empty plan, and with `ransac` = (thr, iters, seed) that of
        match_xfeat_verified_pairs: each chunk's matches go through find_fundamental_batch on the device before the chunk's one
        host sync."""
        presplit = self._lib.xfeat_get_mnn_impl() in (1, 2, 3)   # else: fp32 descriptors, per-pair gather, xfeat_mnn_match_bounded
        order = plan.match_order()
        tp_all = torch.from_numpy(np.ascontiguousarray(plan.table_pairs[order])).to(self.dev)
        ids_all = torch.from_numpy(order.astype(np.int32)).to(self.dev) if ransac else None    # match_order() reorders the pairs
        tab = self._extract_table(images, plan, top_k, want_split=presplit, want_desc=not presplit)
        out: List = [None] * len(order)
        step = PAIRS_MATCH_CHUNK if presplit else 256              # the fp32 fallback gathers (B, top_k, 64) per side
        for o in range(0, len(order), step):
            sel, tp = order[o:o + step], tp_all[o:o + step]
            B = len(sel)
            mk0, mk1, cnt = self._match_table_pairs(tab, tp, top_k, min_cossim, presplit)
            dev_out = [mk0, mk1, cnt]
            if ransac:
                from .geometry import find_fundamental_batch
                F, mask, n_inl = find_fundamental_batch(mk0, mk1, cnt, ransac[0], ransac[1], ransac[2], pair_ids=ids_all[o:o + step])
                dev_out += [F, mask, n_inl]
            host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in dev_out]
            for h, t in zip(host, dev_out):
                h.copy_(t, non_blocking=True)
            torch.cuda.current_stream(self.dev).synchronize()         # the only host sync of this chunk
            c = host[2].tolist()
            self._check_counts(c, what, self._pair_labels(plan, sel))
            a0, a1 = host[0].numpy(), host[1].numpy()
            if not ransac:
                for b, p in enumerate(sel.tolist()):
                    out[p] = (a0[b, :c[b]].copy(), a1[b, :c[b]].copy())
                continue
            Fh, mh, nh = host[3].numpy(), host[4].numpy(), host[5].tolist()
            for b, p in enumerate(sel.tolist()):
                out[p] = {"mkpts0": a0[b, :c[b]].copy(), "mkpts1": a1[b, :c[b]].copy(), "inliers": mh[b, :c[b]].copy(),
                          "n_inliers": nh[b], "F": Fh[b].astype(np.float64) if nh[b] >= 8 else None}
        return out

    @torch.inference_mode()
    def match_xfeat_lighterglue_pairs(self, images, pairs, top_k=None, min_conf: float = 0.1,
                                      prune_min_points: Optional[int] = LG_PRUNE_MIN_POINTS) -> List[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        """match_xfeat_lighterglue_batch over a list of pairs into one set of images (inputs as match_xfeat_pairs): result p equals
        match_xfeat_lighterglue_batch on (images[i], images[j]) alone.  Each referenced image is extracted once; the pairs' sides
        are gathered from the table on the device, up to 256 pairs per LighterGlue launch."""
        if top_k is None: top_k = self.top_k
        keys = [pair_image_key(x) for x in images]
        plan = PairPlan(keys, pairs)
        if len(plan.pairs) == 0:
            return []
        self._lg()                                                  # weights load before any extraction is queued
        tab = self._extract_table(images, plan, top_k, want_split=False, want_desc=True)
        used = np.nonzero(plan.slot >= 0)[0]
        sizes = np.zeros((plan.n_slots, 2), np.float32)
        sizes[plan.slot[used]] = [(keys[i][2], keys[i][1]) for i in used]            # (W, H) of the image as given
        sizes = torch.from_numpy(sizes).to(self.dev)
        out: List = [None] * len(plan.pairs)
        step = 256
        for o in range(0, len(plan.pairs), step):
            sel = np.arange(o, min(o + step, len(plan.pairs)))
            tp = torch.from_numpy(plan.table_pairs[sel].astype(np.int64)).to(self.dev)
            side = [{k: tab[k].index_select(0, tp[:, s]) for k in ("keypoints", "descriptors", "n_valid")} for s in (0, 1)]
            s0, s1 = sizes.index_select(0, tp[:, 0]), sizes.index_select(0, tp[:, 1])
            k0, k1 = side[0]["keypoints"], side[1]["keypoints"]
            idx0, idx1, _, cnt = self.match_lighterglue_batch(k0, side[0]["descriptors"], side[0]["n_valid"], s0, k1,
                                                              side[1]["descriptors"], side[1]["n_valid"], s1, min_conf,
                                                              prune_min_points)
            B = len(sel)
            mk0, mk1, cnt = self._gather_matches(k0, k1, idx0, idx1, cnt, B, top_k)
            c = cnt.tolist()
            self._check_counts(c, "match_xfeat_lighterglue_pairs", self._pair_labels(plan, sel))
            mk0, mk1, i0, i1 = (t.cpu().numpy() for t in (mk0, mk1, idx0, idx1))
            for b, p in enumerate(sel.tolist()):
                out[p] = (mk0[b, :c[b]], mk1[b, :c[b]], np.stack([i0[b, :c[b]], i1[b, :c[b]]], -1))
        return out

    # ------------------------------------------------------------------------------------------------------------
    # semi-dense path
    # ------------------------------------------------------------------------------------------------------------
    def _extract_dense_into(self, x: torch.Tensor, div255: bool, top_k: int, div_scale: float, scale_value: float,
                            out_rows: int, out_offset: int, kpts, desc, scales, pre_scale: Optional[float] = None):
        """extractDense (xfeat.py:356-377) writing k rows at `out_offset`; returns k.  `pre_scale` = s: `x` is the ORIGINAL image and
        extract_dualscale's F.interpolate(scale_factor=s) (xfeat.py:380-381) is folded into the gray conversion -- only used when
        floor(H*s), floor(W*s) are multiples of 32, where preprocess_tensor's own resize is the identity."""
        B, _, Hi, Wi = x.shape
        if pre_scale is not None:
            Hi, Wi = int(math.floor(Hi * pre_scale)), int(math.floor(Wi * pre_scale))
        H, W = (Hi // 32) * 32, (Wi // 32) * 32
        if H == 0 or W == 0:
            raise RuntimeError("image smaller than 32 pixels")
        rh, rw = Hi / H, Wi / W
        xn = self._preprocess(x, H, W, div255, scale=None if pre_scale is None else 1.0 / pre_scale)
        feats, _, rel, _ = self._run_net(xn, B, H, W)
        cells = (H // 8) * (W // 8)
        k = min(cells, top_k)
        ws = self._workspace(self._lib.xfeat_dense_workspace_bytes(B, H, W, top_k))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_detect_dense(self._ctx, feats.data_ptr(), rel.data_ptr(), B, H, W, top_k,
                                                    float(_F32(rw)), float(_F32(rh)), float(_F32(div_scale)),
                                                    float(_F32(scale_value)), out_rows, out_offset, kpts.data_ptr(),
                                                    desc.data_ptr(), _ptr(scales), None, ws.data_ptr(), ws.numel(),
                                                    self._stream()), "xfeat_detect_dense")
        return k

    def _resize(self, x: torch.Tensor, div255: bool, Ho: int, Wo: int, inv_h: float, inv_w: float) -> torch.Tensor:
        """Bilinear resize, align_corners=False, source coordinate (dst + 0.5) * inv - 0.5 (ATen upsample_bilinear2d)."""
        x, code = self._img_args(x)
        B, C, Hi, Wi = x.shape
        out = self._empty((B, C, Ho, Wo))
        sb, sc, sh, sw = x.stride()
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_resize_bilinear(x.data_ptr(), code, B, C, Hi, Wi, sb, sc, sh, sw, int(div255),
                                                       out.data_ptr(), Ho, Wo, float(_F32(inv_h)), float(_F32(inv_w)),
                                                       self._stream()), "xfeat_resize_bilinear")
        return out

    def _resize_scale(self, x: torch.Tensor, div255: bool, s: float) -> torch.Tensor:
        """F.interpolate(x, scale_factor=s, mode='bilinear', align_corners=False) (xfeat.py:380-381)."""
        Hi, Wi = x.shape[-2:]
        return self._resize(x, div255, int(math.floor(Hi * s)), int(math.floor(Wi * s)), 1.0 / s, 1.0 / s)

    def _dense_device(self, x, top_k: int, multiscale: bool, div255: bool = False, s1: float = 0.6, s2: float = 1.3,
                      out: Optional[Dict[str, torch.Tensor]] = None):
        """`out` (multiscale): write 'keypoints', 'descriptors' and 'scales' into these (B, K_max, ...) tensors, e.g. slices of
        an image table with K_max >= k1 + k2 rows per image, instead of fresh (B, k1 + k2, ...) ones; rows past k1 + k2 are not
        written."""
        x = self._to_bchw(x)
        B, _, Hi, Wi = x.shape
        if multiscale:
            k1, k2 = dense_counts(Hi, Wi, top_k, s1, s2)
            if out is None:
                K = k1 + k2
                kpts, desc, scales = self._empty((B, K, 2)), self._empty((B, K, 64)), self._empty((B, K))
            else:
                kpts, desc, scales = out["keypoints"], out["descriptors"], out["scales"]
                K = kpts.shape[1]
            for s, k, off in ((s1, k1, 0), (s2, k2, k1)):
                Hs, Ws = int(math.floor(Hi * s)), int(math.floor(Wi * s))
                if Hs % 32 == 0 and Ws % 32 == 0:
                    # the 3-channel resized image (1.6 GB per 64 x 1280x960 at s = 1.3) is never written: resize + gray in one pass
                    self._extract_dense_into(x, div255, k, s, 1 / s, K, off, kpts, desc, scales, pre_scale=s)
                else:
                    xs = self._resize_scale(x, div255, s)
                    self._extract_dense_into(xs, False, k, s, 1 / s, K, off, kpts, desc, scales)
                    del xs
        else:
            K = min(_dense_cells(Hi, Wi), _dense_cap(top_k))
            kpts, desc, scales = self._empty((B, K, 2)), self._empty((B, K, 64)), self._empty((B, K))
            self._extract_dense_into(x, div255, K, 1.0, 1.0, K, 0, kpts, desc, scales)
        return {"keypoints": kpts, "descriptors": desc, "scales": scales}

    @torch.inference_mode()
    def detectAndComputeDense(self, x, top_k=None, multiscale=True) -> Dict[str, torch.Tensor]:
        """Dense *coarse* descriptors, batched (reference: xfeat.py:105-128): dict of 'keypoints' (B,K,2),
        'descriptors' (B,K,64) un-normalised, 'scales' (B,K); sorted by reliability per scale."""
        if top_k is None: top_k = self.top_k
        return self._dense_device(x, top_k, multiscale)

    def _refine_device(self, d0, d1, idx0, idx1, cnt, fine_conf: float = 0.25):
        B, K0, _ = d0["descriptors"].shape
        K1 = d1["descriptors"].shape[1]
        matches = self._empty((B, K0, 4))
        n_ref = self._empty((B,), torch.int32)
        ws = self._workspace(self._lib.xfeat_refine_workspace_bytes(B, K0))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_refine(self._ctx, d0["descriptors"].data_ptr(), d1["descriptors"].data_ptr(),
                                              d0["keypoints"].data_ptr(), d1["keypoints"].data_ptr(),
                                              d0["scales"].data_ptr(), idx0.data_ptr(), idx1.data_ptr(), cnt.data_ptr(),
                                              B, K0, K1, float(fine_conf), matches.data_ptr(), n_ref.data_ptr(),
                                              ws.data_ptr(), ws.numel(), self._stream()), "xfeat_refine")
        return matches, n_ref

    def _match_star_device(self, im_set1, im_set2, top_k: int, div255=False):
        da, db = (div255 if isinstance(div255, (list, tuple)) else (div255, div255))
        if (isinstance(im_set2, torch.Tensor) and not im_set2.is_cuda and im_set2.dim() == 4
                and isinstance(im_set1, torch.Tensor) and not im_set1.is_cuda):
            # host inputs: the second set travels on the copy stream while the first set is being extracted
            if self._pipe is None:
                self._pipe = XFeat._Pipe(self.dev)
            main, copy = torch.cuda.current_stream(self.dev), self._pipe.copy
            x1 = im_set1.to(self.dev, non_blocking=True)
            x2 = torch.empty_like(im_set2, device=self.dev)       # from the compute stream's pool (it is read there)
            start, done = torch.cuda.Event(), torch.cuda.Event()
            start.record(main)
            with torch.cuda.stream(copy):
                copy.wait_event(start)                            # (the block may still be in use by earlier kernels)
                x2.copy_(im_set2, non_blocking=True)
                done.record(copy)
            o1 = self._dense_device(x1, top_k, True, da)
            main.wait_event(done)
            im_set1, im_set2 = x1, x2
            o2 = self._dense_device(x2, top_k, True, db)
        else:
            o1 = self._dense_device(im_set1, top_k, True, da)
            o2 = self._dense_device(im_set2, top_k, True, db)
        B, K0, _ = o1["descriptors"].shape
        K1 = o2["descriptors"].shape[1]
        if o2["descriptors"].shape[0] != B:
            raise RuntimeError("match_xfeat_star needs both image sets at the same batch size")
        idx0, idx1, cnt = self._mnn_device(o1["descriptors"], None, K0, K0 * 64, o2["descriptors"], None, K1, K1 * 64, B, -1)
        return self._refine_device(o1, o2, idx0, idx1, cnt)

    @torch.inference_mode()
    def match_xfeat_star(self, im_set1, im_set2, top_k=None):
        """Semi-dense matching with refinement, batched (reference: xfeat.py:188-217).
        B > 1 -> List[Tensor (N,4)] (x1,y1,x2,y2) on device; B == 1 -> two np.ndarray (N,2)."""
        if top_k is None: top_k = self.top_k
        im_set1, d1 = self._parse_input(im_set1)
        im_set2, d2 = self._parse_input(im_set2)
        matches, n_ref = self._match_star_device(im_set1, im_set2, top_k, div255=(d1, d2))
        n = n_ref.tolist()
        out = [matches[b, :n[b]] for b in range(len(n))]
        return out if len(n) > 1 else (out[0][:, :2].cpu().numpy(), out[0][:, 2:].cpu().numpy())

    def _mnn_pairs_f32_device(self, tab, rows: torch.Tensor, tp: torch.Tensor, k_max: int):
        """xfeat_mnn_match_pairs_f32 on the dense table's descriptors for the (B, 2) int32 device pair table `tp`."""
        B = tp.shape[0]
        idx0 = self._empty((B, k_max), torch.int64)
        idx1 = self._empty((B, k_max), torch.int64)
        cnt = self._empty((B,), torch.int32)
        ws = self._workspace(self._lib.xfeat_mnn_pairs_f32_workspace_bytes(B, k_max))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_mnn_match_pairs_f32(tab["descriptors"].data_ptr(), rows.data_ptr(), rows.shape[0], k_max,
                                                           tp.data_ptr(), B, idx0.data_ptr(), idx1.data_ptr(), cnt.data_ptr(),
                                                           ws.data_ptr(), ws.numel(), self._stream()), "xfeat_mnn_match_pairs_f32")
        return idx0, idx1, cnt

    def _refine_pairs_device(self, tab, tp: torch.Tensor, idx0, idx1, cnt, k_max: int, fine_conf: float = 0.25):
        B = tp.shape[0]
        matches = self._empty((B, k_max, 4))
        n_ref = self._empty((B,), torch.int32)
        ws = self._workspace(self._lib.xfeat_refine_pairs_workspace_bytes(B, k_max))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_refine_pairs(self._ctx, tab["descriptors"].data_ptr(), tab["keypoints"].data_ptr(),
                                                    tab["scales"].data_ptr(), k_max, tp.data_ptr(), idx0.data_ptr(),
                                                    idx1.data_ptr(), cnt.data_ptr(), B, float(fine_conf), matches.data_ptr(),
                                                    n_ref.data_ptr(), ws.data_ptr(), ws.numel(), self._stream()),
                       "xfeat_refine_pairs")
        return matches, n_ref

    @torch.inference_mode()
    def match_xfeat_star_pairs(self, images, pairs, top_k=None) -> List[Tuple[np.ndarray, np.ndarray]]:
        """match_xfeat_star over a list of pairs into one set of images (inputs as match_xfeat_pairs): result p is what
        match_xfeat_star(images[i], images[j], top_k) returns for pairs[p] = (i, j), bit for bit -- self pairs, repeated pairs
        and both orders included.

        Only images some pair names are extracted, each exactly once per scale, in launch sequences of up to 64 images of one
        bucket, into one dense table of K_max rows per image.  The pairs are then matched and refined straight from the table, as
        many per launch as fit in STAR_PAIRS_MATCH_BYTES, with one host synchronisation per chunk.  The matcher splits every pair's
        operands at the exponent of its own two images' max |x|, as the single-pair call does; under matcher implementations 0
        and 4 each pair goes through the fp32-input matcher on its two table slots instead."""
        if top_k is None: top_k = self.top_k
        keys = [pair_image_key(x) for x in images]
        plan = PairPlan(keys, pairs, PAIRS_EXTRACT_CHUNK)
        if len(plan.pairs) == 0:
            return []
        rows = star_pair_rows(keys, plan, top_k)                    # refuses a too-small image before anything is launched
        k_max = int(rows.max())
        presplit = self._lib.xfeat_get_mnn_impl() in (1, 2, 3)
        order = plan.match_order()
        tp_all = torch.from_numpy(np.ascontiguousarray(plan.table_pairs[order])).to(self.dev)
        rows_dev = torch.from_numpy(rows).to(self.dev)
        n = plan.n_slots
        tab = {"keypoints": self._empty((n, k_max, 2)), "descriptors": self._empty((n, k_max, 64)), "scales": self._empty((n, k_max))}

        def step(cur, out):       # one bucket: one shape, dtype and "/255" flag
            x = cur[0][0] if len(cur) == 1 else torch.cat([t for t, _ in cur])
            self._dense_device(x, top_k, True, cur[0][1], out=out)
        self._fill_table(images, plan, tab, step)

        out: List = [None] * len(order)
        for o0, o1 in star_match_chunks(len(order), k_max):
            sel, tp = order[o0:o1], tp_all[o0:o1]
            B = len(sel)
            if presplit:
                idx0, idx1, cnt = self._mnn_pairs_f32_device(tab, rows_dev, tp, k_max)
            else:
                idx0 = self._empty((B, k_max), torch.int64)
                idx1 = self._empty((B, k_max), torch.int64)
                cnt = self._empty((B,), torch.int32)
                d = tab["descriptors"]
                for b, (si, sj) in enumerate(plan.table_pairs[sel].tolist()):
                    ki, kj = int(rows[si]), int(rows[sj])
                    i0, i1, c = self._mnn_device(d[si], None, ki, ki * 64, d[sj], None, kj, kj * 64, 1, -1)
                    idx0[b, :ki] = i0[0]
                    idx1[b, :ki] = i1[0]
                    cnt[b:b + 1] = c
            matches, n_ref = self._refine_pairs_device(tab, tp, idx0, idx1, cnt, k_max)
            hm = torch.empty(matches.shape, dtype=torch.float32, pin_memory=True)
            hn = torch.empty((B,), dtype=torch.int32, pin_memory=True)
            hm.copy_(matches, non_blocking=True)
            hn.copy_(n_ref, non_blocking=True)
            torch.cuda.current_stream(self.dev).synchronize()         # the only host sync of this chunk
            c = hn.tolist()
            m = hm.numpy()
            for b, p in enumerate(sel.tolist()):
                out[p] = (m[b, :c[b], :2].copy(), m[b, :c[b], 2:].copy())
        return out

    # ------------------------------------------------------------------------------------------------------------
    # LighterGlue matching (csrc/lighterglue.cu)
    # ------------------------------------------------------------------------------------------------------------
    def _lg(self) -> "_LighterGlue":
        if self.lighterglue is None:                    # loaded on first use, as the reference does (xfeat.py:143-145)
            self.lighterglue = _LighterGlue(self, self._lighterglue_weights)
        return self.lighterglue

    @torch.inference_mode()
    def match_lighterglue_batch(self, kpts0, desc0, n0, size0, kpts1, desc1, n1, size1, min_conf: float = 0.1,
                                prune_min_points: Optional[int] = LG_PRUNE_MIN_POINTS):
        """LighterGlue on B pairs of fixed-capacity device inputs, no host sync.  kpts (B,n_max,2) pixel (x,y), desc (B,n_max,64),
        n (B) int32 point counts, size (B,2) image size (W,H); the two sides share n_max.  `prune_min_points`: an image with more
        points than this is pruned after layers 0..4 (LightGlue's point pruning, width_confidence 0.95); None disables pruning.
        Returns device tensors idx0 (ascending), idx1 (B,n_max) int64, scores (B,n_max), n_matches (B) int32."""
        lg = self._lg()
        t = lambda x, dt: x.to(self.dev, dt).contiguous()       # noqa: E731
        kpts0, kpts1, desc0, desc1 = (t(x, torch.float32) for x in (kpts0, kpts1, desc0, desc1))
        size0, size1 = t(torch.as_tensor(size0), torch.float32), t(torch.as_tensor(size1), torch.float32)
        n0, n1 = t(torch.as_tensor(n0), torch.int32), t(torch.as_tensor(n1), torch.int32)
        B, n_max = kpts0.shape[:2]
        if (kpts1.shape != (B, n_max, 2) or kpts0.shape != (B, n_max, 2) or desc0.shape != (B, n_max, 64)
                or desc1.shape != (B, n_max, 64) or size0.shape != (B, 2) or size1.shape != (B, 2)
                or n0.shape != (B,) or n1.shape != (B,)):
            raise RuntimeError("match_lighterglue_batch: kpts (B,n_max,2), desc (B,n_max,64), n (B), size (B,2) on both sides")
        idx0 = self._empty((B, n_max), torch.int64)
        idx1 = self._empty((B, n_max), torch.int64)
        scores = self._empty((B, n_max))
        cnt = self._empty((B,), torch.int32)
        ws = self._workspace(self._lib.xfeat_lg_workspace_bytes(B, n_max))
        T = -1 if prune_min_points is None else int(prune_min_points)
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_lg_match(lg.ctx, B, n_max, kpts0.data_ptr(), desc0.data_ptr(), n0.data_ptr(), size0.data_ptr(),
                                                kpts1.data_ptr(), desc1.data_ptr(), n1.data_ptr(), size1.data_ptr(), float(min_conf),
                                                T, idx0.data_ptr(), idx1.data_ptr(), scores.data_ptr(), cnt.data_ptr(),
                                                ws.data_ptr(), ws.numel(), self._stream()), "xfeat_lg_match")
        return idx0, idx1, scores, cnt

    @torch.inference_mode()
    def match_lighterglue(self, d0, d1, min_conf=0.1, prune_min_points: Optional[int] = LG_PRUNE_MIN_POINTS):
        """Match XFeat sparse features with LighterGlue (reference: xfeat.py:131-162).
        d0, d1: dicts with 'keypoints' (N,2), 'descriptors' (N,64), 'image_size' (W,H).
        Returns mkpts_0, mkpts_1 (N,2) and idx (N,2) int64 as np.ndarray."""
        k0, k1 = d0["keypoints"].to(self.dev).float(), d1["keypoints"].to(self.dev).float()
        n0, n1 = len(k0), len(k1)
        n_max = max(n0, n1, 1)

        def pad(x, n, c):
            out = torch.zeros((1, n_max, c), dtype=torch.float32, device=self.dev)
            out[0, :n] = x.to(self.dev).float().reshape(n, c)
            return out
        idx0, idx1, _, cnt = self.match_lighterglue_batch(
            pad(k0, n0, 2), pad(d0["descriptors"], n0, 64), torch.tensor([n0]), torch.tensor([list(d0["image_size"])]),
            pad(k1, n1, 2), pad(d1["descriptors"], n1, 64), torch.tensor([n1]), torch.tensor([list(d1["image_size"])]),
            min_conf, prune_min_points)
        n = int(cnt.item())
        i0, i1 = idx0[0, :n], idx1[0, :n]
        return k0[i0].cpu().numpy(), k1[i1].cpu().numpy(), torch.stack([i0, i1], -1).cpu().numpy()

    @torch.inference_mode()
    def match_xfeat_lighterglue_batch(self, imgs1, imgs2, top_k=None, min_conf: float = 0.1,
                                      prune_min_points: Optional[int] = LG_PRUNE_MIN_POINTS) -> List[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        """detectAndCompute on both image sets, LighterGlue on every pair b = (imgs1[b], imgs2[b]) and the keypoint gather, all
        on the device with one host synchronisation.  Returns per pair (mkpts_0, mkpts_1, idx (N,2)) as match_lighterglue does."""
        if top_k is None: top_k = self.top_k
        x1, da = self._parse_input(imgs1)
        x2, db = self._parse_input(imgs2)
        x1, x2 = self._to_bchw(x1), self._to_bchw(x2)
        B = x1.shape[0]
        if x2.shape[0] != B:
            raise RuntimeError("the two image sets must have the same batch size")
        if x1.shape[1:] == x2.shape[1:]:
            o = self._detect_sparse_device([x1, x2], top_k, self.detection_threshold, [da, db])
            k0, k1, d0, d1 = o["keypoints"][:B], o["keypoints"][B:], o["descriptors"][:B], o["descriptors"][B:]
            n0, n1 = o["n_valid"][:B], o["n_valid"][B:]
        else:
            o1 = self._detect_sparse_device(x1, top_k, self.detection_threshold, da)
            o2 = self._detect_sparse_device(x2, top_k, self.detection_threshold, db)
            k0, k1, d0, d1, n0, n1 = (o1["keypoints"], o2["keypoints"], o1["descriptors"], o2["descriptors"], o1["n_valid"],
                                      o2["n_valid"])
        size0 = torch.tensor([[x1.shape[3], x1.shape[2]]] * B, dtype=torch.float32)
        size1 = torch.tensor([[x2.shape[3], x2.shape[2]]] * B, dtype=torch.float32)
        idx0, idx1, _, cnt = self.match_lighterglue_batch(k0, d0, n0, size0, k1, d1, n1, size1, min_conf, prune_min_points)
        mk0, mk1, cnt = self._gather_matches(k0, k1, idx0, idx1, cnt, B, top_k)
        c = cnt.tolist()                                              # the only host sync
        self._check_counts(c, "match_xfeat_lighterglue_batch")
        mk0, mk1, i0, i1 = (t.cpu().numpy() for t in (mk0, mk1, idx0, idx1))
        return [(mk0[b, :c[b]], mk1[b, :c[b]], np.stack([i0[b, :c[b]], i1[b, :c[b]]], -1)) for b in range(B)]

    # ------------------------------------------------------------------------------------------------------------
    # the reference's helper methods, each through its own kernel of the library
    # ------------------------------------------------------------------------------------------------------------
    @torch.inference_mode()
    def preprocess_tensor(self, x):
        """Guarantee that image is divisible by 32 (reference: xfeat.py:219-240) -> (x (B,C,_H,_W) float, rh, rw)."""
        x = self._to_bchw(x)
        H, W = x.shape[-2:]
        _H, _W = (H // 32) * 32, (W // 32) * 32
        if _H == 0 or _W == 0:
            raise RuntimeError("image smaller than 32 pixels")
        rh, rw = H / _H, W / _W
        return self._resize(x, False, _H, _W, H / _H, W / _W), rh, rw

    @torch.inference_mode()
    def get_kpts_heatmap(self, kpts, softmax_temp=1.0):
        """(B,65,H/8,W/8) keypoint logits -> (B,1,H,W) heat-map (reference: xfeat.py:242-247)."""
        k = kpts.to(self.dev).float().contiguous()
        B, C, Hc, Wc = k.shape
        if C != 65:
            raise RuntimeError("keypoint logits must have 65 channels")
        heat = self._empty((B, 1, Hc * 8, Wc * 8))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_kpts_heatmap(k.data_ptr(), B, Hc, Wc, float(softmax_temp), heat.data_ptr(), self._stream()),
                       "xfeat_kpts_heatmap")
        return heat

    @torch.inference_mode()
    def NMS(self, x, threshold=0.05, kernel_size=5):
        """(B,1,H,W) heat-map -> (B,N,2) int64 (x,y) of the local maxima above threshold, raster order, zero padded to the
        batch maximum (reference: xfeat.py:249-263)."""
        h = x.to(self.dev).float().contiguous()
        B, _, H, W = h.shape
        ws = self._workspace(self._lib.xfeat_nms_workspace_bytes(B, H, W))
        counts = self._empty((B,), torch.int32)
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_nms_count(h.data_ptr(), B, H, W, int(kernel_size), float(threshold), counts.data_ptr(),
                                                 ws.data_ptr(), ws.numel(), self._stream()), "xfeat_nms_count")
            pad_val = max(counts.tolist())                       # the reference's nonzero() syncs here too
            pos = torch.zeros((B, pad_val, 2), dtype=torch.long, device=self.dev)
            _lib.check(self._lib.xfeat_nms_write(h.data_ptr(), B, H, W, int(kernel_size), float(threshold), pos.data_ptr(),
                                                 pad_val, ws.data_ptr(), ws.numel(), self._stream()), "xfeat_nms_write")
        return pos

    @torch.inference_mode()
    def subpix_softmax2d(self, heatmaps, temp=3):
        """(N,8,8) logits -> (N,2) expected (x,y) offset under softmax(temp * logits) (reference: xfeat.py:292-304)."""
        h = heatmaps.to(self.dev).float().contiguous()
        N, Hh, Wh = h.shape
        if (Hh, Wh) != (8, 8):
            raise RuntimeError("subpix_softmax2d is implemented for 8x8 maps (the fine matcher's output)")
        out = self._empty((N, 2))
        with torch.cuda.device(self.dev):
            _lib.check(self._lib.xfeat_subpix_softmax2d(h.data_ptr(), N, float(temp), out.data_ptr(), self._stream()),
                       "xfeat_subpix_softmax2d")
        return out

    @torch.inference_mode()
    def refine_matches(self, d0, d1, matches, batch_idx, fine_conf=0.25):
        """Refine the coarse matches of one pair (reference: xfeat.py:306-325) -> Tensor (n,4) (x1,y1,x2,y2)."""
        idx0, idx1 = matches[batch_idx]
        n = int(idx0.shape[0])
        sub0 = {k: d0[k][batch_idx:batch_idx + 1].contiguous() for k in ("descriptors", "keypoints", "scales")}
        sub1 = {k: d1[k][batch_idx:batch_idx + 1].contiguous() for k in ("descriptors", "keypoints")}
        K0 = sub0["descriptors"].shape[1]
        if n == 0:
            return self._empty((0, 4))
        if n > K0:
            raise RuntimeError("more matches than coarse features")
        i0 = torch.zeros((1, K0), dtype=torch.int64, device=self.dev)
        i1 = torch.zeros((1, K0), dtype=torch.int64, device=self.dev)
        i0[0, :n] = idx0.to(self.dev)
        i1[0, :n] = idx1.to(self.dev)
        cnt = torch.full((1,), n, dtype=torch.int32, device=self.dev)
        m, n_ref = self._refine_device(sub0, sub1, i0, i1, cnt, fine_conf)
        return m[0, :int(n_ref.item())]

    def create_xy(self, h, w, dev):
        """(h*w, 2) integer (x,y) grid, x fastest (reference: xfeat.py:350-354)."""
        y, x = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing='ij')
        return torch.cat([x[..., None], y[..., None]], -1).reshape(-1, 2)

    @torch.inference_mode()
    def extractDense(self, x, top_k=8_000):
        """Top-k most reliable 1/8-resolution cells: (mkpts (B,k,2), feats (B,k,64)) (reference: xfeat.py:356-377)."""
        o = self._dense_device(x, top_k, False)
        return o["keypoints"], o["descriptors"]

    @torch.inference_mode()
    def extract_dualscale(self, x, top_k, s1=0.6, s2=1.3):
        """Dense extraction at two scales (reference: xfeat.py:379-394) -> (mkpts, scales, feats)."""
        o = self._dense_device(x, top_k, True, False, s1, s2)
        return o["keypoints"], o["scales"], o["descriptors"]

    # ------------------------------------------------------------------------------------------------------------
    # input helpers (reference semantics)
    # ------------------------------------------------------------------------------------------------------------
    def _parse_input(self, x):
        """parse_input (xfeat.py:396-403): 3-D -> add batch dim; numpy (B,H,W,C) uint8 -> the '/255' is applied
        on the device (flag), tensors pass through un-scaled.  Returns (tensor (B,C,H,W), div255 flag)."""
        if len(x.shape) == 3:
            x = x[None, ...]
        if isinstance(x, np.ndarray):
            t = torch.from_numpy(np.ascontiguousarray(x)).permute(0, 3, 1, 2)
            if t.dtype != torch.uint8:
                return t.float() / 255, False
            return t, True
        return x, False

    def parse_input(self, x):
        """Reference-compatible parse_input (xfeat.py:396-403) returning a float tensor."""
        if len(x.shape) == 3:
            x = x[None, ...]
        if isinstance(x, np.ndarray):
            x = torch.tensor(x).permute(0, 3, 1, 2) / 255
        return x
