"""Pair lists over one image table: the kernels (xfeat_mnn_match_pairs, xfeat_gather_matches_pairs) against the per-pair presplit
matcher bit for bit, and XFeat.match_xfeat_pairs / match_xfeat_lighterglue_pairs / the sparse evaluation harness against
their per-pair public calls, bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from accelerated_features_b200 import _lib
from accelerated_features_b200 import xfeat as xfeat_mod
from tests.split_ref import split_act
from tests.test_gpu_mnn_tc import mnn_impl

pytestmark = pytest.mark.gpu

N_MAX = 4096


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    from oracle import build_lighterglue
    try:
        lg = build_lighterglue.path()
    except RuntimeError:
        lg = None
    return XFeat(device=0, lighterglue_weights=lg)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. kernels
# ---------------------------------------------------------------------------------------------------------------------------
COUNTS = [4096, 4096, 0, 1, 511, 2049, _lib.N_OVERFLOW]


@pytest.fixture(scope="module")
def table():
    """7 images: unit descriptors (image 1 a noisy copy of image 0, image 5 shares rows with image 4, so pairs have many
    matches), their operand rows [hi | lo] of desc * 2^13 (zero past the count), counts and keypoints."""
    g = torch.Generator().manual_seed(11)
    d = torch.randn(len(COUNTS), N_MAX, 64, generator=g)
    d[1] = d[0] + 0.3 * torch.randn(N_MAX, 64, generator=g)
    d[5, :511] = d[4, :511] + 0.2 * torch.randn(511, 64, generator=g)
    d = F.normalize(d, dim=-1)
    hi, lo = split_act(d * 2.0 ** 13)
    rows = torch.cat([hi, lo], -1).half()
    for i, n in enumerate(COUNTS):
        if n >= 0:
            rows[i, n:] = 0
    kpts = torch.rand(len(COUNTS), N_MAX, 2, generator=g) * 640
    return rows.cuda(), torch.tensor(COUNTS, dtype=torch.int32).cuda(), kpts.cuda()


def pair_list():
    n = len(COUNTS)
    p = [(i, j) for i in range(n) for j in range(n)]            # (i, i), both orders, every pair touching images 2 and 6
    p += [(0, 1), (1, 0), (0, 1), (4, 5), (6, 6)]               # duplicates
    return p


def run_pairs(xf, rows, n, kpts, pairs, thr):
    lib = xf._lib
    P = len(pairs)
    tp = torch.tensor(pairs, dtype=torch.int32).cuda()
    idx0 = torch.full((P, N_MAX), -7, dtype=torch.int64, device="cuda")
    idx1 = torch.full_like(idx0, -7)
    cnt = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.xfeat_mnn_pairs_workspace_bytes(P, N_MAX), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.xfeat_mnn_match_pairs(rows.data_ptr(), n.data_ptr(), rows.shape[0], N_MAX, rows.shape[1], tp.data_ptr(), P, 13,
                                         float(thr), idx0.data_ptr(), idx1.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(),
                                         st), "xfeat_mnn_match_pairs")
    o0 = torch.zeros((P, N_MAX, 2), device="cuda")
    o1 = torch.zeros_like(o0)
    _lib.check(lib.xfeat_gather_matches_pairs(kpts.data_ptr(), N_MAX, tp.data_ptr(), idx0.data_ptr(), idx1.data_ptr(), cnt.data_ptr(),
                                              P, o0.data_ptr(), o1.data_ptr(), st), "xfeat_gather_matches_pairs")
    torch.cuda.synchronize()
    return idx0.cpu(), idx1.cpu(), cnt.cpu(), o0.cpu(), o1.cpu()


def run_one(xf, rows, n, i, j, thr):
    """xfeat_mnn_match_presplit on images (i, j) alone."""
    i0, i1, c = xf._mnn_presplit_device(rows[i:i + 1], n[i:i + 1], rows[j:j + 1], n[j:j + 1], N_MAX, rows.shape[1], 1, thr)
    torch.cuda.synchronize()
    return i0[0].cpu(), i1[0].cpu(), int(c[0])


@pytest.mark.parametrize("impl", [1, 2, 3])
@pytest.mark.parametrize("thr", [-1.0, 0.82])
def test_kernel_pairs_equal_single_pair_presplit(xf, table, impl, thr):
    rows, n, kpts = table
    pairs = pair_list()
    with mnn_impl(xf, impl):
        idx0, idx1, cnt, o0, o1 = run_pairs(xf, rows, n, kpts, pairs, thr)
        refs = [run_one(xf, rows, n, i, j, thr) for i, j in pairs]
    k = kpts.cpu()
    total = 0
    for p, ((i, j), (r0, r1, rc)) in enumerate(zip(pairs, refs)):
        c = int(cnt[p])
        assert c == rc, f"pair {p} ({i}, {j}): {c} matches, single-pair call {rc}"
        if COUNTS[i] < 0 or COUNTS[j] < 0:
            assert c == _lib.N_OVERFLOW
            continue
        assert torch.equal(idx0[p, :c], r0[:c]) and torch.equal(idx1[p, :c], r1[:c]), f"pair {p} ({i}, {j})"
        assert torch.equal(o0[p, :c], k[i][idx0[p, :c]]) and torch.equal(o1[p, :c], k[j][idx1[p, :c]]), f"pair {p} gather"
        if min(COUNTS[i], COUNTS[j]) == 0:
            assert c == 0
        total += c
    assert total > 10000                                        # the copies and the shared rows give real match lists


def test_kernel_pairs_rejects_other_impls(xf, table):
    rows, n, kpts = table
    with mnn_impl(xf, 0):
        with pytest.raises(_lib.XFeatLibraryError, match="does not take pre-split"):
            run_pairs(xf, rows, n, kpts, [(0, 1)], -1)


# ---------------------------------------------------------------------------------------------------------------------------
# 2.-5. the public calls
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def images(assets_vga):
    ref, tgt = assets_vga
    crop = np.ascontiguousarray(tgt[60:360, 100:500])                             # 300 x 400
    big = F.interpolate(torch.from_numpy(ref).permute(2, 0, 1)[None].float().cuda() / 255, size=(1184, 864),
                        mode="bilinear", align_corners=False)[0].contiguous()    # (3, 1184, 864) float on the device
    gray = np.ascontiguousarray(ref.mean(-1).astype(np.uint8))                     # (480, 640) grayscale
    return [ref, tgt, crop, big, gray]


def single(x):
    """The image as match_xfeat takes it (its numpy input must be (H,W,C))."""
    return x[:, :, None] if isinstance(x, np.ndarray) and x.ndim == 2 else x


def count_net_rows(xf, monkeypatch):
    rows = []
    real = xf._run_net

    def wrapped(xn, B, H, W, want_logits=False):
        rows.append(B)
        return real(xn, B, H, W, want_logits)
    monkeypatch.setattr(xf, "_run_net", wrapped)
    return rows


@pytest.mark.parametrize("impl", [1, 0])
def test_api_pairs_equal_match_xfeat(xf, images, impl, monkeypatch):
    unused = np.zeros((256, 256, 3), np.uint8)                   # referenced by no pair: never extracted
    imgs = images[:3] + [unused] + images[3:]
    idx = [0, 1, 2, 4, 5]
    pairs = [(i, j) for i in idx for j in idx]
    with mnn_impl(xf, impl):
        rows = count_net_rows(xf, monkeypatch)
        got = xf.match_xfeat_pairs(imgs, np.asarray(pairs), top_k=4096)
        assert sum(rows) == 5, rows                             # each referenced image once
        monkeypatch.undo()
        n_total = 0
        for p, (i, j) in enumerate(pairs):
            w0, w1 = xf.match_xfeat(single(imgs[i]), single(imgs[j]), top_k=4096)
            assert np.array_equal(got[p][0], w0) and np.array_equal(got[p][1], w1), f"pair {p} = ({i}, {j})"
            n_total += len(w0)
    assert n_total > 25 * 200


def test_api_pairs_many_images_chunks(xf, assets_vga, monkeypatch):
    """More than one extraction chunk of a bucket (70 VGA images), a second bucket, several matcher chunks, min_cossim."""
    ref, tgt = assets_vga
    rng = np.random.default_rng(5)
    imgs = []
    for k in range(70):
        base = ref if k % 2 == 0 else tgt
        im = np.clip(base.astype(np.int16) + rng.integers(-12, 13, base.shape), 0, 255).astype(np.uint8)
        imgs.append(im[:, ::-1].copy() if k % 3 == 0 else im)
    imgs += [np.ascontiguousarray(ref[:320, :448]), np.ascontiguousarray(tgt[:320, :448])]
    pairs = rng.integers(0, len(imgs), (60, 2))
    pairs[:4] = [[0, 70], [71, 1], [69, 68], [70, 71]]
    monkeypatch.setattr(xfeat_mod, "PAIRS_MATCH_CHUNK", 16)
    rows = count_net_rows(xf, monkeypatch)
    got = xf.match_xfeat_pairs(imgs, pairs, top_k=2048, min_cossim=0.82)
    assert sum(rows) == len(np.unique(pairs)) and max(rows) <= 64, rows
    monkeypatch.undo()
    for p, (i, j) in enumerate(pairs.tolist()):
        w0, w1 = xf.match_xfeat(imgs[i], imgs[j], top_k=2048, min_cossim=0.82)
        assert np.array_equal(got[p][0], w0) and np.array_equal(got[p][1], w1), f"pair {p} = ({i}, {j})"


def test_api_pairs_overflow_names_pairs(xf, images, monkeypatch):
    """An image whose NMS candidate list overflowed (its count XF_N_OVERFLOW, set here in the table after the extraction) fails
    every pair that names it, and the error names those pairs and images."""
    imgs = images[:3]
    pairs = [(0, 1), (2, 0), (1, 1), (1, 2)]
    plan = xfeat_mod.PairPlan([xfeat_mod.pair_image_key(x) for x in imgs], pairs)
    real = xf._extract_table

    def overflow_image_2(*a, **k):
        tab = real(*a, **k)
        tab["n_valid"][int(plan.slot[2])] = _lib.N_OVERFLOW
        return tab
    monkeypatch.setattr(xf, "_extract_table", overflow_image_2)
    with pytest.raises(_lib.XFeatLibraryError) as e:
        xf.match_xfeat_pairs(imgs, pairs, top_k=1024)
    msg = str(e.value)
    assert "pair 1 (images 2, 0)" in msg and "pair 3 (images 1, 2)" in msg and "pair 0 " not in msg, msg


def test_lighterglue_pairs_equal_batch(xf, images):
    if xf._lighterglue_weights is None:
        pytest.skip("LighterGlue weights not built (oracle/build_lighterglue.py)")
    imgs = images[:3]
    pairs = [(i, j) for i in range(3) for j in range(3)] + [(0, 1)]
    got = xf.match_xfeat_lighterglue_pairs(imgs, pairs, top_k=2048)
    for p, (i, j) in enumerate(pairs):
        w = xf.match_xfeat_lighterglue_batch(imgs[i], imgs[j], top_k=2048)[0]
        for a, b in zip(got[p], w):
            assert np.array_equal(a, b), f"pair {p} = ({i}, {j})"
    assert sum(len(g[0]) for g in got) > 1000


def test_harness_sparse_repeated_images(xf, assets_vga):
    from accelerated_features_b200.evalharness import batched_matcher
    ref, tgt = assets_vga
    small = np.ascontiguousarray(ref[:320, :448])
    pairs = [(ref, tgt), (tgt, ref), (ref, small), (small, small), (ref, tgt), (tgt, small.copy())]
    got = batched_matcher(xf, "sparse", top_k=2048)(pairs)
    for (a, b), (g0, g1) in zip(pairs, got):
        s0, s1 = xf.match_xfeat(a, b, top_k=2048)
        assert np.array_equal(g0, s0) and np.array_equal(g1, s1)
