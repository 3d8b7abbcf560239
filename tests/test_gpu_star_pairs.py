"""Semi-dense pair lists over one image table: xfeat_mnn_match_pairs_f32 against xfeat_mnn_match on each pair alone and
xfeat_refine_pairs against xfeat_refine on each pair's own slices, bit for bit; XFeat.match_xfeat_star_pairs and the star mode of
the evaluation harness against per-pair match_xfeat_star calls, bit for bit."""
import contextlib

import numpy as np
import pytest
import torch

from accelerated_features_b200 import _lib
from accelerated_features_b200 import xfeat as xfeat_mod

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat(device=0)


@contextlib.contextmanager
def mnn_impl(xf, impl):
    old = xf._lib.xfeat_get_mnn_impl()
    xf._lib.xfeat_set_mnn_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_mnn_impl(old)


@contextlib.contextmanager
def conv_impl(xf, impl):
    old = xf._lib.xfeat_get_conv_impl()
    xf._lib.xfeat_set_conv_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_conv_impl(old)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. kernels
# ---------------------------------------------------------------------------------------------------------------------------
K_MAX = 5000
COUNTS = [0, 1, 511, 4096, K_MAX, 3000, 3000, 2000, 1500]
B_TIE, C_TIE, R1, R2, Q = 5, 6, 10, 11, 20


@pytest.fixture(scope="module")
def table():
    """9 images of un-normalised descriptors (n_images, K_MAX, 64) with the counts above; image 7 has max |x| ~ 2^18 and image 8
    ~ 2^-6, 2^24 apart.  Images 3 / 4 and 0-2 share rows with noise, so pairs have many matches.

    Images 5 (B) and 6 (C), max |x| = 1, hold a tie that only the pair's own exponent breaks: rows R1 and R2 of B are e_0 and
    e_0 + 2^-22 e_1, row Q of C is e_1, and every other row of B has x_1 < 0 and of C x_0, x_1 < 0.  Split at the pair's
    exponent (2^13), 2^-22 becomes 2^-9, an exact fp16: S(Q, R2) = 2^-22 > S(Q, R1) = 0 and (Q, R2) is a mutual match.  Split at
    the table's exponent (image 7's, 2^-5), it becomes 2^-27 and rounds to 0 in hi and lo: Q ties R1 and R2, the lower row R1
    wins, and the match is (Q, R1)."""
    g = torch.Generator().manual_seed(23)
    d = torch.randn(len(COUNTS), K_MAX, 64, generator=g)
    d[4] = d[3, torch.arange(K_MAX) % 4096] + 0.3 * torch.randn(K_MAX, 64, generator=g)
    d[2, :511] = d[3, :511] + 0.2 * torch.randn(511, 64, generator=g)
    d[7] *= 2.0 ** 16
    d[8] *= 2.0 ** -8
    for t in (B_TIE, C_TIE):
        d[t] = torch.rand(K_MAX, 64, generator=g) * 1.8 - 0.9
    d[B_TIE, :, 1] = -(d[B_TIE, :, 1].abs() + 0.01)
    d[C_TIE, :, 0] = -(d[C_TIE, :, 0].abs() + 0.01)
    d[C_TIE, :, 1] = -(d[C_TIE, :, 1].abs() + 0.01)
    d[B_TIE, R1] = 0
    d[B_TIE, R1, 0] = 1.0
    d[B_TIE, R2] = d[B_TIE, R1]
    d[B_TIE, R2, 1] = 2.0 ** -22
    d[C_TIE, Q] = 0
    d[C_TIE, Q, 1] = 1.0
    for i, n in enumerate(COUNTS):
        d[i, n:] = float("nan")                                  # rows past the count are never read
    return d.cuda(), torch.tensor(COUNTS, dtype=torch.int32).cuda()


def pair_list():
    n = len(COUNTS)
    return [(i, j) for i in range(n) for j in range(n)] + [(B_TIE, C_TIE), (3, 4), (0, 0)]   # every ordered pair, duplicates


def run_pairs_f32(xf, d, n, pairs):
    lib = xf._lib
    P = len(pairs)
    tp = torch.tensor(pairs, dtype=torch.int32).cuda()
    idx0 = torch.full((P, K_MAX), -7, dtype=torch.int64, device="cuda")
    idx1 = torch.full_like(idx0, -7)
    cnt = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.xfeat_mnn_pairs_f32_workspace_bytes(P, K_MAX), dtype=torch.uint8, device="cuda")
    rc = lib.xfeat_mnn_match_pairs_f32(d.data_ptr(), n.data_ptr(), d.shape[0], K_MAX, tp.data_ptr(), P, idx0.data_ptr(),
                                       idx1.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, idx0, idx1, cnt


def run_one(xf, d, n, i, j):
    """xfeat_mnn_match on images (i, j) alone (their counts, abs_bound 0, min_cossim -1)."""
    i0, i1, c = xf._mnn_device(d[i], n[i:i + 1], K_MAX, K_MAX * 64, d[j], n[j:j + 1], K_MAX, K_MAX * 64, 1, -1)
    torch.cuda.synchronize()
    return i0[0].cpu(), i1[0].cpu(), int(c[0])


@pytest.mark.parametrize("impl", [1, 2, 3])
def test_kernel_pairs_f32_equal_single_pair(xf, table, impl):
    d, n = table
    pairs = pair_list()
    with mnn_impl(xf, impl):
        rc, idx0, idx1, cnt = run_pairs_f32(xf, d, n, pairs)
        _lib.check(rc, "xfeat_mnn_match_pairs_f32")
        refs = [run_one(xf, d, n, i, j) for i, j in pairs]
    idx0, idx1, cnt = idx0.cpu(), idx1.cpu(), cnt.cpu()
    total = 0
    for p, ((i, j), (r0, r1, rc_)) in enumerate(zip(pairs, refs)):
        c = int(cnt[p])
        assert c == rc_, f"pair {p} ({i}, {j}): {c} matches, single-pair call {rc_}"
        assert torch.equal(idx0[p, :c], r0[:c]) and torch.equal(idx1[p, :c], r1[:c]), f"pair {p} ({i}, {j})"
        if min(COUNTS[i], COUNTS[j]) == 0:
            assert c == 0
        total += c
    assert total > 20000
    # the tie: only the pair's own exponent gives (Q, R2); the table's would give (Q, R1)
    for p, (i, j) in enumerate(pairs):
        if (i, j) == (C_TIE, B_TIE):
            m = dict(zip(idx0[p, :cnt[p]].tolist(), idx1[p, :cnt[p]].tolist()))
            assert m.get(Q) == R2, m.get(Q)
        if (i, j) == (B_TIE, C_TIE):
            m = dict(zip(idx1[p, :cnt[p]].tolist(), idx0[p, :cnt[p]].tolist()))
            assert m.get(Q) == R2, m.get(Q)


@pytest.mark.parametrize("impl", [0, 4])
def test_kernel_pairs_f32_refuses_other_impls(xf, table, impl):
    d, n = table
    with mnn_impl(xf, impl):
        rc, *_ = run_pairs_f32(xf, d, n, [(3, 4)])
    assert rc == 4                                               # XF_E_UNSUPPORTED
    assert "does not take pre-split" in xf._lib.xfeat_last_error().decode()


@pytest.mark.parametrize("conv", [2, 0])
@pytest.mark.parametrize("fine_conf", [0.0, 0.25])
def test_refine_pairs_equal_single_pair(xf, conv, fine_conf):
    g = torch.Generator().manual_seed(31)
    counts = [7, 1200, 4096, 300, 0]
    nI = len(counts)
    desc = (torch.randn(nI, K_MAX, 64, generator=g) * 2).cuda()
    kpts = (torch.rand(nI, K_MAX, 2, generator=g) * 900).cuda()
    scales = (torch.rand(nI, K_MAX, generator=g) + 0.5).cuda()
    pairs = [(i, j) for i in range(nI) for j in range(nI)] + [(1, 2)]
    P = len(pairs)
    idx0 = torch.zeros(P, K_MAX, dtype=torch.int64)
    idx1 = torch.zeros(P, K_MAX, dtype=torch.int64)
    cnt = torch.zeros(P, dtype=torch.int32)
    for p, (i, j) in enumerate(pairs):
        c = min(counts[i], counts[j]) if p % 3 else min(counts[i], counts[j]) // 2
        cnt[p] = c
        if c:
            idx0[p, :c] = torch.randperm(counts[i], generator=g)[:c]
            idx1[p, :c] = torch.randint(0, counts[j], (c,), generator=g)
    idx0, idx1, cnt = idx0.cuda(), idx1.cuda(), cnt.cuda()
    tp = torch.tensor(pairs, dtype=torch.int32).cuda()
    tab = {"descriptors": desc, "keypoints": kpts, "scales": scales}
    with conv_impl(xf, conv):
        got, n_got = xf._refine_pairs_device(tab, tp, idx0, idx1, cnt, K_MAX, fine_conf)
        refs = []
        for p, (i, j) in enumerate(pairs):
            d0 = {"descriptors": desc[i:i + 1], "keypoints": kpts[i:i + 1], "scales": scales[i:i + 1]}
            d1 = {"descriptors": desc[j:j + 1], "keypoints": kpts[j:j + 1], "scales": scales[j:j + 1]}
            refs.append(xf._refine_device(d0, d1, idx0[p:p + 1], idx1[p:p + 1], cnt[p:p + 1], fine_conf))
        torch.cuda.synchronize()
    got, n_got = got.cpu(), n_got.cpu()
    kept = 0
    for p, (m, nr) in enumerate(refs):
        k = int(nr[0])
        assert int(n_got[p]) == k, f"pair {p}"
        assert torch.equal(got[p, :k], m[0, :k].cpu()), f"pair {p} {pairs[p]}"
        kept += k
    if fine_conf == 0.0:
        assert kept > 1000                                      # conf > 0 keeps every row


# ---------------------------------------------------------------------------------------------------------------------------
# 2. the public call and the harness
# ---------------------------------------------------------------------------------------------------------------------------
TOPK = 4096


@pytest.fixture(scope="module")
def images(assets_vga):
    ref, tgt = assets_vga
    crop = np.ascontiguousarray(ref[:320, :448])                                   # 320 x 448
    odd = np.ascontiguousarray(tgt[7:400, 13:563])                                 # 393 x 550: resize path at both scales
    small = np.ascontiguousarray(ref[100:196, 200:328].mean(-1).astype(np.uint8))   # (96, 128) grayscale: K_i < K_max
    flt = ref[40:440, 20:620].astype(np.float64)                                   # numpy float: "/255" on the host
    host_t = torch.from_numpy(tgt).permute(2, 0, 1).float() / 255                   # torch (3,H,W) on the host
    dev_t = torch.from_numpy(ref[::-1].copy()).permute(2, 0, 1)[None].cuda()        # torch (1,3,H,W) uint8 on the device
    return [ref, tgt, crop, odd, small, flt, host_t, dev_t]


def single(x):
    """The image as match_xfeat_star takes it (its numpy input must be (H,W,C))."""
    return x[:, :, None] if isinstance(x, np.ndarray) and x.ndim == 2 else x


def count_net_rows(xf, monkeypatch):
    rows = []
    real = xf._run_net

    def wrapped(xn, B, H, W, want_logits=False):
        rows.append(B)
        return real(xn, B, H, W, want_logits)
    monkeypatch.setattr(xf, "_run_net", wrapped)
    return rows


def check_against_single(xf, imgs, pairs, got):
    total = 0
    for p, (i, j) in enumerate(pairs):
        w0, w1 = xf.match_xfeat_star(single(imgs[i]), single(imgs[j]), top_k=TOPK)
        assert np.array_equal(got[p][0], w0) and np.array_equal(got[p][1], w1), f"pair {p} = ({i}, {j})"
        assert got[p][0].dtype == w0.dtype and got[p][0].shape == w0.shape
        total += len(w0)
    return total


def test_star_pairs_equal_match_xfeat_star(xf, images, monkeypatch):
    unused = np.zeros((256, 256, 3), np.uint8)                  # referenced by no pair: never extracted
    imgs = images[:2] + [unused] + images[2:]
    idx = [0, 1, 3, 4, 5, 6, 7, 8]
    pairs = [(i, j) for i in idx for j in idx] + [(0, 1), (5, 5), (8, 3)]
    rows = count_net_rows(xf, monkeypatch)
    got = xf.match_xfeat_star_pairs(imgs, np.asarray(pairs), top_k=TOPK)
    assert sum(rows) == 2 * len(idx), rows      # each referenced image once per scale
    monkeypatch.undo()
    assert len(got) == len(pairs)
    assert check_against_single(xf, imgs, pairs, got) > 50 * 300


@pytest.mark.parametrize("impl", [1, 2, 3, 0])
def test_star_pairs_chunked(xf, images, impl, monkeypatch):
    """Extraction chunks of 2 images, matcher chunks of 3 pairs, under each matcher implementation (0: the per-pair fallback)."""
    imgs = images
    rng = np.random.default_rng(impl)
    pairs = rng.integers(0, len(imgs), (20, 2))
    pairs[:3] = [[4, 4], [0, 4], [4, 0]]
    k_max = max(sum(xfeat_mod.dense_counts(*xfeat_mod.pair_image_key(x)[1:3], TOPK)) for x in imgs)
    monkeypatch.setattr(xfeat_mod, "PAIRS_EXTRACT_CHUNK", 2)
    monkeypatch.setattr(xfeat_mod, "STAR_PAIRS_MATCH_BYTES", 3 * xfeat_mod.star_pair_bytes(k_max))
    with mnn_impl(xf, impl):
        rows = count_net_rows(xf, monkeypatch)
        got = xf.match_xfeat_star_pairs(imgs, pairs, top_k=TOPK)
        assert sum(rows) == 2 * len(np.unique(pairs)) and max(rows) <= 2, rows
        monkeypatch.undo()
        check_against_single(xf, imgs, pairs.tolist(), got)


def test_star_pairs_empty(xf, images):
    assert xf.match_xfeat_star_pairs(images, np.zeros((0, 2), np.int64)) == []


def test_harness_star_repeated_images(xf, assets_vga):
    from accelerated_features_b200.evalharness import batched_matcher
    ref, tgt = assets_vga
    small = np.ascontiguousarray(ref[:320, :448])
    pairs = [(ref, tgt), (tgt, ref), (ref, small), (small, small), (ref, tgt), (tgt, small.copy())]
    got = batched_matcher(xf, "star", top_k=2048)(pairs)
    for (a, b), (g0, g1) in zip(pairs, got):
        s0, s1 = xf.match_xfeat_star(a, b, top_k=2048)
        assert np.array_equal(g0, s0) and np.array_equal(g1, s1)
