"""wgmma (tensor-core, split-fp16) implementation of xfeat_mnn_match against the CPU oracle.

The tensor-core scan computes S = hi.hi + hi.lo + lo.hi with fp32 accumulation: agreement with the fp32 oracle is exact
except where the arg-max is separated from the runner-up by less than accumulation noise; any difference must be
confined to such near-tie rows / columns (documented protocol, SURVEY 7.1)."""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import xfeat_oracle as orc  # noqa: E402


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


@contextlib.contextmanager
def mnn_impl(xf, impl):
    old = xf._lib.xfeat_get_mnn_impl()
    xf._lib.xfeat_set_mnn_impl(impl)
    try:
        yield
    finally:
        xf._lib.xfeat_set_mnn_impl(old)


def check_modulo_ties(f1, f2, got, want, eps_rel=3e-6):
    """Exact equality of the match lists, or every differing pair touches a row / column of S = F1 F2^T whose top-1 / top-2
    gap is below eps_rel * max|S| (fp32 accumulation noise).  Gaps are computed for the differing rows / columns only, so the
    check stays cheap at 32k x 32k."""
    g0, g1 = got
    w0, w1 = want
    if np.array_equal(g0, w0) and np.array_equal(g1, w1):
        return 0
    f1d, f2d = f1.double(), f2.double()
    wset = {(int(a), int(b)) for a, b in zip(w0, w1)}
    gset = {(int(a), int(b)) for a, b in zip(g0, g1)}
    diff = sorted(wset ^ gset)
    assert len(diff) <= 64, f"{len(diff)} differing pairs"

    def gap(v):
        if v.numel() < 2:
            return 1e9
        t = torch.topk(v, 2).values
        return float(t[0] - t[1])

    gaps, smax = [], 0.0
    for a, b in diff:
        r, c = f1d[a] @ f2d.t(), f1d @ f2d[b]
        smax = max(smax, float(r.abs().max()), float(c.abs().max()))
        gaps.append((gap(r), gap(c)))
    eps = eps_rel * smax
    for (a, b), (rg, cg) in zip(diff, gaps):
        assert rg < eps or cg < eps, f"robust pair ({a},{b}) differs (row gap {rg:.3e}, col gap {cg:.3e}, eps {eps:.3e})"
    return len(diff)


def run(xf, f1, f2, thr):
    i0, i1 = xf.match(f1.cuda(), f2.cuda(), thr)
    return i0.cpu().numpy(), i1.cpu().numpy()


TC_IMPLS = [4, 1, 2, 3]   # 4: filter + exact re-score (default), 1: one 3-term GEMM per direction, 2: single GEMM (row + column arg-max), 3: 1 with one CTA per work item


@pytest.mark.parametrize("impl", TC_IMPLS)
def test_tc_golden(xf, golden, impl):
    g = golden("g5_mnn.npz")
    f1, f2 = torch.from_numpy(g["f1"]), torch.from_numpy(g["f2"])
    with mnn_impl(xf, impl):
        for thr, sfx in ((-1, ""), (0.82, "_082"), (0.3, "_03")):
            got = run(xf, f1, f2, thr)
            nd = check_modulo_ties(f1, f2, got, (g["idx0" + sfx], g["idx1" + sfx]))
            print(f"thr={thr}: {len(got[0])} matches, {nd} tie-differences")


@pytest.mark.parametrize("impl", TC_IMPLS)
@pytest.mark.parametrize("n1,n2", [(1, 1), (5, 300), (129, 127), (256, 256), (257, 511), (1000, 2048), (4096, 4096), (2500, 777)])
def test_tc_vs_oracle_sizes(xf, n1, n2, impl):
    g = torch.Generator().manual_seed(n1 * 7 + n2)
    f1 = F.normalize(torch.randn(n1, 64, generator=g), dim=-1)
    f2 = F.normalize(torch.randn(n2, 64, generator=g), dim=-1)
    with mnn_impl(xf, impl):
        for thr in (-1, 0.3):
            w0, w1 = orc.mnn_match(f1, f2, thr)
            got = run(xf, f1, f2, thr)
            nd = check_modulo_ties(f1, f2, got, (w0.numpy(), w1.numpy()))
            assert nd <= max(2, n1 // 500)


@pytest.mark.parametrize("n", [8192, 16384, 32768])
def test_default_impl_vs_oracle_c5_sweep(xf, n):
    """BASELINE config 5 (MNN sweep 2k..32k): the upper half of the sweep against the oracle, default implementation."""
    g = torch.Generator().manual_seed(0)
    f1 = F.normalize(torch.randn(n, 64, generator=g), dim=-1)
    f2 = F.normalize(torch.randn(n, 64, generator=g), dim=-1)
    w0, w1 = orc.mnn_match(f1, f2, -1)
    got = run(xf, f1, f2, -1)
    nd = check_modulo_ties(f1, f2, got, (w0.numpy(), w1.numpy()))
    from tests.parity_util import record
    record(f"mnn_c5_n{n}", mutual=len(got[0]), oracle=len(w0), tie_differences=nd)
    assert nd <= max(2, n // 2000)


@pytest.mark.parametrize("impl", TC_IMPLS)
def test_tc_equals_simt_on_real_descriptors(xf, assets_vga, impl):
    """Descriptors of the asset pair: both implementations must return the same matches (modulo near-ties)."""
    ref, tgt = assets_vga
    out = xf.detectAndCompute(np.stack([ref, tgt]).transpose(0, 3, 1, 2).astype(np.float32) / 255, top_k=4096) \
        if False else xf.detectAndCompute(torch.from_numpy(np.stack([ref, tgt])).permute(0, 3, 1, 2).float() / 255, top_k=4096)
    d0, d1 = out[0]["descriptors"], out[1]["descriptors"]
    with mnn_impl(xf, 0):
        a0, a1 = xf.match(d0, d1, -1)
    with mnn_impl(xf, impl):
        b0, b1 = xf.match(d0, d1, -1)
        c0, c1 = xf.match(d0, d1, 0.82)
    nd = check_modulo_ties(d0.cpu(), d1.cpu(), (b0.cpu().numpy(), b1.cpu().numpy()), (a0.cpu().numpy(), a1.cpu().numpy()))
    print(f"asset pair: simt {len(a0)} matches, tensor cores {len(b0)}, differing pairs {nd}; 0.82 -> {len(c0)}")
    w0, w1 = orc.mnn_match(d0.cpu(), d1.cpu(), 0.82)
    check_modulo_ties(d0.cpu(), d1.cpu(), (c0.cpu().numpy(), c1.cpu().numpy()), (w0.numpy(), w1.numpy()))
    assert nd <= 4


@pytest.mark.parametrize("impl", TC_IMPLS)
def test_tc_batched_ragged_unnormalised(xf, impl):
    g = torch.Generator().manual_seed(11)
    B, N = 5, 700
    f1 = torch.randn(B, N, 64, generator=g) * 3.0
    f2 = torch.randn(B, N, 64, generator=g) * 3.0
    n1 = [700, 1, 128, 333, 0]
    n2 = [700, 700, 129, 5, 40]
    with mnn_impl(xf, impl):
        idx0, idx1, cnt = xf._mnn_device(f1.cuda(), torch.tensor(n1, dtype=torch.int32).cuda(), N, N * 64, f2.cuda(),
                                         torch.tensor(n2, dtype=torch.int32).cuda(), N, N * 64, B, -1)
    c = cnt.tolist()
    for b in range(B):
        if n1[b] == 0 or n2[b] == 0:
            assert c[b] == 0
            continue
        w0, w1 = orc.mnn_match(f1[b, :n1[b]], f2[b, :n2[b]], -1)
        check_modulo_ties(f1[b, :n1[b]], f2[b, :n2[b]], (idx0[b, :c[b]].cpu().numpy(), idx1[b, :c[b]].cpu().numpy()),
                          (w0.numpy(), w1.numpy()))


@pytest.mark.parametrize("impl", TC_IMPLS)
def test_tc_full_size_identity(xf, impl):
    """64 x (4096 x 4096): matching a set against itself returns the identity (size-independent property)."""
    g = torch.Generator().manual_seed(5)
    f = F.normalize(torch.randn(64, 4096, 64, generator=g), dim=-1).cuda()
    with mnn_impl(xf, impl):
        idx0, idx1, cnt = xf._mnn_device(f, None, 4096, 4096 * 64, f, None, 4096, 4096 * 64, 64, -1)
    assert cnt.tolist() == [4096] * 64
    assert torch.equal(idx0, idx1) and torch.equal(idx0[3], torch.arange(4096, device="cuda"))


@pytest.mark.parametrize("impl", [0, 1, 2, 3, 4])
def test_exact_ties_first_index(xf, impl):
    """Duplicate descriptors give bit-equal similarities: torch's first-index rule decides (xfeat.py:333-339).  Rows 3/700
    of set 1 and rows 10/450 of set 2 are duplicated; values are small integers / 8 so every product and sum is exact in
    every implementation and the oracle comparison is bit for bit."""
    g = torch.Generator().manual_seed(21)
    f1 = torch.randint(-4, 5, (900, 64), generator=g).float() / 8
    f2 = torch.randint(-4, 5, (600, 64), generator=g).float() / 8
    f2[:300] = f1[:300]            # guaranteed strong matches
    f1[700] = f1[3]
    f1[701] = f1[3]
    f2[450] = f2[10]
    w0, w1 = orc.mnn_match(f1, f2, -1)
    with mnn_impl(xf, impl):
        g0, g1 = run(xf, f1, f2, -1)
    assert np.array_equal(g0, w0.numpy()) and np.array_equal(g1, w1.numpy())
    assert 3 in g0 and 700 not in g0 and 701 not in g0


@pytest.mark.parametrize("impl", TC_IMPLS)
def test_bounded_scale_matches_measured_scale(xf, impl):
    """xfeat_mnn_match_bounded(abs_bound=1) on unit-norm descriptors: same matches as the max-reduction path (the bound only
    picks the power-of-two operand scale), and the same as the oracle modulo accumulation-noise ties."""
    g = torch.Generator().manual_seed(77)
    B, N = 3, 1500
    f1 = F.normalize(torch.randn(B, N, 64, generator=g), dim=-1)
    f2 = F.normalize(torch.randn(B, N, 64, generator=g), dim=-1)
    n1 = torch.tensor([1500, 1024, 7], dtype=torch.int32)
    n2 = torch.tensor([1500, 900, 1500], dtype=torch.int32)
    with mnn_impl(xf, impl):
        a = xf._mnn_device(f1.cuda(), n1.cuda(), N, N * 64, f2.cuda(), n2.cuda(), N, N * 64, B, 0.1)
        b = xf._mnn_device(f1.cuda(), n1.cuda(), N, N * 64, f2.cuda(), n2.cuda(), N, N * 64, B, 0.1, abs_bound=1.0)
    ca, cb = a[2].tolist(), b[2].tolist()
    for i in range(B):
        w0, w1 = orc.mnn_match(f1[i, :n1[i]], f2[i, :n2[i]], 0.1)
        for got, c in ((a, ca), (b, cb)):
            check_modulo_ties(f1[i, :n1[i]], f2[i, :n2[i]], (got[0][i, :c[i]].cpu().numpy(), got[1][i, :c[i]].cpu().numpy()),
                              (w0.numpy(), w1.numpy()))


def test_fast_equals_three_term_kernel(xf, assets_vga):
    """Implementation 4 (filter + exact re-score) against implementation 1 (three-term GEMM everywhere): IDENTICAL index lists,
    on unit-norm, unnormalised (star path) and near-duplicate (many ambiguous rows) descriptor sets, ragged counts included."""
    g = torch.Generator().manual_seed(123)
    cases = []
    f1 = F.normalize(torch.randn(6, 1100, 64, generator=g), dim=-1)
    f2 = F.normalize(torch.randn(6, 1100, 64, generator=g), dim=-1)
    cases.append((f1, f2, [1100, 1000, 513, 512, 3, 1100], [1100, 257, 1100, 640, 1100, 1]))
    cases.append((torch.randn(3, 900, 64, generator=g) * 13.0, torch.randn(3, 900, 64, generator=g) * 9.0, None, None))
    base = F.normalize(torch.randn(1, 700, 64, generator=g), dim=-1)
    near = F.normalize(base + 1e-4 * torch.randn(1, 700, 64, generator=g), dim=-1)       # every row has a runner-up within ~1e-4
    cases.append((torch.cat([base, near], 1), torch.cat([near, base], 1), None, None))
    for f1, f2, n1, n2 in cases:
        B, N = f1.shape[0], f1.shape[1]
        n1d = None if n1 is None else torch.tensor(n1, dtype=torch.int32).cuda()
        n2d = None if n2 is None else torch.tensor(n2, dtype=torch.int32).cuda()
        res = {}
        for impl in (1, 4):
            with mnn_impl(xf, impl):
                res[impl] = xf._mnn_device(f1.cuda(), n1d, N, N * 64, f2.cuda(), n2d, N, N * 64, B, -1)
        assert torch.equal(res[1][2], res[4][2])
        for b, c in enumerate(res[1][2].tolist()):
            assert torch.equal(res[1][0][b, :c], res[4][0][b, :c]) and torch.equal(res[1][1][b, :c], res[4][1][b, :c])


@pytest.mark.parametrize("impl", [1, 3])
def test_presplit_operands_equal_split_pass(xf, assets_vga, impl):
    """xfeat_detect_sparse_split writes the matcher's operand rows itself; xfeat_mnn_match_presplit on them must return exactly
    what xfeat_mnn_match_bounded returns after its own split pass over the fp32 descriptors (ragged counts, B = 3)."""
    ref, tgt = assets_vga
    x = torch.from_numpy(np.stack([ref, tgt, ref[::-1].copy(), tgt, ref, tgt[:, ::-1].copy()])).permute(0, 3, 1, 2).float() / 255
    with mnn_impl(xf, impl):
        o = xf._detect_sparse_device(x, 3000, 0.05, want_split=True)
        d, n, sp = o["descriptors"], o["n_valid"], o["desc_split"]
        assert sp.shape == (6, 3072, 128) and sp.dtype == torch.float16
        a = xf._mnn_device(d[:3], n[:3], 3000, 3000 * 64, d[3:], n[3:], 3000, 3000 * 64, 3, 0.5, abs_bound=1.0)
        b = xf._mnn_presplit_device(sp[:3], n[:3], sp[3:], n[3:], 3000, 3072, 3, 0.5)
    assert torch.equal(a[2], b[2])
    for i, c in enumerate(a[2].tolist()):
        assert torch.equal(a[0][i, :c], b[0][i, :c]) and torch.equal(a[1][i, :c], b[1][i, :c])
    # the rows are hi + lo = descriptor * 2^13, zero past n_valid
    nv = int(n[0])
    rec = (sp[0, :nv, :64].float() + sp[0, :nv, 64:].float()) / 8192.0
    assert (rec - d[0, :nv]).abs().max().item() < 1e-6 and float(sp[0, nv:].abs().sum()) == 0.0
