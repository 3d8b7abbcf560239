"""The single-GEMM matcher (implementation 1: S = F1.F2^T once per pair, row and column arg-max from the same accumulator tiles)
against the persistent kernel with one GEMM per direction (implementation 2): idx0, idx1 and the counts must be IDENTICAL --
both add the same three split-fp16 products in the same order, so the column arg-max of S12 equals the row arg-max of S21
bit for bit -- and equal to the fp32 CUDA-core implementation 0 modulo accumulation-noise near-ties.  The cases aim at the
parts of the new kernel that implementation 2 does not have: masked columns of the last tile and rows of the last row block,
the column tie rule across lanes, warps, slabs and row blocks (lowest row through the shared-memory combine and the global
atomic), and the persistent schedule at batch sizes around the SM count.  The CPU test reads the ptxas log of the build."""
import glob
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_mnn_tc import check_modulo_ties, mnn_impl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    return XFeat()


def match(xf, impl, f1, n1, f2, n2, thr=-1.0):
    """_mnn_device on (B, N, 64) host tensors with optional per-pair counts; returns host (idx0, idx1, counts)."""
    B, N1, N2 = f1.shape[0], f1.shape[1], f2.shape[1]
    n1d = None if n1 is None else torch.tensor(n1, dtype=torch.int32).cuda()
    n2d = None if n2 is None else torch.tensor(n2, dtype=torch.int32).cuda()
    with mnn_impl(xf, impl):
        i0, i1, c = xf._mnn_device(f1.cuda(), n1d, N1, N1 * 64, f2.cuda(), n2d, N2, N2 * 64, B, thr)
    torch.cuda.synchronize()
    return i0.cpu(), i1.cpu(), c.cpu()


def assert_same(a, b):
    assert torch.equal(a[2], b[2]), f"counts differ: {a[2].tolist()} vs {b[2].tolist()}"
    for i, c in enumerate(a[2].tolist()):
        assert torch.equal(a[0][i, :c], b[0][i, :c]) and torch.equal(a[1][i, :c], b[1][i, :c]), f"pair {i} differs"


def check_vs_simt(xf, f1, n1, f2, n2, got):
    ref = match(xf, 0, f1, n1, f2, n2)
    for i in range(f1.shape[0]):
        a = f1.shape[1] if n1 is None else n1[i]
        b = f2.shape[1] if n2 is None else n2[i]
        c, w = int(got[2][i]), int(ref[2][i])
        check_modulo_ties(f1[i, :a], f2[i, :b], (got[0][i, :c].numpy(), got[1][i, :c].numpy()),
                          (ref[0][i, :w].numpy(), ref[1][i, :w].numpy()))


@pytest.mark.gpu
@pytest.mark.parametrize("n1,n2", [(1, 1), (1, 300), (300, 1), (129, 127), (255, 257), (1000, 777), (777, 1000), (513, 4100)])
def test_fused_equals_two_gemm_sizes(xf, n1, n2):
    g = torch.Generator().manual_seed(n1 * 31 + n2)
    f1 = F.normalize(torch.randn(1, n1, 64, generator=g), dim=-1)
    f2 = F.normalize(torch.randn(1, n2, 64, generator=g), dim=-1)
    got = match(xf, 1, f1, None, f2, None)
    assert_same(got, match(xf, 2, f1, None, f2, None))
    check_vs_simt(xf, f1, None, f2, None, got)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 64, 65])
def test_fused_equals_two_gemm_ragged(xf, B):
    """Ragged counts with empty sides (one or both), unnormalised descriptors (operand scale), B around the SM count."""
    g = torch.Generator().manual_seed(B)
    N = 700
    f1 = torch.randn(B, N, 64, generator=g) * 5.0
    f2 = torch.randn(B, N, 64, generator=g) * 3.0
    n1 = torch.randint(0, N + 1, (B,), generator=g).tolist()
    n2 = torch.randint(0, N + 1, (B,), generator=g).tolist()
    edge = [(0, 5), (5, 0), (0, 0), (1, N), (N, 1), (256, 256), (257, 255), (N, N)]
    for i, (a, b) in enumerate(edge[:B]):
        n1[i], n2[i] = a, b
    got = match(xf, 1, f1, n1, f2, n2)
    assert_same(got, match(xf, 2, f1, n1, f2, n2))
    for i in range(B):
        if n1[i] == 0 or n2[i] == 0:
            assert int(got[2][i]) == 0
    if B == 1:
        check_vs_simt(xf, f1, n1, f2, n2, got)


@pytest.mark.gpu
def test_fused_exact_column_and_row_ties(xf):
    """Bit-equal similarities decide by the first index.  Copies of one set-1 row sit in rows of different lanes, warps and
    slabs of one 256-row block and in other row blocks, so the column arg-max of every column must pick the lowest row
    through the in-warp, shared-memory and global combines; duplicated set-2 rows in different column tiles test the row
    side.  Values are multiples of 1/8 with small integers: every product and sum is exact, so the oracle agrees bit for bit."""
    from oracle import xfeat_oracle as orc
    g = torch.Generator().manual_seed(3)
    n1, n2 = 1400, 900
    f1 = torch.randint(-4, 5, (n1, 64), generator=g).float() / 8
    f2 = torch.randint(-4, 5, (n2, 64), generator=g).float() / 8
    f2[:400] = f1[:400]
    # copies of row 300 (block 1, slab 0, warp 2): the lowest, row 100, is in block 0; the others in later lanes / warps /
    # slabs of block 1 and in blocks 2 and 5.  Column 300 (set 2's copy of the original row 300) must pick row 100.
    for r in (1399, 1290, 700, 600, 520, 511, 395, 384, 320, 310, 301, 302, 100):
        f1[r] = f1[300]
    # row 17 = warp 1, lane group 1, h = 0; copies in the same thread (25, 81, 89: h = 1..3), an earlier lane group of a later
    # h (24: group 0, h = 1), another lane group (18), warp (33) and slab 1 (129 ...)
    for r in (18, 24, 25, 33, 81, 89, 129, 130, 160, 200, 255):
        f1[r] = f1[17]
    for c in (128, 256, 899, 450):
        f2[c] = f2[10]
    f1b, f2b = f1[None], f2[None]
    got = match(xf, 1, f1b, None, f2b, None)
    assert_same(got, match(xf, 2, f1b, None, f2b, None))
    w0, w1 = orc.mnn_match(f1, f2, -1)
    c = int(got[2][0])
    assert np.array_equal(got[0][0, :c].numpy(), w0.numpy()) and np.array_equal(got[1][0, :c].numpy(), w1.numpy())
    pairs = dict(zip(got[0][0, :c].tolist(), got[1][0, :c].tolist()))
    assert pairs.get(100) == 300 and 300 not in pairs and pairs.get(17) == 17


@pytest.mark.gpu
def test_fused_equals_two_gemm_with_threshold(xf):
    """min_cossim reads the packed VALUE of best12: thresholds at quantiles of the matched similarities put many rows on
    either side, so a wrong value (or a wrong power-of-two operand scale on unnormalised input) changes the lists."""
    g = torch.Generator().manual_seed(17)
    B, N = 3, 1500
    base = torch.randn(B, N, 64, generator=g)
    f1 = base * 2.0
    f2 = (base + 0.8 * torch.randn(B, N, 64, generator=g)) * 0.5
    n1, n2 = [1500, 1000, 777], [1500, 1200, 300]
    allm = match(xf, 2, f1, n1, f2, n2)
    sims = torch.cat([(f1[b, allm[0][b, :c]] * f2[b, allm[1][b, :c]]).sum(-1) for b, c in enumerate(allm[2].tolist())])
    for q in (0.25, 0.5, 0.75):
        thr = float(torch.quantile(sims, q))
        got = match(xf, 1, f1, n1, f2, n2, thr)
        want = match(xf, 2, f1, n1, f2, n2, thr)
        assert_same(got, want)
        assert 0 < int(got[2].sum()) < int(allm[2].sum())


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16384, 32768])
def test_fused_equals_two_gemm_large(xf, n):
    g = torch.Generator().manual_seed(n)
    f1 = F.normalize(torch.randn(1, n, 64, generator=g), dim=-1)
    f2 = F.normalize(torch.randn(1, n - 1000, 64, generator=g), dim=-1)
    assert_same(match(xf, 1, f1, None, f2, None), match(xf, 2, f1, None, f2, None))


@pytest.mark.gpu
def test_fused_presplit_bench_shape(xf, assets_vga):
    """The bench workload's matcher call: 64 pairs x top_k 4096, operands written by xfeat_detect_sparse_split."""
    ref, tgt = assets_vga
    imgs = []
    for i in range(64):
        a, b = (ref, tgt) if i % 2 == 0 else (tgt, ref)
        if i % 4 >= 2:
            a = a[:, ::-1].copy()
        if i % 8 >= 4:
            b = b[::-1].copy()
        imgs.append((a, b))
    x = torch.from_numpy(np.stack([a for a, _ in imgs] + [b for _, b in imgs])).permute(0, 3, 1, 2).float() / 255
    res = {}
    for impl in (1, 2):
        with mnn_impl(xf, impl):
            o = xf._detect_sparse_device(x, 4096, 0.05, want_split=True)
            d, n, sp = o["descriptors"], o["n_valid"], o["desc_split"]
            res[impl] = xf._mnn_presplit_device(sp[:64], n[:64], sp[64:], n[64:], 4096, sp.shape[1], 64, -1)
            if impl == 2:
                split_pass = xf._mnn_device(d[:64], n[:64], 4096, 4096 * 64, d[64:], n[64:], 4096, 4096 * 64, 64, -1,
                                            abs_bound=1.0)
    torch.cuda.synchronize()
    assert int(res[1][2].sum()) > 64 * 100
    for other in (res[2], split_pass):
        assert_same(tuple(t.cpu() for t in res[1]), tuple(t.cpu() for t in other))


def test_build_log_fused_matcher_no_spills():
    """ptxas report of mnn_tc.cu: the matcher kernels do not spill and no wgmma is serialised (C7519 / C7520)."""
    path = os.path.join(ROOT, "accelerated_features_b200", "build", "mnn_tc.o.log")
    if not os.path.exists(path):
        from accelerated_features_b200.build import build_library
        build_library(force=True)
    text = open(path).read()
    assert "C7519" not in text and "C7520" not in text, "ptxas serialises wgmma in mnn_tc.cu"
    kernels = dict(re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes spill stores", text, re.S))
    fused = [k for k in kernels if "mnn_tc_persist_kernel" in k]
    assert fused, "no ptxas -v output for mnn_tc_persist_kernel"
    for fn, spill in kernels.items():
        if "mnn_tc" in fn:
            assert int(spill) == 0, f"{fn} spills {spill} B"
