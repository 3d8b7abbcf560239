"""Float64 restatement of the mutual-nearest-neighbour matchers (mnn.cu, mnn_tc.cu, mnn_fast.cu) with derived error bounds.

The operation (xfeat.py:327-348): S = F1 F2^T; row i's partner is the first column holding the row's maximum, column j's partner
the first row holding the column's maximum; (i, j) is returned when both agree, in ascending i, and, when min_cossim > 0, only
when S[i, j] > min_cossim (strict).  `Stats` computes that in float64, chunked over rows so that 32k x 32k fits on a GPU.

The split (split_kernel, split_norm_kernel; `split`): s = 2^(14 - e) with frexp(max|x|) = (m, e) -- max|x| is the caller's
abs_bound when given, else the measured maximum over the valid rows of both sets (of the whole batch in xfeat_mnn_match, of the
pair's two images in xfeat_mnn_match_pairs_f32) -- then a = x s (exact), hi = fp16_rn(a), lo = fp16_rn(a - hi), fp16 subnormals
included.  The presplit entry points take hi / lo rows the caller built at s = 2^scale_log2.

Bounds on |computed S - S| per entry (`bound`), in the units of x; P = |F1| |F2|^T and A1_i = sum_k |x1_ik| (likewise A2_j):

- Implementation 0 (mnn_scan_kernel): 64 fp32 FMAs from +0, round to nearest (u = 2^-24), so |err| <= gamma_64 P with
  gamma_n = n u / (1 - n u).  The min_cossim test of implementation 4 re-dots the two fp32 rows in the same order and has the same
  bound (`thr_bound`).
- Implementations 1-4 and the presplit paths: S s^2 is the fp32 sum of the 192 products hi.hi, hi.lo, lo.hi, each exact in fp32
  (11 x 11 significand bits).  Write a = hi + lo + r.  Per element, in scaled units:
      |a - hi| <= 2^-11 |a| + 2^-25     (half an fp16 ulp, or half the subnormal spacing 2^-24)
      |r|      <= 2^-22 |a| + 2^-24,     |lo| <= 1.001 * 2^-11 |a| + 2^-23,     |hi| <= (1 + 2^-11) |a| + 2^-25.
  The exact product minus the three kept terms is hi1 r2 + r1 hi2 + lo1 lo2 + lo1 r2 + r1 lo2 + r1 r2, so the representation
  error (dropped lo.lo included) is at most 3.01 * 2^-22 P s^2 + 2^-23 (A1 + A2) s + 2^-38.  The 192 products sum to at most
  1.0025 P s^2 + 2^-22 (A1 + A2) s + 2^-38 in magnitude.  How wgmma rounds its fp32 accumulation on Hopper has not been measured:
  the bound assumes each of the 191 additions, in any order, truncates (u = 2^-23), so the accumulation adds gamma_191 times that
  magnitude.  The packed value is then multiplied by 2^-2(14-e) (exact).  Implementation 4 re-scores every row whose hi-only gap
  is within its filter's tau with the same three-term kernel, and keeps the hi-only arg-max elsewhere, which the filter proves
  is the three-term one: the same bound holds for its arg-max.
  Float64 S itself is off by at most 64 * 2^-53 P; 1e-13 P covers it.

`admissible` turns the bound into a verdict on a returned list.  Every entry's computed value is within B of S, so a returned
(i, j) must have S[i, j*] - S[i, j] <= B[i, j*] + B[i, j] for row i's float64 maximum j*, and likewise for its column; a row
whose runner-up cannot reach its maximum within the bounds (and the same for the column) has one possible answer.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import numpy as np
import torch

U_RN = 2.0 ** -24       # fp32 round to nearest
U_TR = 2.0 ** -23       # fp32 truncation (the assumption for wgmma accumulation)
TERMS = ("hi.hi", "hi.lo", "lo.hi")


def gamma(n: int, u: float) -> float:
    return n * u / (1.0 - n * u)


def scale_log2_for(mx: float) -> int:
    """log2 of the operand scale the kernels choose for max |x| = mx (0 when mx = 0)."""
    mx = float(np.float32(mx))
    if not mx > 0:
        return 0
    return 14 - math.frexp(mx)[1]


def valid_absmax(f: torch.Tensor, counts) -> float:
    """max |x| over the first counts[b] rows of each f[b] (counts None: all rows), as absmax_kernel measures it."""
    m = 0.0
    for b in range(f.shape[0]):
        n = f.shape[1] if counts is None else max(0, min(int(counts[b]), f.shape[1]))
        if n:
            m = max(m, float(f[b, :n].abs().max()))
    return m


def split(x: torch.Tensor, scale_log2: int):
    """(hi, lo) fp16 tensors of x * 2^scale_log2, as split_kernel builds them (the product in fp32 is exact)."""
    a = x.float() * (2.0 ** scale_log2)
    hi = a.half()
    lo = (a - hi.float()).half()
    return hi, lo


def emulate(f1: torch.Tensor, f2: torch.Tensor, scale_log2: int, terms=TERMS) -> torch.Tensor:
    """S from the selected split terms, summed exactly (float64), in the units of x."""
    h1, l1 = (t.double() for t in split(f1, scale_log2))
    h2, l2 = (t.double() for t in split(f2, scale_log2))
    ops = {"hi.hi": (h1, h2), "hi.lo": (h1, l2), "lo.hi": (l1, h2)}
    acc = torch.zeros(f1.shape[0], f2.shape[0], dtype=torch.float64, device=f1.device)
    for t in terms:
        acc = acc + ops[t][0] @ ops[t][1].t()
    return acc * 2.0 ** (-2 * scale_log2)


def bound(impl: int, scale_log2: int = 0) -> Callable[[torch.Tensor, torch.Tensor], torch.Tensor]:
    """B(a, b) -> (len(a), len(b)) float64 bound on |computed S - S| for the arg-max of `impl` (see the module docstring)."""
    def b0(a, b):
        p = a.double().abs() @ b.double().abs().t()
        return (gamma(64, U_RN) + 1e-13) * p

    def b3(a, b):
        s = 2.0 ** scale_log2
        ad, bd = a.double().abs(), b.double().abs()
        p = (ad @ bd.t()) * (s * s)
        sa, sb = ad.sum(1)[:, None] * s, bd.sum(1)[None, :] * s
        rep = 3.01 * 2.0 ** -22 * p + 2.0 ** -23 * (sa + sb) + 2.0 ** -38
        mag = 1.0025 * p + 2.0 ** -22 * (sa + sb) + 2.0 ** -38
        return (rep + gamma(191, U_TR) * mag) / (s * s) + 1e-13 * p / (s * s)
    return b0 if impl == 0 else b3


def thr_bound(impl: int, scale_log2: int = 0):
    """Bound on the value the min_cossim test compares: the fp32 re-dot for implementation 4, the packed value otherwise."""
    return bound(0) if impl in (0, 4) else bound(impl, scale_log2)


def _first_argmax(s: torch.Tensor, dim: int):
    m = s.max(dim, keepdim=True).values
    n = s.shape[dim]
    shape = [1, 1]
    shape[dim] = n
    ar = torch.arange(n, device=s.device).reshape(shape)
    idx = torch.where(s == m, ar, torch.full_like(ar, n)).min(dim).values
    return m.squeeze(dim), idx


class Stats:
    """Row and column maxima of S in float64 with their first indices, the bound there, and which rows / columns are ambiguous
    (a competitor within the bounds).  f1 (n1, 64), f2 (n2, 64), on any device."""

    def __init__(self, f1: torch.Tensor, f2: torch.Tensor, B: Callable, chunk: int = 4096):
        self.f1, self.f2, self.B = f1, f2, B
        n1, n2 = f1.shape[0], f2.shape[0]
        dev = f1.device
        f2d = f2.double()
        rm, ra, rb, ramb = [], [], [], []
        cmax = torch.full((n2,), -math.inf, dtype=torch.float64, device=dev)
        carg = torch.zeros(n2, dtype=torch.long, device=dev)
        cb = torch.zeros(n2, dtype=torch.float64, device=dev)
        t1 = torch.full((n2,), -math.inf, dtype=torch.float64, device=dev)
        t1i = torch.full((n2,), -1, dtype=torch.long, device=dev)
        t2 = torch.full((n2,), -math.inf, dtype=torch.float64, device=dev)
        for r0 in range(0, n1, chunk):
            a = f1[r0:r0 + chunk]
            s = a.double() @ f2d.t()
            bb = B(a, f2)
            m, j = _first_argmax(s, 1)
            bj = bb.gather(1, j[:, None])[:, 0]
            t = s + bb
            t.scatter_(1, j[:, None], -math.inf)
            rm.append(m), ra.append(j), rb.append(bj)
            ramb.append(t.max(1).values >= m - bj)
            # columns: running first maximum and the two largest S + B with their rows
            m2, i2 = _first_argmax(s, 0)
            upd = m2 > cmax
            cmax = torch.where(upd, m2, cmax)
            carg = torch.where(upd, i2 + r0, carg)
            cb = torch.where(upd, bb.gather(0, i2[None, :])[0], cb)
            t = s + bb
            k = min(2, t.shape[0])
            tv, ti = t.topk(k, 0)
            cv = torch.cat([t1[None], t2[None], tv], 0)
            ci = torch.cat([t1i[None], torch.full_like(t1i, -1)[None], ti + r0], 0)
            v, o = cv.topk(2, 0)
            t1, t2, t1i = v[0], v[1], ci.gather(0, o[:1])[0]
        self.row_max, self.row_arg, self.row_b = torch.cat(rm), torch.cat(ra), torch.cat(rb)
        self.row_amb = torch.cat(ramb)
        self.col_max, self.col_arg, self.col_b = cmax, carg, cb
        excl = torch.where(t1i == carg, t2, t1)
        self.col_amb = excl >= cmax - cb

    def mutual(self):
        """Float64 mutual pairs (idx0 ascending)."""
        n1 = self.row_arg.shape[0]
        i = torch.arange(n1, device=self.row_arg.device)
        keep = self.col_arg[self.row_arg] == i
        return i[keep], self.row_arg[keep]


def _diag_bound(Bfn, a, b):
    """Bound of the pairs (a[k], b[k]) only: B on the diagonal, without forming the full block."""
    out = []
    for k0 in range(0, a.shape[0], 2048):
        blk = Bfn(a[k0:k0 + 2048], b[k0:k0 + 2048])
        out.append(torch.diagonal(blk))
    return torch.cat(out) if out else torch.zeros(0, dtype=torch.float64, device=a.device)


def reference(f1: torch.Tensor, f2: torch.Tensor, min_cossim: float):
    """Exact float64 MNN with torch's tie rule and the strict threshold (applied when min_cossim > 0): (idx0, idx1) int64."""
    st = Stats(f1, f2, lambda a, b: torch.zeros(a.shape[0], b.shape[0], dtype=torch.float64, device=a.device))
    i, j = st.mutual()
    if min_cossim > 0 and len(i):
        s = (f1[i].double() * f2[j].double()).sum(1)
        k = s > min_cossim
        i, j = i[k], j[k]
    return i, j


def admissible(got0, got1, st: Stats, min_cossim: float, Bt: Optional[Callable] = None, exact: bool = False) -> float:
    """Checks a returned list (got0, got1) against the float64 statistics `st` (built with the arg-max bound); Bt bounds the
    thresholded value (default: st.B).  exact: the inputs make S exact in every implementation, so the list must equal the
    float64 one bit for bit.  Returns the worst error-to-bound ratio over the returned pairs: how far (in units of the allowance
    B + B) a returned partner's float64 value lies below its row's or column's maximum, or a kept value below the threshold."""
    dev = st.row_arg.device
    g0 = torch.as_tensor(got0, dtype=torch.long).to(dev)
    g1 = torch.as_tensor(got1, dtype=torch.long).to(dev)
    n1, n2 = st.row_arg.shape[0], st.col_arg.shape[0]
    assert g0.shape == g1.shape, "idx0 / idx1 lengths differ"
    if len(g0):
        assert int(g0.min()) >= 0 and int(g0.max()) < n1, "idx0 out of range"
        assert int(g1.min()) >= 0 and int(g1.max()) < n2, "idx1 out of range"
        assert bool((g0[1:] > g0[:-1]).all()), "idx0 not strictly ascending"
    w0, w1 = st.mutual()
    thr_on = min_cossim > 0
    if exact:
        if thr_on and len(w0):
            s = (st.f1[w0].double() * st.f2[w1].double()).sum(1)
            k = s > min_cossim
            w0, w1 = w0[k], w1[k]
        assert torch.equal(g0, w0) and torch.equal(g1, w1), \
            f"exact case: {len(g0)} pairs returned, float64 has {len(w0)}; first differences " \
            f"{sorted(set(zip(g0.tolist(), g1.tolist())) ^ set(zip(w0.tolist(), w1.tolist())))[:6]}"
        return 0.0
    worst = 0.0
    if len(g0):
        a, b = st.f1[g0], st.f2[g1]
        s = (a.double() * b.double()).sum(1)
        bij = _diag_bound(st.B, a, b)
        # row: the returned column against the row's float64 maximum
        jr = st.row_arg[g0]
        allow_r = bij + st.row_b[g0]
        def_r = st.row_max[g0] - s
        # column: the returned row against the column's float64 maximum
        allow_c = bij + st.col_b[g1]
        def_c = st.col_max[g1] - s
        bad = (def_r > allow_r) | (def_c > allow_c)
        if bool(bad.any()):
            k = int(torch.nonzero(bad)[0, 0])
            raise AssertionError(f"pair ({int(g0[k])}, {int(g1[k])}) not admissible: row max {float(st.row_max[g0[k]]):.9g} at "
                                 f"{int(jr[k])}, column max {float(st.col_max[g1[k]]):.9g} at {int(st.col_arg[g1[k]])}, "
                                 f"S {float(s[k]):.9g}, B {float(bij[k]):.3e}")
        r = torch.maximum(def_r / allow_r.clamp_min(1e-300), def_c / allow_c.clamp_min(1e-300)).clamp_min(0)
        worst = max(worst, float(r.max()))
        if thr_on:
            bt = _diag_bound(Bt or st.B, a, b)
            below = s + bt <= min_cossim
            if bool(below.any()):
                k = int(torch.nonzero(below)[0, 0])
                raise AssertionError(f"pair ({int(g0[k])}, {int(g1[k])}) kept at S {float(s[k]):.9g} <= threshold "
                                     f"{min_cossim:.9g} - B {float(bt[k]):.3e}")
            d = ((min_cossim - s) / bt.clamp_min(1e-300)).clamp_min(0)
            worst = max(worst, float(d.max()))
    # every unambiguous float64 pair above the threshold band must be there, with that partner
    sure = ~st.row_amb[w0] & ~st.col_amb[w1]
    w0, w1 = w0[sure], w1[sure]
    if thr_on and len(w0):
        a, b = st.f1[w0], st.f2[w1]
        s = (a.double() * b.double()).sum(1)
        bt = _diag_bound(Bt or st.B, a, b)
        k = s - bt > min_cossim
        w0, w1 = w0[k], w1[k]
    part = torch.full((n1,), -1, dtype=torch.long, device=dev)
    part[g0] = g1
    miss = part[w0] != w1
    if bool(miss.any()):
        k = int(torch.nonzero(miss)[0, 0])
        raise AssertionError(f"unambiguous float64 pair ({int(w0[k])}, {int(w1[k])}) returned as "
                             f"{int(part[w0[k]])} ({int(miss.sum())} such rows)")
    return worst


def filter_tau(nh: float, nl: float, hmax: float, lmax: float, k: float = 2.1) -> float:
    """Implementation 4's filter threshold (mnn_fast.cu, mnn_fast_kernel) in float64, scaled units: a row whose hi-only top-1 /
    top-2 gap exceeds it keeps its hi-only arg-max.  nh, nl: ||hi||, ||lo|| of the row; hmax, lmax: the largest ||hi||, ||lo||
    over the other set.  The kernel rounds its norms up by 1.0001 before this.  k: the factor on the Cauchy-Schwarz term."""
    return k * (nh * lmax + nl * hmax) + 6.2e-5 * nh * hmax


def filter_rows(f_rows: torch.Tensor, f_cols: torch.Tensor, scale_log2: int, n_rows: int, n_cols: int, k: float = 2.1):
    """For each of the first n_rows rows: the hi-only top-1 / top-2 gap and its tau (scaled units), as mnn_fast_kernel sees them
    against the first n_cols rows of the other set.  Returns (gap, tau, hi-only arg-max) float64 / int64 tensors."""
    h1, l1 = (t.double() for t in split(f_rows[:n_rows], scale_log2))
    h2, l2 = (t.double() for t in split(f_cols[:n_cols], scale_log2))
    st = h1 @ h2.t()
    top = st.topk(2, 1) if n_cols > 1 else None
    gap = (top.values[:, 0] - top.values[:, 1]) if top is not None else torch.full((n_rows,), math.inf, dtype=torch.float64)
    nh, nl = h1.norm(dim=1) * 1.0001, l1.norm(dim=1) * 1.0001
    hmax, lmax = float(h2.norm(dim=1).max()) * 1.0001, float(l2.norm(dim=1).max()) * 1.0001
    tau = torch.tensor([filter_tau(float(a), float(b), hmax, lmax, k) for a, b in zip(nh, nl)], dtype=torch.float64)
    return gap, tau, _first_argmax(st, 1)[1]


# hi-only x component of the filter-border gadgets: 410 flips the hi-only arg-max with a gap 1.7x the Cauchy-Schwarz term, 600
# keeps it just inside tau, 800 and 1024 put it just outside (see filter_border_sets)
BORDER_ALPHAS = (410.0, 600.0, 800.0, 1024.0)
BORDER_SCALE_LOG2 = 13     # abs_bound 1.0


def filter_border_sets(n1: int = 700, n2: int = 600, seed: int = 0):
    """Two descriptor sets (n1, 64), (n2, 64) in [-1, 1] whose rows sit on both sides of implementation 4's filter, in both
    directions.  In units of 2^-13 (the scale abs_bound = 1 selects), gadget g of direction 0 uses components (2g, 2g + 1):
        row g of set 1:            (alpha_g, 1024)                         hi only (lo = 0)
        rows 2g, 2g + 1 of set 2:  (4100, 2050.875), (4104, 2049.125)       hi (4100, 2050), (4104, 2050); lo (0, +-0.875)
    The hi-only scan prefers row 2g + 1 by 4 alpha_g; the exact values prefer row 2g by 1.75 * 1024 - 4 alpha_g.  With ||lo||max =
    0.875 and ||hi||max ~ 4588 over set 2, the gap 4 alpha_g is 1.7x the Cauchy-Schwarz term at alpha = 410 (so the hi-only arg-max is
    wrong, and only the factor 2.1 sends the row to the re-scoring pass), inside tau at 600 and outside it at 800 and 1024.
    Direction 1 mirrors this in components 8 + (2g, 2g + 1) with the roles of the sets swapped.  The other rows are integer
    vectors (lo = 0) in components 16..63, orthogonal to every gadget.  Returns (f1, f2) float32 and the gadget rows
    {direction: [(row, exact partner, hi-only partner)]}."""
    g = torch.Generator().manual_seed(seed)
    s = 2.0 ** -BORDER_SCALE_LOG2
    f1 = torch.zeros(n1, 64, dtype=torch.float64)
    f2 = torch.zeros(n2, 64, dtype=torch.float64)
    f1[:, 16:] = torch.randint(-200, 201, (n1, 48), generator=g).double()
    f2[:, 16:] = torch.randint(-200, 201, (n2, 48), generator=g).double()
    rows = {0: [], 1: []}
    ng = len(BORDER_ALPHAS)
    for d, (fa, fb) in enumerate(((f1, f2), (f2, f1))):
        for k, alpha in enumerate(BORDER_ALPHAS):
            c = 8 * d + 2 * k
            r, p = 2 * ng + k, 2 * k          # the single row follows the other direction's pairs; its pair is rows p, p + 1
            fa[r] = 0
            fa[r, c], fa[r, c + 1] = alpha, 1024.0
            for q, row in ((p, (4100.0, 2050.875)), (p + 1, (4104.0, 2049.125))):
                fb[q] = 0
                fb[q, c], fb[q, c + 1] = row
            rows[d].append((r, p, p + 1))
    return (f1 * s).float(), (f2 * s).float(), rows
