"""LighterGlue's stages (csrc/lighterglue.cu) against float64 at the ragged and tile-edge counts of tests/lg_edge_cases.py: the
descriptors after 0, 1 and 6 layers, the assignment's row and column maxima and arg-maxima (also the assignment kernel alone on
synthetic descriptors), the match filter (exactly, against
the plain-numpy rule applied to the same run's assignment), first-index ties between duplicated points, padding and counts,
and pruning at the threshold's edges.  Bounds: tests/test_lighterglue_edges_ref.py (each >= 5x the float32 oracle's error)."""
import numpy as np
import pytest
import torch

from oracle import lighterglue_oracle as lo
from tests import lg_edge_cases as E
from tests.test_gpu_lighterglue import _debug, _dev
from tests.test_lighterglue_edges_ref import case_tol
from tests.test_lighterglue_oracle import LAYER_TOL, NEAR_TIE_EPS, load_case, match_set_diff, near_tie

pytestmark = pytest.mark.gpu

N_OVERFLOW = -1          # XF_N_OVERFLOW


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    from oracle import build_lighterglue
    return XFeat(device=0, lighterglue_weights=build_lighterglue.path())


@pytest.fixture(scope="module")
def sd():
    return lo.load_state()


@pytest.fixture(scope="module")
def oracle64(sd):
    """case name -> {n_layers: float64 oracle result}, computed on first use."""
    cache = {}

    def get(name, n_layers):
        if (name, n_layers) not in cache:
            cache[name, n_layers] = lo.match(sd, *E.case_args(name), dtype=np.float64, n_layers=n_layers)
        return cache[name, n_layers]
    return get


def dev_args(arrays):
    return tuple(_dev(a, torch.int32) if a.dtype == np.int32 else _dev(a) for a in arrays)


def run_debug(xf, pairs, n_max, n_layers, prune=None, fill=0.0, counts=None):
    """xfeat_lg_debug on host pairs; `counts` (n0, n1) overrides the point counts passed to the kernel."""
    a = list(E.batch_arrays(pairs, n_max, fill))
    if counts is not None:
        a[2], a[6] = np.asarray(counts[0], np.int32), np.asarray(counts[1], np.int32)
    return _debug(xf, dev_args(a), n_max, n_layers, prune, want_assign=n_layers == 6)


def run_match(xf, pairs, n_max, min_conf=0.1, prune=None, fill=0.0, counts=None):
    a = list(E.batch_arrays(pairs, n_max, fill))
    if counts is not None:
        a[2], a[6] = np.asarray(counts[0], np.int32), np.asarray(counts[1], np.int32)
    out = xf.match_lighterglue_batch(*dev_args(a), min_conf=min_conf, prune_min_points=prune)
    return tuple(t.cpu().numpy() for t in out)


def pair_matches(res, b):
    i0, i1, sc, nm = res
    n = max(int(nm[b]), 0)
    return i0[b, :n], i1[b, :n], sc[b, :n], int(nm[b])


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def assert_same_matches(got, want, what):
    for g, w in zip(got, want):
        assert same_bits(g, w), what


# --------------------------------------------------------------------------------------------------------------------------------
# a. layers
# --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_layers", [0, 1, 6])
def test_layers_vs_float64_edges(xf, sd, oracle64, n_layers):
    """Descriptors after 0, 1 and 6 layers (no pruning), both sides of every case, in one batch at n_max = 1937 and alone at the
    case's own n_max; the two runs must agree bit for bit (a row's arithmetic does not depend on where its tile sits)."""
    pairs = [E.case_args(c) for c in E.CASES]
    xb, indb, cntb, _, _ = run_debug(xf, pairs, E.N_MAX_ALL, n_layers)
    m = lo._Model(sd, np.float64)
    for b, c in enumerate(E.CASES):
        xs, inds, cnts, _, _ = run_debug(xf, [pairs[b]], c.n_max, n_layers)
        if n_layers == 0:
            want = [m.lin("input_proj", pairs[b][3 * s + 1].astype(np.float64)) for s in range(2)]
            tol = LAYER_TOL[0]
        else:
            want = oracle64(c.name, n_layers)["x"]
            tol = case_tol(c.name, f"layer{n_layers}")
        for s, n in enumerate((c.n0, c.n1)):
            assert cntb[s, b] == n and cnts[s, 0] == n
            assert (indb[s, b, :n] == np.arange(n)).all() and (inds[s, 0, :n] == np.arange(n)).all()
            err = np.abs(xb[s, b, :n] - want[s]).max()
            print(f"{c.name} layers={n_layers} side {s}: max err {err:.3g} (bound {tol:.3g})")
            assert err <= tol, (c.name, s)
            assert same_bits(xb[s, b, :n], xs[s, 0, :n]), (c.name, s, "batch != single")


# --------------------------------------------------------------------------------------------------------------------------------
# b. assignment
# --------------------------------------------------------------------------------------------------------------------------------
def test_assignment_vs_float64_edges(xf, oracle64):
    """Row and column maxima (as scores exp(best)) and arg-maxima after layer 6 against float64, every case, batch and single;
    an arg-max may differ only where float64's top-2 gap is below NEAR_TIE_EPS."""
    pairs = [E.case_args(c) for c in E.CASES]
    _, _, _, best, arg = run_debug(xf, pairs, E.N_MAX_ALL, 6)
    for b, c in enumerate(E.CASES):
        _, _, _, best1, arg1 = run_debug(xf, [pairs[b]], c.n_max, 6)
        r = oracle64(c.name, 6)
        tol = case_tol(c.name, "score")
        for s, n, key in ((0, c.n0, "row"), (1, c.n1, "col")):
            assert same_bits(best[s, b, :n], best1[s, 0, :n]) and same_bits(arg[s, b, :n], arg1[s, 0, :n]), (c.name, s)
            err = np.abs(np.exp(best[s, b, :n].astype(np.float64)) - np.exp(r[f"{key}_max"])).max()
            bad = np.nonzero(arg[s, b, :n] != r[f"{key}_arg"])[0]
            print(f"{c.name} {key}s: score err {err:.3g} (bound {tol:.3g}), {len(bad)} arg-max differ")
            assert err <= tol, (c.name, key)
            assert (r[f"{key}_gap"][bad] < NEAR_TIE_EPS).all(), (c.name, key, bad)


ASSIGN_COUNTS = [(1, 1), (2, 3), (3, 2), (63, 65), (64, 64), (65, 63), (130, 97), (0, 5)]
ASSIGN_TOL = 5e-5        # lse and best (log space) of the synthetic rows below: 96-term fp32 dot products of size < 5


def test_assign_kernel_vs_float64_synthetic(xf):
    """The assignment kernel alone (xfeat_lg_debug_assign) on synthetic descriptors whose similarities are O(1), at ragged
    counts with n_max = 130, against float64: lse, best and the first arg-max, with duplicated key rows tying inside and across
    64-row tiles.  The model's own descriptors give S >= 45 on every row's maximum, where a key row wrongly left in the
    log-sum-exp with S = 0 changes nothing in fp32; here it changes lse by O(1)."""
    from accelerated_features_b200 import _lib
    rs = np.random.RandomState(3)
    B, n_max = len(ASSIGN_COUNTS), 130
    md = np.zeros((2, B, n_max, 96), np.float32)
    lz = np.zeros((2, B, n_max), np.float32)
    cnt = np.array(ASSIGN_COUNTS, np.int32).T.copy()
    for b in range(B):
        for s in range(2):
            n = cnt[s, b]
            md[s, b, :n] = rs.randn(n, 96) * 0.35
            lz[s, b, :n] = -3 * rs.rand(n)
        if cnt[1, b] >= 97:           # rows 3 and 10 match each other across the pair, and each has a copy: inside tile 0 (row
            for src, dst in ((3, 9), (10, 80)):          # 9) and in tile 1 (row 80), so their maxima tie between two indices
                md[1, b, src] = md[0, b, src]
                md[1, b, dst], lz[1, b, dst] = md[1, b, src], lz[1, b, src]
                md[0, b, dst], lz[0, b, dst] = md[0, b, src], lz[0, b, src]
    out = [torch.zeros((2, B, n_max), device="cuda") for _ in range(2)] + [torch.full((2, B, n_max), -7, dtype=torch.int32,
                                                                                      device="cuda")]
    dmd, dlz, dcnt = _dev(md), _dev(lz), _dev(cnt, torch.int32)
    _lib.check(xf._lib.xfeat_lg_debug_assign(dmd.data_ptr(), dlz.data_ptr(), dcnt.data_ptr(), B, n_max,
                                             *[t.data_ptr() for t in out], torch.cuda.current_stream().cuda_stream),
               "xfeat_lg_debug_assign")
    lse, best, arg = (t.cpu().numpy() for t in out)
    n_dup = 0
    for b in range(B):
        n0, n1 = cnt[:, b]
        if n0 == 0 or n1 == 0:
            assert (arg[:, b] == -7).all()            # nothing to assign: outputs untouched
            continue
        m0, m1 = md[0, b, :n0].astype(np.float64), md[1, b, :n1].astype(np.float64)
        S = (m0[:, None, :] * m1[None, :, :]).sum(-1)           # per element: copied rows give identical columns
        l0, l1 = np.logaddexp.reduce(S, 1), np.logaddexp.reduce(S, 0)
        sc = (S - l0[:, None]) + (S - l1[None, :]) + (lz[0, b, :n0, None].astype(np.float64) + lz[1, b, None, :n1])
        for s, (lw, a) in enumerate(((l0, sc), (l1, sc.T))):
            n = len(lw)
            err_l = np.abs(lse[s, b, :n] - lw).max()
            err_b = np.abs(best[s, b, :n] - a.max(1)).max()
            srt = -np.sort(-a, 1)
            gap = srt[:, 0] - srt[:, 1] if a.shape[1] > 1 else np.full(n, np.inf)
            first = a.argmax(1)
            tie = np.abs(gap) == 0
            bad = np.nonzero((arg[s, b, :n] != first) & (gap >= NEAR_TIE_EPS) | (arg[s, b, :n] != first) & tie)[0]
            n_dup += int(tie.sum())
            print(f"counts {(n0, n1)} side {s}: lse err {err_l:.3g}, best err {err_b:.3g} (bound {ASSIGN_TOL:.3g}), "
                  f"{int(tie.sum())} exact ties")
            assert err_l <= ASSIGN_TOL and err_b <= ASSIGN_TOL, (n0, n1, s)
            assert len(bad) == 0, (n0, n1, s, bad)
    assert n_dup >= 2


# --------------------------------------------------------------------------------------------------------------------------------
# c. the match filter
# --------------------------------------------------------------------------------------------------------------------------------
def test_match_filter_exact(xf):
    """match_lighterglue_batch's matches equal finalize_rule applied to the same run's assignment (xfeat_lg_debug), at min_conf
    0, 0.1 and a score the run produces; scores are within 2 ulp of exp(best) and idx0 strictly ascending.  Against the run's
    own scores the threshold is exact: a match whose score equals min_conf is dropped (the test is score > min_conf)."""
    pairs = [E.case_args(c) for c in E.CASES]
    n_max = E.N_MAX_ALL
    _, ind, cnt, best, arg = run_debug(xf, pairs, n_max, 6)
    base = run_match(xf, pairs, n_max, min_conf=0.0)
    big = E.CASE_IDS.index("1536x1537")
    sc_big = np.sort(pair_matches(base, big)[2])
    at = float(sc_big[len(sc_big) // 2])
    for mc in (0.0, 0.1, at):
        res = run_match(xf, pairs, n_max, min_conf=mc)
        rule = E.finalize_rule(best, arg, ind, cnt, mc)
        n_excused = 0
        for b, c in enumerate(E.CASES):
            i0, i1, sc, nm = pair_matches(res, b)
            assert nm >= 0 and (np.diff(i0) > 0).all(), c.name
            row = np.searchsorted(ind[0, b, :cnt[0, b]], i0)
            want_sc = np.exp(best[0, b, row].astype(np.float64))
            assert (np.abs(sc - want_sc) <= 2 * np.spacing(want_sc.astype(np.float32))).all(), c.name
            # rule vs kernel, excusing rows whose score is within 1e-6 of min_conf (expf and numpy's exp may round apart)
            near = set(np.nonzero(np.abs(np.exp(best[0, b, :cnt[0, b]].astype(np.float64)) - mc) <= 1e-6)[0].tolist())
            n_excused += len(near)
            got = {int(i): int(j) for i, j in zip(i0, i1) if i not in near}
            want = {int(i): int(j) for i, j in zip(rule[b][0], rule[b][1]) if i not in near}
            assert got == want, (c.name, mc, match_set_diff(list(got), list(got.values()), list(want), list(want.values())))
            # exact, against the kernel's own scores at min_conf 0 (same inputs, same bits)
            b0, b1, bs, _ = pair_matches(base, b)
            keep = bs > np.float32(mc)
            assert same_bits(i0, b0[keep]) and same_bits(i1, b1[keep]) and same_bits(sc, bs[keep]), (c.name, mc)
        print(f"min_conf {mc:.9g}: {int(res[3].clip(0).sum())} matches, {n_excused} rows excused")
    assert len(sc_big) > 10 and (sc_big == np.float32(at)).sum() >= 1
    assert len(pair_matches(run_match(xf, pairs, n_max, min_conf=at), big)[0]) < (sc_big >= np.float32(at)).sum()


# --------------------------------------------------------------------------------------------------------------------------------
# d. ties between duplicated points
# --------------------------------------------------------------------------------------------------------------------------------
# (source match of the 4096-point golden, positions of its two copies on side 0, on side 1): one pair of copies inside one 64-row
# tile, one across tiles, on each side
TIE_SLOTS = [(0, (5, 9), (7, 60)), (1, (20, 150), (30, 200)), (2, (70, 71), (130, 66))]
TIE_N = (230, 241)


def tie_case():
    """A pair built from the 4096-point asset pair with three confidently matched points duplicated (keypoint and descriptor) on
    both sides.  Returns the oracle arguments and the duplicate sets {side: [[lower, higher], ...]}."""
    g = load_case("lg_assets_4096")
    top = np.argsort(-g["scores"])[:3]
    src = [(int(g["idx0"][t]), int(g["idx1"][t])) for t in top]
    rs = np.random.RandomState(11)
    args, dups = [], {0: [], 1: []}
    for s, n in enumerate(TIE_N):
        used = {p[s] for p in src}
        rest = [i for i in rs.permutation(4096) if i not in used]
        rows = [None] * n
        for k, (_, *pos) in enumerate(TIE_SLOTS):
            for p in pos[s]:
                rows[p] = src[k][s]
            dups[s].append(sorted(pos[s]))
        free = [p for p in range(n) if rows[p] is None]
        for p, i in zip(free, sorted(rest[:len(free)])):
            rows[p] = i
        args += [g[f"kpts{s}"][rows], g[f"desc{s}"][rows], tuple(float(v) for v in g[f"size{s}"])]
    return tuple(args), dups


def score_matrix64(sd, x):
    """The float64 log-assignment of final descriptors x = (x0, x1)."""
    m = lo._Model(sd, np.float64)
    md = [m.lin("log_assignment.5.final_proj", v) / 96 ** 0.25 for v in x]
    z = [m.matchability(5, v) for v in x]
    S = md[0] @ md[1].T
    return lo._logsoftmax(S, 1) + lo._logsoftmax(S, 0) + (lo._logsigmoid(z[0])[:, None] + lo._logsigmoid(z[1])[None, :])


def test_duplicate_points_tie_to_lowest_index(xf, sd):
    """Duplicated points keep bit-identical descriptors through six layers wherever their rows sit; a row or column whose float64
    maximum falls on a duplicate set (away from any other near-tie) takes the set's lowest index; no match goes to a higher copy."""
    pair, dups = tie_case()
    n_max = max(TIE_N)
    x, _, cnt, best, arg = run_debug(xf, [pair], n_max, 6)
    for s in range(2):
        for lo_, hi in dups[s]:
            assert same_bits(x[s, 0, lo_], x[s, 0, hi]), (s, lo_, hi)
            assert same_bits(best[s, 0, lo_], best[s, 0, hi]) and arg[s, 0, lo_] == arg[s, 0, hi], (s, lo_, hi)
    r = lo.match(sd, *pair, dtype=np.float64)
    sc = score_matrix64(sd, r["x"])
    checked = 0
    for s in range(2):
        m = sc if s == 0 else sc.T                    # queries of side s against keys of the other side
        for q in range(TIE_N[s]):
            top = int(np.argmax(m[q]))
            for group in dups[1 - s]:
                if top not in group:
                    continue
                others = np.delete(m[q], group)
                if m[q, top] - others.max() < NEAR_TIE_EPS:
                    continue
                assert arg[s, 0, q] == min(group), (s, q, group, arg[s, 0, q])
                checked += 1
    print(f"{checked} rows / columns tie on a duplicate set")
    assert checked >= 2 * len(TIE_SLOTS)
    i0, i1, _, nm = pair_matches(run_match(xf, [pair], n_max, min_conf=0.0), 0)
    higher = [{g[1] for g in dups[s]} for s in range(2)]
    assert nm > 0 and not set(i0.tolist()) & higher[0] and not set(i1.tolist()) & higher[1]
    assert all((g[0], h[0]) in set(zip(i0.tolist(), i1.tolist())) for g, h in zip(dups[0], dups[1])), "copies must match"


# --------------------------------------------------------------------------------------------------------------------------------
# e. padding and counts
# --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prune", [None, 1536])
def test_nan_padding_gives_zero_padding_bits(xf, prune):
    """Rows past each count filled with NaN give the same bits as zero padding: no kernel reads a padding row."""
    pairs = [E.case_args(c) for c in E.CASES]
    n_max = E.N_MAX_ALL
    for n_layers in ((1, 6) if prune is None else (3,)):
        a = run_debug(xf, pairs, n_max, n_layers, prune, fill=0.0)
        z = run_debug(xf, pairs, n_max, n_layers, prune, fill=np.nan)
        assert same_bits(a[2], z[2])
        for b in range(len(pairs)):
            for s in range(2):
                n = a[2][s, b]
                assert same_bits(a[0][s, b, :n], z[0][s, b, :n]) and same_bits(a[1][s, b, :n], z[1][s, b, :n]), (b, s)
                assert np.isfinite(a[0][s, b, :n]).all()
                if n_layers == 6:
                    assert same_bits(a[3][s, b, :n], z[3][s, b, :n]) and same_bits(a[4][s, b, :n], z[4][s, b, :n]), (b, s)
    a, z = run_match(xf, pairs, n_max, 0.0, prune, 0.0), run_match(xf, pairs, n_max, 0.0, prune, np.nan)
    assert same_bits(a[3], z[3])
    for b in range(len(pairs)):
        assert_same_matches(pair_matches(a, b)[:3], pair_matches(z, b)[:3], b)


def test_count_above_n_max_is_clamped(xf):
    """A count above n_max behaves as n_max (on either side or both)."""
    pair = E.case_args("64x64")
    want = run_match(xf, [pair], 64, 0.0)
    want_x = run_debug(xf, [pair], 64, 6)
    assert want[3][0] > 0
    for counts in (([69], [64]), ([64], [1000]), ([65], [65])):
        got = run_match(xf, [pair], 64, 0.0, counts=counts)
        assert_same_matches(pair_matches(got, 0), pair_matches(want, 0), counts)
        gx = run_debug(xf, [pair], 64, 6, counts=counts)
        assert (gx[2] == 64).all()
        for w, g in zip(want_x, gx):                 # every row is valid: count = n_max
            assert same_bits(w, g), counts


def test_overflow_count_is_reported_and_isolated(xf):
    """XF_N_OVERFLOW on either side reports XF_N_OVERFLOW for that pair; every other pair of the batch is bit-identical to its
    single-pair call."""
    pairs = [E.case_args(c) for c in E.CASES]
    n0 = np.array([c.n0 for c in E.CASES], np.int32)
    n1 = np.array([c.n1 for c in E.CASES], np.int32)
    n0[2], n1[5], n0[8], n1[8] = N_OVERFLOW, N_OVERFLOW, N_OVERFLOW, N_OVERFLOW
    for prune in (None, 1536):
        res = run_match(xf, pairs, E.N_MAX_ALL, 0.0, prune, counts=(n0, n1))
        assert [int(v) for v in res[3][[2, 5, 8]]] == [N_OVERFLOW] * 3
        for b, c in enumerate(E.CASES):
            if b in (2, 5, 8):
                continue
            one = run_match(xf, [pairs[b]], c.n_max, 0.0, prune)
            assert pair_matches(res, b)[3] == pair_matches(one, 0)[3] > 0, c.name
            assert_same_matches(pair_matches(res, b)[:3], pair_matches(one, 0)[:3], c.name)


def test_empty_side_gives_no_matches(xf):
    """(0, n) and (n, 0) give 0 matches, alone and beside non-empty pairs."""
    k0, d0, s0, k1, d1, s1 = E.case_args("700x1900")
    empty = [(k0[:0], d0[:0], s0, k1, d1, s1), (k0, d0, s0, k1[:0], d1[:0], s1)]
    full = E.case_args("65x63")
    for p in empty:
        assert pair_matches(run_match(xf, [p], E.N_MAX_ALL, 0.0), 0)[3] == 0
    res = run_match(xf, [empty[0], full, empty[1]], E.N_MAX_ALL, 0.0)
    assert res[3][0] == 0 and res[3][2] == 0 and res[3][1] > 0
    assert_same_matches(pair_matches(res, 1), pair_matches(run_match(xf, [full], 130, 0.0), 0), "beside empty pairs")


# --------------------------------------------------------------------------------------------------------------------------------
# f. pruning at the threshold's edges
# --------------------------------------------------------------------------------------------------------------------------------
def gpu_keep_sets(xf, pair, n_max, T):
    """The kernel's pruning decisions after layers 0..4 as keep masks over each side's points at that layer (None: not pruned),
    checking that each count is the number kept and that the surviving indices stay strictly ascending."""
    n = (len(pair[0]), len(pair[3]))
    inds = [np.arange(n[0]), np.arange(n[1])]
    keep_sets = []
    for layer in range(1, 6):
        _, ind, cnt, _, _ = run_debug(xf, [pair], n_max, layer, T)
        ks = []
        for s in range(2):
            new = ind[s, 0, :cnt[s, 0]]
            assert (np.diff(new) > 0).all() and np.isin(new, inds[s]).all(), (layer, s)
            k = np.isin(inds[s], new)
            assert k.sum() == cnt[s, 0]
            if len(inds[s]) <= T:
                assert k.all(), (layer, s, "an image at or below the threshold is not pruned")
                k = None
            ks.append(k)
            inds[s] = new
        keep_sets.append(ks)
    return keep_sets, inds


def test_prune_threshold_equal_to_count_is_unpruned(xf):
    """T equal to the largest count (1900) gives the same bits as prune_min_points=None; T one below it prunes that image."""
    pairs = [E.case_args(c) for c in E.CASES]
    T = max(max(c.n0, c.n1) for c in E.CASES)
    assert T == 1900
    want = run_match(xf, pairs, E.N_MAX_ALL, 0.0, None)
    got = run_match(xf, pairs, E.N_MAX_ALL, 0.0, T)
    assert same_bits(want[3], got[3])
    for b in range(len(pairs)):
        assert_same_matches(pair_matches(got, b), pair_matches(want, b), b)
    wx, gx = run_debug(xf, pairs, E.N_MAX_ALL, 6, None), run_debug(xf, pairs, E.N_MAX_ALL, 6, T)
    assert same_bits(wx[2], gx[2])
    b = E.CASE_IDS.index("700x1900")
    assert same_bits(wx[0][0, b, :700], gx[0][0, b, :700]) and same_bits(wx[0][1, b, :1900], gx[0][1, b, :1900])
    _, _, cnt, _, _ = run_debug(xf, pairs, E.N_MAX_ALL, 5, T - 1)
    print(f"T = {T - 1}: 700x1900 counts after five layers {cnt[:, b].tolist()}")
    assert cnt[1, b] < 1900 and cnt[0, b] == 700
    assert all(cnt[:, i].tolist() == [c.n0, c.n1] for i, c in enumerate(E.CASES) if i != b)


@pytest.mark.parametrize("case,T", [("1536x1537", 1536), ("1536x1537", 1535), ("700x1900", 699), ("700x1900", 700)])
def test_pruned_edges_vs_oracle(xf, sd, case, T):
    """Pruning with one image above T and the other at it (only the one above is pruned), and with both above: the kernel's keep
    sets equal keep_rule on float64 z except near-ties of sigmoid(z) at 0.05, and the float64 oracle replayed with the kernel's
    keep sets gives the kernel's matches up to near-ties."""
    c = E.BY_NAME[case]
    pair = E.case_args(c)
    keep_sets, inds = gpu_keep_sets(xf, pair, c.n_max, T)
    pruned = [any(ks[s] is not None and not ks[s].all() for ks in keep_sets) for s in range(2)]
    assert pruned == [c.n0 > T, c.n1 > T], pruned
    rep = lo.match(sd, *pair, keep_sets=keep_sets, dtype=np.float64)
    n_diff = 0
    for layer, (ks, zs) in enumerate(zip(keep_sets, rep["z"])):
        for s in range(2):
            if ks[s] is None:
                assert zs[s] is None
                continue
            bad = np.nonzero(lo.keep_rule(zs[s]) != ks[s])[0]
            n_diff += len(bad)
            p = 1 / (1 + np.exp(-zs[s][bad]))
            assert (np.abs(p - 0.05) < NEAR_TIE_EPS).all(), (layer, s, p)
    i0, i1, _, nm = pair_matches(run_match(xf, [pair], c.n_max, 0.1, T), 0)
    diff = match_set_diff(i0, i1, rep["idx0"], rep["idx1"])
    print(f"{case} T={T}: final counts {[len(i) for i in inds]}, {nm} matches, oracle {len(rep['idx0'])}, {len(diff)} differ, "
          f"{n_diff} keep decisions differ")
    pos = {int(v): i for i, v in enumerate(rep["ind"][0])}
    assert len(diff) <= 8
    for i in diff:
        assert i in pos and near_tie(rep, pos[i], 0.1), i
