"""CPU checks behind tests/test_gpu_lighterglue_edges.py: on every edge case of tests/lg_edge_cases.py the tolerances the GPU test
applies are at least 5x the float32 oracle's own error against float64, and the plain-numpy match filter reproduces the oracle's
matches.  Needs the staged matcher weights (oracle/build_lighterglue.py), no GPU."""
import numpy as np
import pytest

from oracle import lighterglue_oracle as lo
from tests import lg_edge_cases as E
from tests.test_lighterglue_oracle import LAYER_TOL, SCORE_TOL


@pytest.fixture(scope="module")
def sd():
    return lo.load_state()


def case_tol(name, kind):
    """The bound the GPU test applies to case `name`: 'layer1', 'layer6' or 'score'."""
    shared = {"layer1": LAYER_TOL[1], "layer6": LAYER_TOL[6], "score": SCORE_TOL}[kind]
    return E.CASE_TOL.get((name, kind), shared)


def test_case_table():
    for c in E.CASES:
        a = E.case_args(c)
        assert (len(a[0]), len(a[3])) == (c.n0, c.n1) and max(c.n0, c.n1) <= c.n_max <= E.N_MAX_ALL
        assert a[1].shape == (c.n0, 64) and a[4].shape == (c.n1, 64) and np.isfinite(a[1]).all()
    assert E.N_MAX_ALL % 64 == 17
    geo = [c.geometry for c in E.CASES]
    assert all(geo.count(g) >= 2 for g in ("asset", "portrait", "mixed", "corners"))
    k0, _, (W, H), *_ = E.case_args("700x1900")
    assert [[0, 0], [W, H], [W, 0], [0, H]] == k0[:4].tolist() and ((k0 < 0) | (k0 > [W, H])).any()
    _, _, s0, _, _, s1 = E.case_args("65x63")
    assert s0 != s1
    _, _, (W, H), *_ = E.case_args("64x64")
    assert H > W
    for c in E.CASE_TOL:
        assert c[0] in E.BY_NAME and E.CASE_TOL[c] > {"layer1": LAYER_TOL[1], "layer6": LAYER_TOL[6], "score": SCORE_TOL}[c[1]]


def test_padder_and_batch():
    a = np.arange(6, dtype=np.float32).reshape(3, 2)
    p = E.pad(a, 5, np.nan)
    assert np.array_equal(p[:3], a) and np.isnan(p[3:]).all()
    assert (E.pad(a, 5)[3:] == 0).all()
    pairs = [E.case_args("2x3"), E.case_args("1x1")]
    k0, d0, n0, s0, k1, d1, n1, s1 = E.batch_arrays(pairs, 64, np.nan)
    assert k0.shape == (2, 64, 2) and d1.shape == (2, 64, 64) and n0.tolist() == [2, 1] and n1.tolist() == [3, 1]
    assert np.isnan(d0[0, 2:]).all() and np.isnan(k1[1, 1:]).all() and np.array_equal(d1[0, :3], pairs[0][4])
    assert s0.shape == (2, 2) and s0[0].tolist() == list(pairs[0][2])


def test_finalize_rule_strict_threshold_and_mapping():
    best = np.log(np.array([[[0.5, 0.25, 0.75, 0.9]], [[0, 0, 0, 0]]], np.float32))
    arg = np.array([[[1, 0, 2, 2]], [[1, 0, 1, 0]]], np.int32)
    ind = np.array([[[3, 5, 8, 9]], [[10, 11, 12, 13]]], np.int32)
    cnt = np.array([[4], [4]])
    i0, i1, sc = E.finalize_rule(best, arg, ind, cnt, 0.0)[0]
    assert i0.tolist() == [3, 5] and i1.tolist() == [11, 10]          # rows 2, 3: not mutual
    i0, _, _ = E.finalize_rule(best, arg, ind, cnt, float(np.exp(best[0, 0, 1])))[0]
    assert i0.tolist() == [3]                                       # exp(best) == min_conf is not a match
    assert E.finalize_rule(best, arg, ind, np.array([[4], [0]]), 0.0)[0][0].size == 0


@pytest.mark.parametrize("case", E.CASE_IDS)
def test_edge_tolerances_cover_fp32(sd, case):
    """LAYER_TOL after 1 and 6 layers and SCORE_TOL (or the case's own bound) are >= 5x the float32 oracle's error against
    float64, in the form of test_layer_tolerances_cover_fp32 / test_score_tolerance_covers_fp32."""
    a = E.case_args(case)
    for n in (1, 6):
        r32 = lo.match(sd, *a, n_layers=n)
        r64 = lo.match(sd, *a, dtype=np.float64, n_layers=n)
        e = max(np.abs(r32["x"][s] - r64["x"][s]).max() for s in range(2))
        tol = case_tol(case, f"layer{n}")
        print(f"{case}: {n} layers: fp32 {e:.3g}, bound {tol:.3g}")
        assert 5 * e <= tol
    e = max(np.abs(r32["mscore"] - r64["mscore"]).max(), np.abs(np.exp(r32["col_max"]) - np.exp(r64["col_max"])).max())
    tol = case_tol(case, "score")
    print(f"{case}: scores: fp32 {e:.3g}, bound {tol:.3g}")
    assert 5 * e <= tol


@pytest.mark.parametrize("case", E.CASE_IDS)
@pytest.mark.parametrize("min_conf", [0.0, 0.1])
def test_finalize_rule_reproduces_oracle(sd, case, min_conf):
    c = E.BY_NAME[case]
    r = lo.match(sd, *E.case_args(c), min_conf=min_conf, dtype=np.float64)
    best = np.stack([E.pad(r["row_max"], c.n_max), E.pad(r["col_max"], c.n_max)]).astype(np.float64)
    arg = np.zeros((2, c.n_max), np.int64)
    arg[0, :c.n0], arg[1, :c.n1] = r["row_arg"], r["col_arg"]
    ind = np.stack([np.arange(c.n_max)] * 2)
    i0, i1, sc = E.finalize_rule(best, arg, ind, np.array([c.n0, c.n1]), min_conf)[0]
    print(f"{case} min_conf {min_conf}: {len(i0)} matches")
    assert np.array_equal(i0, r["idx0"]) and np.array_equal(i1, r["idx1"]) and np.array_equal(sc, r["scores"])
    if min_conf == 0.0 and c.n0 > 0 and c.n1 > 0:
        assert len(i0) > 0
