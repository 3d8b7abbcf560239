"""CPU checks of the LighterGlue oracle (oracle/lighterglue_oracle.py) against transformers' independent LightGlue
(tests/golden/lg_*.npz, tools/make_golden_lighterglue.py), the weight packer, the pruning rule, and the error model that sets the
tolerances of tests/test_gpu_lighterglue.py.

Tolerances.  The kernels compute in fp32 on the CUDA cores (no split operands), so the budget is fp32's own rounding, amplified by
12 residual blocks with |x| up to ~29: on the 1024-point asset pair the float32 oracle is 4.8e-6 off float64 after one layer,
3.4e-3 after six; on the match scores of the 4096-point pair it is 2.4e-4 off and transformers' fp32 run 3.5e-4.  Each bound is
at least 5x that (test_layer_tolerances_cover_fp32, test_score_tolerance_covers_fp32).

The golden inputs are the asset pair's extracted keypoints and descriptors, the descriptors stored as int8 q and read as q / 128
(exact in fp32), which keeps the files small; the goldens were computed on exactly these inputs.  The matcher weights are not in
the repository: build() stages them into oracle/_ref (oracle/build_lighterglue.py).
For the attention kernel the error model below also proves the bound is at most 1/5 of the error of a kernel that rounded its
operands to fp16."""
import os

import numpy as np
import pytest

from oracle import lighterglue_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["lg_assets_1024", "lg_ragged", "lg_assets_4096"]

ATTN_TOL = 4e-6                                   # attention output, relative to max |v|
LAYER_TOL = {0: 2e-6, 1: 5e-5, 6: 2e-2}           # descriptors after n layers, absolute
SCORE_TOL = 2e-3                                  # match scores exp(row max) against float64, absolute
NEAR_TIE_EPS = 1e-3                               # log-assignment gaps, |mscore - min_conf|, |sigmoid(z) - 0.05|


def load_case(name):
    """A golden case; the stored int8 descriptors q decode to the inputs q / 128 (exact in fp32)."""
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as z:
        g = {k: z[k] for k in z.files}
    for s in range(2):
        g[f"desc{s}"] = g.pop(f"desc{s}_q").astype(np.float32) / np.float32(128)
    return g


def golden_args(g):
    return (g["kpts0"], g["desc0"], tuple(g["size0"]), g["kpts1"], g["desc1"], tuple(g["size1"]))


def match_set_diff(a0, a1, b0, b1):
    """Rows i (image-0 index) whose match differs between the two sets."""
    a, b = dict(zip(np.asarray(a0).tolist(), np.asarray(a1).tolist())), dict(zip(np.asarray(b0).tolist(), np.asarray(b1).tolist()))
    return sorted(i for i in set(a) | set(b) if a.get(i) != b.get(i))


def near_tie(orc, i, min_conf, eps=NEAR_TIE_EPS):
    """Row i of the oracle's (surviving) points: its match decision may flip under fp32 rounding."""
    j = int(orc["row_arg"][i])
    return (abs(float(orc["mscore"][i]) - min_conf) < eps or orc["row_gap"][i] < eps or orc["col_gap"][j] < eps
            or any(orc["col_gap"][jj] < eps for jj in np.nonzero(orc["col_arg"] == i)[0]))


@pytest.fixture(scope="module")
def sd():
    return lo.load_state()


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_transformers_golden(sd, case):
    g = load_case(case)
    r = lo.match(sd, *golden_args(g), min_conf=float(g["min_conf"]), dtype=np.float64)
    diff = match_set_diff(r["idx0"], r["idx1"], g["idx0"], g["idx1"])
    assert all(near_tie(r, i, float(g["min_conf"])) for i in diff) and len(diff) <= 8, diff
    got = dict(zip(r["idx0"].tolist(), r["scores"].tolist()))
    err = max(abs(got[i] - s) for i, s in zip(g["idx0"].tolist(), g["scores"].tolist()) if i in got)
    assert err <= SCORE_TOL, err
    n0 = len(g["kpts0"])
    assert abs(r["x"][0].sum() - g["x0_sum"]) <= 1e-5 * np.abs(r["x"][0]).sum()
    assert np.abs(r["x"][0][::97] - g["x0_probe"]).max() <= LAYER_TOL[6] and n0 == len(r["x"][0])


def test_weight_packer_round_trip(sd):
    from accelerated_features_b200 import weights as W
    blob = W.pack_lighterglue(sd)
    o = 0

    def take(shape):
        nonlocal o
        n = int(np.prod(shape))
        a = blob[o:o + n].reshape(shape)
        o += -(-n // 4) * 4
        return a
    assert np.array_equal(take((64, 96)), sd["input_proj.weight"].T)
    assert np.array_equal(take((96,)), sd["input_proj.bias"])
    assert np.array_equal(take((2, 48)), sd["posenc.Wr.weight"].T)
    for i in range(6):
        p = f"transformers.{i}."
        w = take((96, 288)).T
        for c in range(3):                     # [q | k | v] blocks = interleaved rows c, c+3, ...
            assert np.array_equal(w[96 * c:96 * (c + 1)], sd[p + "self_attn.Wqkv.weight"][c::3])
        assert np.array_equal(take((288,))[96:192], sd[p + "self_attn.Wqkv.bias"][1::3])
        for blk in ("self_attn", "cross_attn"):
            if blk == "cross_attn":
                w = take((96, 192)).T
                assert np.array_equal(w[:96], sd[p + "cross_attn.to_qk.weight"]) and np.array_equal(w[96:], sd[p + "cross_attn.to_v.weight"])
                take((192,))
                assert np.array_equal(take((96, 96)), sd[p + "cross_attn.to_out.weight"].T)
                take((96,))
            else:
                assert np.array_equal(take((96, 96)), sd[p + "self_attn.out_proj.weight"].T)
                take((96,))
            q = p + blk + ".ffn."
            assert np.array_equal(take((192, 192)), sd[q + "0.weight"].T)
            for name in ("0.bias", "1.weight", "1.bias"):
                assert np.array_equal(take((192,)), sd[q + name])
            assert np.array_equal(take((192, 96)), sd[q + "3.weight"].T)
            assert np.array_equal(take((96,)), sd[q + "3.bias"])
    for i in range(6):
        p = f"log_assignment.{i}."
        assert np.array_equal(take((96, 96)), sd[p + "final_proj.weight"].T)
        take((96,))
        assert np.array_equal(take((96,)), sd[p + "matchability.weight"][0])
        assert np.array_equal(take((1,)), sd[p + "matchability.bias"])
    assert o == blob.size


def test_packed_size_matches_library():
    from accelerated_features_b200 import _lib, weights as W
    from accelerated_features_b200.build import build_library
    build_library()
    assert W.pack_lighterglue(lo.load_state()).size == _lib.load().xfeat_lg_packed_weight_floats()


def test_missing_weights_are_reported(tmp_path):
    from accelerated_features_b200 import weights as W
    with pytest.raises(FileNotFoundError, match="xfeat-lighterglue.pt"):
        W.load_lighterglue_state(str(tmp_path / "absent.pt"))


def test_published_and_resaved_weights_load_alike(sd, tmp_path):
    """The published .pt's `matcher.*` keys (extractor keys beside them) load to the same state as the re-saved .npz."""
    from accelerated_features_b200 import weights as W
    pub = {"matcher." + k: v for k, v in sd.items()}
    pub["extractor.model.net.skip1.1.bias"] = np.zeros(24, np.float32)
    got = W.load_lighterglue_state(pub)
    assert sorted(got) == sorted(sd) and all(np.array_equal(got[k], sd[k]) for k in sd)


def test_prune_threshold_at_or_above_n_is_unpruned(sd):
    g = load_case("lg_assets_1024")
    a = lo.match(sd, *golden_args(g))
    b = lo.match(sd, *golden_args(g), prune_min_points=1024)
    assert all(k is None for ks in b["keep"] for k in ks)
    for key in ("idx0", "idx1", "scores"):
        assert np.array_equal(a[key], b[key])
    c = lo.match(sd, *golden_args(g), prune_min_points=1023)
    assert any(k is not None and not k.all() for ks in c["keep"] for k in ks)


def test_keep_rule():
    logit = np.log(0.05 / 0.95)
    z = np.array([logit - 1e-3, logit + 1e-3, -50.0, 50.0, 0.0], np.float32)
    assert lo.keep_rule(z).tolist() == [False, True, False, True, True]


def test_replayed_keep_sets_reproduce_pruning(sd):
    g = load_case("lg_assets_1024")
    a = lo.match(sd, *golden_args(g), prune_min_points=512)
    b = lo.match(sd, *golden_args(g), keep_sets=a["keep"])
    for key in ("idx0", "idx1", "scores"):
        assert np.array_equal(a[key], b[key])


def test_empty_and_one_point(sd):
    g = load_case("lg_assets_1024")
    k0, d0, s0, k1, d1, s1 = golden_args(g)
    r = lo.match(sd, k0[:0], d0[:0], s0, k1, d1, s1)
    assert len(r["idx0"]) == 0 and len(r["scores"]) == 0
    r = lo.match(sd, k0, d0, s0, k1[:0], d1[:0], s1)
    assert len(r["idx0"]) == 0
    r = lo.match(sd, k0[:1], d0[:1], s0, k1[:1], d1[:1], s1, min_conf=0.0)
    assert r["idx0"].tolist() == [0] and r["idx1"].tolist() == [0]      # one point each: trivially mutual
    assert 0 < r["scores"][0] <= 1


def test_attention_error_model(sd):
    """ATTN_TOL is >= 5x the fp32 kernel's error and <= 1/5 of the error of fp16-rounded operands (asset activations, layer 0)."""
    g = load_case("lg_assets_1024")
    m = lo._Model(sd, np.float64)
    x = m.lin("input_proj", g["desc0"].astype(np.float64))
    qkv = m.lin("transformers.0.self_attn.Wqkv", x)
    q, k, v = qkv[:, 0::3], qkv[:, 1::3], qkv[:, 2::3]

    def att(q, k, v, dt):
        q, k, v = (t.astype(dt) for t in (q, k, v))
        s = (q @ k.T) / dt(np.sqrt(96))
        s = np.exp(s - s.max(1, keepdims=True))
        return (s / s.sum(1, keepdims=True)) @ v
    ref = att(q, k, v, np.float64)
    scale = np.abs(v).max()
    e32 = np.abs(att(q, k, v, np.float32) - ref).max() / scale
    h = lambda t: t.astype(np.float16).astype(np.float64)    # noqa: E731
    e16 = np.abs(att(h(q), h(k), h(v), np.float64) - ref).max() / scale
    print(f"attention: fp32 {e32:.3g}, fp16 operands {e16:.3g}, tolerance {ATTN_TOL:.3g}")
    assert 5 * e32 <= ATTN_TOL <= e16 / 5


def test_layer_tolerances_cover_fp32(sd):
    g = load_case("lg_assets_1024")
    for n in (1, 6):
        a = lo.match(sd, *golden_args(g), n_layers=n)
        b = lo.match(sd, *golden_args(g), dtype=np.float64, n_layers=n)
        e = max(np.abs(a["x"][s] - b["x"][s]).max() for s in range(2))
        print(f"{n} layers: fp32 {e:.3g}, tolerance {LAYER_TOL[n]:.3g}")
        assert 5 * e <= LAYER_TOL[n]


@pytest.mark.parametrize("case", CASES)
def test_score_tolerance_covers_fp32(sd, case):
    """SCORE_TOL >= 5x the float32 oracle's and transformers' fp32 score error against float64, on every golden case."""
    g = load_case(case)
    a = lo.match(sd, *golden_args(g))
    b = lo.match(sd, *golden_args(g), dtype=np.float64)
    e32 = np.abs(a["mscore"] - b["mscore"]).max()
    want = dict(zip(b["idx0"].tolist(), b["scores"].tolist()))
    eg = max(abs(want[i] - s) for i, s in zip(g["idx0"].tolist(), g["scores"].tolist()))
    print(f"{case}: fp32 oracle {e32:.3g}, transformers fp32 {eg:.3g}, tolerance {SCORE_TOL:.3g}")
    assert 5 * max(e32, eg) <= SCORE_TOL
