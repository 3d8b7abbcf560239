"""LighterGlue on the H100 (csrc/lighterglue.cu) against the CPU oracle (oracle/lighterglue_oracle.py) and the goldens that
transformers' independent LightGlue produced (tests/golden/lg_*.npz).  Tolerances: tests/test_lighterglue_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import lighterglue_oracle as lo
from tests.test_lighterglue_oracle import (ATTN_TOL, LAYER_TOL, NEAR_TIE_EPS, SCORE_TOL, golden_args, load_case,
                                           match_set_diff, near_tie)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def xf():
    from accelerated_features_b200 import XFeat
    from oracle import build_lighterglue
    return XFeat(device=0, lighterglue_weights=build_lighterglue.path())


@pytest.fixture(scope="module")
def sd():
    return lo.load_state()


def _dev(a, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dt)


def _batch_inputs(cases, n_max):
    """cases: list of (kpts0, desc0, size0, kpts1, desc1, size1) -> padded device tensors in match_lighterglue_batch order."""
    B = len(cases)
    k = np.zeros((2, B, n_max, 2), np.float32)
    d = np.zeros((2, B, n_max, 64), np.float32)
    n = np.zeros((2, B), np.int32)
    s = np.zeros((2, B, 2), np.float32)
    for b, c in enumerate(cases):
        for side in range(2):
            kk, dd, ss = c[3 * side:3 * side + 3]
            k[side, b, :len(kk)], d[side, b, :len(kk)], n[side, b], s[side, b] = kk, dd, len(kk), ss
    return (_dev(k[0]), _dev(d[0]), _dev(n[0], torch.int32), _dev(s[0]),
            _dev(k[1]), _dev(d[1]), _dev(n[1], torch.int32), _dev(s[1]))


def _debug(xf, args, n_max, n_layers, prune, want_assign=False):
    lib = xf._lib
    B = args[0].shape[0]
    x = torch.zeros((2, B, n_max, 96), device="cuda")
    ind = torch.zeros((2, B, n_max), dtype=torch.int32, device="cuda")
    cnt = torch.zeros((2, B), dtype=torch.int32, device="cuda")
    best = torch.zeros((2, B, n_max), device="cuda") if want_assign else None
    arg = torch.zeros((2, B, n_max), dtype=torch.int32, device="cuda") if want_assign else None
    ws = torch.empty(lib.xfeat_lg_workspace_bytes(B, n_max), dtype=torch.uint8, device="cuda")
    from accelerated_features_b200 import _lib
    _lib.check(lib.xfeat_lg_debug(xf._lg().ctx, B, n_max, *[a.data_ptr() for a in args], -1 if prune is None else prune, n_layers,
                                  x.data_ptr(), ind.data_ptr(), cnt.data_ptr(), None if best is None else best.data_ptr(),
                                  None if arg is None else arg.data_ptr(), ws.data_ptr(), ws.numel(),
                                  torch.cuda.current_stream().cuda_stream), "xfeat_lg_debug")
    torch.cuda.synchronize()
    return x.cpu().numpy(), ind.cpu().numpy(), cnt.cpu().numpy(), (None if best is None else best.cpu().numpy()), \
        (None if arg is None else arg.cpu().numpy())


@pytest.mark.parametrize("n", [1, 63, 64, 65, 4096, 8192])
@pytest.mark.parametrize("cross", [0, 1])
def test_attention_stage_vs_float64(xf, sd, n, cross):
    """The attention kernel alone on the asset pair's layer-0 activations (q, k, v of image 0 and 1, tiled to n rows), ragged
    counts n and n - n//3, against float64."""
    g = load_case("lg_assets_4096")
    m = lo._Model(sd, np.float64)
    xs = [m.lin("input_proj", g[f"desc{s}"].astype(np.float64)) for s in range(2)]
    qkv = [m.lin("transformers.0.self_attn.Wqkv", x) for x in xs]
    reps = -(-n // 4096)
    rows = np.stack([np.tile(q, (reps, 1))[:n] for q in qkv]).astype(np.float32)       # (2, n, 288)
    counts = np.array([n, max(1, n - n // 3)], np.int32)
    q, k, v = (_dev(rows[..., c::3].copy()) for c in range(3))
    out = torch.zeros((2, n, 96), device="cuda")
    cnt = _dev(counts, torch.int32)
    tiles_per_cta = -(-int(counts.min()) // 64)
    assert n < 64 or tiles_per_cta >= min(n // 64, 40), "each CTA must walk many key tiles"
    from accelerated_features_b200 import _lib
    _lib.check(xf._lib.xfeat_lg_debug_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), 96, cnt.data_ptr(), 2, n, cross,
                                                out.data_ptr(), torch.cuda.current_stream().cuda_stream), "attention")
    qd, kd, vd = (t.double() for t in (q, k, v))
    for gi in range(2):
        gk = (gi + 1) % 2 if cross else gi
        nq, nk = counts[gi], counts[gk]
        s = (qd[gi, :nq] @ kd[gk, :nk].T) / np.sqrt(96.0)
        want = torch.softmax(s, 1) @ vd[gk, :nk]
        err = (out[gi, :nq].double() - want).abs().max().item()
        scale = vd[gk, :nk].abs().max().item()
        print(f"n={n} cross={cross} g={gi}: max err {err:.3g} (bound {ATTN_TOL * scale:.3g})")
        assert err <= ATTN_TOL * scale
        assert out[gi, nq:].abs().max().item() == 0 if nq < n else True


@pytest.mark.parametrize("n_layers", [0, 1, 6])
def test_layers_vs_float64(xf, sd, n_layers):
    """Descriptors after 0, 1 and 6 layers (no pruning) on the 1024-point asset pair against the float64 oracle."""
    g = load_case("lg_assets_1024")
    args = _batch_inputs([golden_args(g)], 1024)
    x, ind, cnt, _, _ = _debug(xf, args, 1024, n_layers, None)
    assert cnt.tolist() == [[1024], [1024]] and (ind[:, 0] == np.arange(1024)).all()
    m = lo._Model(sd, np.float64)
    want = lo.match(sd, *golden_args(g), dtype=np.float64, n_layers=n_layers)["x"] if n_layers else \
        [m.lin("input_proj", g[f"desc{s}"].astype(np.float64)) for s in range(2)]
    for s in range(2):
        err = np.abs(x[s, 0] - want[s]).max()
        print(f"layers={n_layers} side {s}: max err {err:.3g} (bound {LAYER_TOL[n_layers]:.3g})")
        assert err <= LAYER_TOL[n_layers]


def test_assignment_maxima_vs_float64(xf, sd):
    """Log-assignment row / column maxima and arg-maxima after layer 5 (1024-point asset pair, no pruning) against float64."""
    g = load_case("lg_assets_1024")
    _, _, cnt, best, arg = _debug(xf, _batch_inputs([golden_args(g)], 1024), 1024, 6, None, want_assign=True)
    orc = lo.match(sd, *golden_args(g), dtype=np.float64)
    # compared as scores exp(row max): the log values of unmatchable rows reach -28, where fp32 itself is 2.6e-3 off
    err = np.abs(np.exp(best[0, 0].astype(np.float64)) - orc["mscore"]).max()
    print(f"row max as score: err {err:.3g} (bound {SCORE_TOL}); log-space err {np.abs(best[0, 0] - orc['row_max']).max():.3g}")
    assert err <= SCORE_TOL
    for s, key, gap in ((0, "row_arg", "row_gap"), (1, "col_arg", "col_gap")):
        bad = np.nonzero(arg[s, 0] != orc[key])[0]
        print(f"side {s}: {len(bad)} arg-max differ")
        assert len(bad) <= 8 and (orc[gap][bad] < NEAR_TIE_EPS).all()


@pytest.mark.parametrize("case", ["lg_assets_4096", "lg_assets_1024", "lg_ragged"])
def test_match_lighterglue_vs_golden(xf, sd, case):
    g = load_case(case)
    d0 = {"keypoints": torch.from_numpy(g["kpts0"]), "descriptors": torch.from_numpy(g["desc0"]),
          "image_size": tuple(int(v) for v in g["size0"])}
    d1 = {"keypoints": torch.from_numpy(g["kpts1"]), "descriptors": torch.from_numpy(g["desc1"]),
          "image_size": tuple(int(v) for v in g["size1"])}
    mk0, mk1, idx = xf.match_lighterglue(d0, d1, min_conf=float(g["min_conf"]), prune_min_points=None)
    assert np.array_equal(mk0, g["kpts0"][idx[:, 0]]) and np.array_equal(mk1, g["kpts1"][idx[:, 1]])
    assert (np.diff(idx[:, 0]) > 0).all()
    orc = lo.match(sd, *golden_args(g), dtype=np.float64)
    diff = match_set_diff(idx[:, 0], idx[:, 1], g["idx0"], g["idx1"])
    print(f"{case}: {len(idx)} matches, golden {len(g['idx0'])}, {len(diff)} differ")
    assert len(diff) <= 8
    for i in diff:
        assert near_tie(orc, i, float(g["min_conf"])), f"row {i} differs and is not a near-tie"
    # scores of the common matches
    args = _batch_inputs([golden_args(g)], max(len(g["kpts0"]), len(g["kpts1"])))
    i0, i1, sc, cnt = xf.match_lighterglue_batch(*args, min_conf=float(g["min_conf"]), prune_min_points=None)
    n = int(cnt.item())
    got = dict(zip(i0[0, :n].tolist(), sc[0, :n].tolist()))
    want = dict(zip(orc["idx0"].tolist(), orc["scores"].tolist()))       # against float64 (the golden is itself fp32)
    err = max(abs(got[i] - want[i]) for i in set(got) & set(want))
    print(f"{case}: max score err {err:.3g} (bound {SCORE_TOL})")
    assert err <= SCORE_TOL


def test_pruned_vs_oracle(xf, sd):
    """Pruning at the default threshold on the 4096-point pair: every keep decision that differs from the oracle's is a near-tie
    of sigmoid(z) at 0.05; the oracle replayed with the GPU's keep sets gives the GPU's matches."""
    g = load_case("lg_assets_4096")
    args = _batch_inputs([golden_args(g)], 4096)
    T = 1536
    inds = [np.arange(4096), np.arange(4096)]
    keep_sets = []
    for layer in range(1, 6):
        _, ind, cnt, _, _ = _debug(xf, args, 4096, layer, T)
        ks = []
        for s in range(2):
            new = ind[s, 0, :cnt[s, 0]]
            ks.append(np.isin(inds[s], new) if len(inds[s]) > T else None)
            if ks[-1] is None:
                assert len(new) == len(inds[s])
            inds[s] = new
        keep_sets.append(ks)
    assert any(k is not None and not k.all() for ks in keep_sets for k in ks), "the case must prune"
    rep = lo.match(sd, *golden_args(g), keep_sets=keep_sets)
    n_diff = 0
    for layer, (ks, zs) in enumerate(zip(keep_sets, rep["z"])):
        for s in range(2):
            if ks[s] is None:
                continue
            mine = lo.keep_rule(zs[s])
            bad = np.nonzero(mine != ks[s])[0]
            n_diff += len(bad)
            p = 1 / (1 + np.exp(-zs[s][bad].astype(np.float64)))
            assert (np.abs(p - 0.05) < NEAR_TIE_EPS).all(), (layer, s, p)
    idx0, idx1, sc, cnt = xf.match_lighterglue_batch(*args, min_conf=float(g["min_conf"]), prune_min_points=T)
    n = int(cnt.item())
    diff = match_set_diff(idx0[0, :n].cpu().numpy(), idx1[0, :n].cpu().numpy(), rep["idx0"], rep["idx1"])
    print(f"pruned: final counts {[len(i) for i in inds]}, {n} matches, oracle {len(rep['idx0'])}, {len(diff)} differ, "
          f"{n_diff} keep decisions differ")
    # differing rows are given in original indices; map to the oracle's surviving rows for the near-tie check
    pos = {int(v): i for i, v in enumerate(rep["ind"][0])}
    assert len(diff) <= 8
    for i in diff:
        assert i in pos and near_tie(rep, pos[i], float(g["min_conf"]))


def test_batch_is_bit_identical_to_single_pairs(xf):
    """A ragged batch of 64 pairs (counts include 0, 1 and n_max) gives the same bits as 64 single-pair calls."""
    g = load_case("lg_assets_1024")
    rs = np.random.RandomState(5)
    n_max = 1024
    cases = []
    for b in range(64):
        n0 = [0, 1, n_max, 5][b] if b < 4 else int(rs.randint(0, n_max + 1))
        n1 = [n_max, 1, n_max, 0][b] if b < 4 else int(rs.randint(0, n_max + 1))
        i0, i1 = np.sort(rs.permutation(n_max)[:n0]), np.sort(rs.permutation(n_max)[:n1])
        cases.append((g["kpts0"][i0], g["desc0"][i0], g["size0"], g["kpts1"][i1], g["desc1"][i1], g["size1"]))
    for prune in (None, 512):
        idx0, idx1, sc, cnt = xf.match_lighterglue_batch(*_batch_inputs(cases, n_max), prune_min_points=prune)
        idx0, idx1, sc, cnt = idx0.cpu().numpy(), idx1.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy()
        assert cnt[0] == 0 and cnt[3] == 0 and cnt[2] > 0
        for b, c in enumerate(cases):
            nm = max(len(c[0]), len(c[3]), 1)
            j0, j1, s1, c1 = xf.match_lighterglue_batch(*_batch_inputs([c], nm), prune_min_points=prune)
            k = int(c1.item())
            assert k == cnt[b], b
            assert np.array_equal(j0[0, :k].cpu().numpy(), idx0[b, :k]) and np.array_equal(j1[0, :k].cpu().numpy(), idx1[b, :k])
            assert np.array_equal(s1[0, :k].cpu().numpy().view(np.uint32), sc[b, :k].view(np.uint32)), b


def test_end_to_end_matches_detect_then_match(xf, assets_vga):
    ref, tgt = assets_vga
    x = torch.from_numpy(np.stack([ref, tgt])).permute(0, 3, 1, 2).float() / 255
    got = xf.match_xfeat_lighterglue_batch(x, x.flip(0), top_k=2048)
    for b in range(2):
        f0 = xf.detectAndCompute(x[b:b + 1], top_k=2048)[0]
        f1 = xf.detectAndCompute(x[1 - b:2 - b], top_k=2048)[0]
        f0["image_size"] = f1["image_size"] = (x.shape[3], x.shape[2])
        mk0, mk1, idx = xf.match_lighterglue(f0, f1)
        print(f"pair {b}: {len(idx)} matches")
        assert len(idx) > 100
        assert np.array_equal(idx, got[b][2]) and np.array_equal(mk0, got[b][0]) and np.array_equal(mk1, got[b][1])
