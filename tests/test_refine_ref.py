"""refine_ref.py (the float64 batch restatement of refine_matches) against the float32 oracle on the asset pair's coarse matches,
within the oracle's own float32 error.  The second pair of the batch is the reversed pair with desc1 cut to fewer rows than desc0,
so the reference's separate n_max / n1_max strides are checked against the oracle's per-image indexing.  Runs on the CPU."""
import pytest
import torch

from oracle import xfeat_oracle as orc
from tests import refine_ref as rr
from tests import split_ref as sr

U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def coarse(oracle_state, assets_vga):
    ref, tgt = assets_vga
    with torch.inference_mode():
        feats = orc.backbone(oracle_state, torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0))["feats"]
    f = feats.permute(0, 2, 3, 1).reshape(2, -1, 64).contiguous()                     # (2, 4800, 64), un-normalised
    xy = (orc.create_xy(60, 80) * 8).float()
    g = torch.Generator().manual_seed(2)
    sc = torch.where(torch.rand(2, f.shape[1], generator=g) < 0.2, 1 / 0.6, 1 / 1.3).float()
    return f, xy, sc


def test_refine_ref_matches_oracle(oracle_state, coarse):
    f, xy, sc = coarse
    n1 = 3001                                                  # desc1 rows != desc0 rows: n1_max < n_max
    d0 = {"descriptors": f, "keypoints": xy.expand(2, -1, -1).contiguous(), "scales": sc}
    d1 = {"descriptors": f.flip(0)[:, :n1].contiguous(), "keypoints": (xy[:n1] + 0.25).expand(2, -1, -1).contiguous(),
          "scales": torch.ones(2, n1)}
    idxs = orc.batch_match(d0["descriptors"], d1["descriptors"])
    n_max = f.shape[1]
    idx0 = torch.zeros(2, n_max, dtype=torch.long)
    idx1 = torch.zeros(2, n_max, dtype=torch.long)
    cnt = torch.tensor([len(i0) for i0, _ in idxs])
    for b, (i0, i1) in enumerate(idxs):
        idx0[b, :len(i0)], idx1[b, :len(i1)] = i0, i1
    got = rr.refine_ref(oracle_state, d0["descriptors"], d1["descriptors"], d0["keypoints"], d1["keypoints"], d0["scales"],
                        idx0, idx1, cnt, 0.25)
    for b in range(2):
        want, st = orc.refine_matches(oracle_state, d0, d1, idxs, b, return_stages=True)
        r = got[b]
        assert r["n"] == len(idxs[b][0]) > 100
        e32 = float((st["logits"].double() - r["logits"]).abs().max())          # the float32 oracle's own logit error
        dconf = (st["conf"].double() - r["conf"]).abs()
        band = rr.conf_band(r["conf"], e32)
        assert bool((dconf <= band).all()), f"pair {b}: the derived confidence band does not cover the float32 oracle"
        unsure = (r["conf"] - 0.25).abs() <= band
        assert torch.equal(st["good"] | unsure, r["keep"] | unsure), f"pair {b}: kept sets differ outside the band"
        # d E[x] / d l_k = 3 p_k (x_k - E[x]): a logit error e moves an offset by at most 3 * 8 * e
        both = st["good"] & r["keep"]
        tol = 24 * e32 * float(sc.max()) + 4 * 640 * U32
        err = float((st["offsets"].double()[both] * d0["scales"][b, idxs[b][0]][both, None] -
                     (r["xy0"][both] - d0["keypoints"][b, idxs[b][0]][both].double())).abs().max())
        print(f"pair {b}: {r['n']} coarse, {int(r['keep'].sum())} kept, {int(unsure.sum())} in the band; float32 oracle "
              f"logit error {e32:.2e}, max |dconf| / band {float((dconf / band).max()):.3f}, offset error {err:.2e} "
              f"(bound {tol:.1e})")
        assert err <= tol
        assert torch.equal(want[:, 2:], r["xy1"][st["good"]])
        assert float((want[:, :2].double() - r["xy0"][st["good"]]).abs().max()) <= tol + 640 * U32


def test_refine_ref_counts_and_pairs(oracle_state, coarse):
    """Counts are clamped to [0, n_max], XF_N_OVERFLOW refines nothing, and a pair table picks the images."""
    f, xy, sc = coarse
    n_max = 50
    d = f[:, :n_max].contiguous()
    k = xy[:n_max].expand(2, -1, -1).contiguous()
    s = sc[:, :n_max].contiguous()
    ar = torch.arange(n_max).expand(4, -1).contiguous()
    out = rr.refine_ref(oracle_state, d, d, k, k, s, ar, ar, torch.tensor([-1, 0, n_max + 5, 7]), -1.0,
                        pairs=torch.tensor([[0, 1], [1, 1], [1, 0], [0, 1]]))
    assert [o["n"] for o in out] == [0, 0, n_max, 7]
    assert torch.equal(out[3]["rows"], torch.arange(7))                   # fine_conf < 0 keeps every live row (conf >= 1/64)
    assert float(out[2]["conf"].min()) >= 1 / 64
    x = torch.cat([d[1], d[0]], 1).double()
    want = sr.reference_chain(oracle_state, sr.FINE_MATCHER, x)
    assert torch.equal(out[2]["logits"], want)
