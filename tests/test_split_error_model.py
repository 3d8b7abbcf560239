"""CPU proof that each tensor-core tolerance of tests/split_ref.py can see a lost split term: on the real weights and real
activations of the asset pair, every bound is >= 5x the error of the exact three-term split arithmetic and <= 1/5 of the error
with any one of hi.whi, hi.wlo, lo.whi dropped.  A looser bound would let a kernel that skips a term pass."""
import pytest
import torch

from oracle import xfeat_oracle as orc
from tests import split_ref as sr


@pytest.fixture(scope="module")
def stages(oracle_state, assets_vga):
    ref, tgt = assets_vga
    x = torch.cat([orc.parse_input(ref), orc.parse_input(tgt)], 0)
    with torch.inference_mode():
        st = orc.backbone(oracle_state, x)
        st["b5_0"] = sr.reference(oracle_state, 13, st["x4"]).float()
        st["b5_1"] = sr.reference(oracle_state, 14, st["b5_0"]).float()
        st["b5_2"] = sr.reference(oracle_state, 15, st["b5_1"]).float()
    return st


def _max_abs(ref):
    return lambda y: (y - ref).abs().max()


# (layer id, name, input stage): every configuration of the convolution kernels (8-, 24-, 64- and 128-channel operands,
# stride 2, 1x1, two N tiles, the stem skip branch)
CONV_LAYERS = [(2, "block1.2", "b1_1"), (3, "block1.3+skip1", "b1_2"), (5, "block2.0", "x1s"), (6, "block2.1", "b2_0"),
               (7, "block3.0", "x2"), (8, "block3.1", "b3_0"), (9, "block3.2", "b3_1"), (10, "block4.0", "x3"),
               (13, "block5.0", "x4"), (14, "block5.1", "b5_0"), (15, "block5.2", "b5_1"), (16, "block5.3", "b5_2"),
               (17, "block_fusion.0", "fusion_in")]


@pytest.mark.parametrize("case", CONV_LAYERS, ids=lambda c: c[1])
def test_conv_tc_bound(oracle_state, stages, case):
    layer, name, key = case
    x = stages[key]
    skip = stages["xn"][:, 0] if layer == 3 else None
    with torch.inference_mode():
        ref = sr.reference(oracle_state, layer, x, skip)
        scale = ref.abs().max()
        model = sr.error_model(lambda t: sr.emulate(oracle_state, layer, x, t, skip), lambda y: (y - ref).abs().max() / scale)
    print(f"{name}: CONV_TC_TOL {sr.CONV_TC_TOL:.1e}; {sr.fmt_model(model)}")
    sr.check_bound(f"CONV_TC_TOL ({name})", sr.CONV_TC_TOL, model)


def test_keypoint_head_bounds(oracle_state, stages):
    u = orc.unfold8(stages["xn"])
    with torch.inference_mode():
        logits = sr.reference_chain(oracle_state, sr.KEYPOINT_HEAD, u)
        heat = orc.kpts_heatmap(logits)
        m_log = sr.error_model(lambda t: sr.emulate_chain(oracle_state, sr.KEYPOINT_HEAD, u, t), _max_abs(logits))
        m_heat = sr.error_model(lambda t: orc.kpts_heatmap(sr.emulate_chain(oracle_state, sr.KEYPOINT_HEAD, u, t)), _max_abs(heat))
    print(f"keypoint logits: {sr.fmt_model(m_log)}\nheat: {sr.fmt_model(m_heat)}")
    sr.check_bound("KPT_LOGITS_TOL", sr.KPT_LOGITS_TOL, m_log)
    sr.check_bound("HEAT_TOL", sr.HEAT_TOL, m_heat)


def test_reliability_head_bound(oracle_state, stages):
    f = stages["feats"]
    with torch.inference_mode():
        rel = torch.sigmoid(sr.reference_chain(oracle_state, sr.HEATMAP_HEAD, f))
        model = sr.error_model(lambda t: torch.sigmoid(sr.emulate_chain(oracle_state, sr.HEATMAP_HEAD, f, t)), _max_abs(rel))
    print(f"reliability: {sr.fmt_model(model)}")
    sr.check_bound("RELIABILITY_TOL", sr.RELIABILITY_TOL, model)


def test_fine_matcher_bounds(oracle_state, stages):
    """Real coarse-feature pairs: the mutual nearest neighbours between the two images' dense feature maps."""
    with torch.inference_mode():
        x = sr.coarse_pairs(stages["feats"][0], stages["feats"][1])
        assert len(x) >= 500
        logits = sr.reference_chain(oracle_state, sr.FINE_MATCHER, x)
        xy = orc.subpix_softmax2d(logits.view(-1, 8, 8))
        m_log = sr.error_model(lambda t: sr.emulate_chain(oracle_state, sr.FINE_MATCHER, x, t), _max_abs(logits))
        m_xy = sr.error_model(lambda t: orc.subpix_softmax2d(sr.emulate_chain(oracle_state, sr.FINE_MATCHER, x, t).view(-1, 8, 8)),
                              _max_abs(xy))
    print(f"fine matcher ({len(x)} rows) logits: {sr.fmt_model(m_log)}\nsub-pixel offsets: {sr.fmt_model(m_xy)}")
    sr.check_bound("FINE_MATCHER_TOL", sr.FINE_MATCHER_TOL, m_log)
    sr.check_bound("SUBPIX_TOL", sr.SUBPIX_TOL, m_xy)


def test_emulation_is_exact_on_representable_operands(oracle_state):
    """Sanity of the emulation itself: activations that are fp16-exact have lo = 0, so dropping lo.whi changes nothing, and the
    three-term result differs from float64 only by the weight split."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(300, 128, generator=g).half().float()
    with torch.inference_mode():
        a = sr.emulate(oracle_state, 27, x)
        b = sr.emulate(oracle_state, 27, x, ("hi.whi", "hi.wlo"))
        assert torch.equal(a, b)
        assert float((a - sr.reference(oracle_state, 27, x)).abs().max()) < 1e-5
    assert sr.min_tiles_per_cta(128 * 132 * 3, 132) == 3 and sr.min_tiles_per_cta(128 * (132 * 3 - 1), 132) == 2
