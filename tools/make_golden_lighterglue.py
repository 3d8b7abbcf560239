"""Generate tests/golden/lg_*.npz: LighterGlue matches from an independent implementation, Hugging Face transformers'
`LightGlueForKeypointMatching` (eager attention, fp32, CPU, point pruning off), loaded with the published matcher weights.

Build-machine tool, like tools/make_golden.py: needs the reference checkout (assets, weights/xfeat-lighterglue.pt) and a Python
environment with `transformers` >= 5 (path overridable: --python or $LG_ORACLE_PYTHON; the script re-runs itself there).

Cases: the reference's asset pair at top_k 4096 and 1024 (features from the CPU oracle's detectAndCompute), and a seeded ragged
pair (700 vs 1900 of those points, the second image at 0.8x its size).  The descriptors are stored as int8 q with the input
defined as q / 128 (exact in fp32; |error| <= 1/256 against the extracted unit-norm descriptors), which keeps the files small;
the goldens are computed on exactly those inputs.  transformers normalises both images with one (H, W), so each image's keypoints
are pre-mapped (in float64) to the coordinates that yield its own normalisation (k - size/2) / (max(W, H)/2).
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("XFEAT_REFERENCE", "/root/reference")
DEFAULT_PY = os.environ.get("LG_ORACLE_PYTHON", "/opt/prime-rl/.venv/bin/python")
N_LAYERS = 6


def transformers_state(sd):
    """Published `matcher.*` names (lighterglue.py:40-46 renaming applied) -> transformers' LightGlue names."""
    import torch
    out = {}
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    out["input_projection.weight"], out["input_projection.bias"] = t(sd["input_proj.weight"]), t(sd["input_proj.bias"])
    out["positional_encoder.projector.weight"] = t(sd["posenc.Wr.weight"])
    for i in range(N_LAYERS):
        p, q = f"transformers.{i}.", f"transformer_layers.{i}."
        w, b = sd[p + "self_attn.Wqkv.weight"], sd[p + "self_attn.Wqkv.bias"]
        for c, name in enumerate("qkv"):                        # interleaved rows: q, k, v = 3i, 3i+1, 3i+2
            out[q + f"self_attention.{name}_proj.weight"] = t(w[c::3])
            out[q + f"self_attention.{name}_proj.bias"] = t(b[c::3])
        out[q + "self_attention.o_proj.weight"] = t(sd[p + "self_attn.out_proj.weight"])
        out[q + "self_attention.o_proj.bias"] = t(sd[p + "self_attn.out_proj.bias"])
        for name in ("q", "k"):
            out[q + f"cross_attention.{name}_proj.weight"] = t(sd[p + "cross_attn.to_qk.weight"])
            out[q + f"cross_attention.{name}_proj.bias"] = t(sd[p + "cross_attn.to_qk.bias"])
        out[q + "cross_attention.v_proj.weight"] = t(sd[p + "cross_attn.to_v.weight"])
        out[q + "cross_attention.v_proj.bias"] = t(sd[p + "cross_attn.to_v.bias"])
        out[q + "cross_attention.o_proj.weight"] = t(sd[p + "cross_attn.to_out.weight"])
        out[q + "cross_attention.o_proj.bias"] = t(sd[p + "cross_attn.to_out.bias"])
        for blk, mlp in (("self_attn", "self_mlp"), ("cross_attn", "cross_mlp")):
            for a, b_ in (("0", "fc1"), ("1", "layer_norm"), ("3", "fc2")):
                for s in ("weight", "bias"):
                    out[q + f"{mlp}.{b_}.{s}"] = t(sd[p + f"{blk}.ffn.{a}.{s}"])
        for s in ("weight", "bias"):
            out[f"match_assignment_layers.{i}.final_projection.{s}"] = t(sd[f"log_assignment.{i}.final_proj.{s}"])
            out[f"match_assignment_layers.{i}.matchability.{s}"] = t(sd[f"log_assignment.{i}.matchability.{s}"])
            if i < N_LAYERS - 1:
                out[f"token_confidence.{i}.token.{s}"] = t(sd[f"token_confidence.{i}.token.0.{s}"])
    return out


def build_model(sd):
    import torch
    from transformers import LightGlueConfig, LightGlueForKeypointMatching
    cfg = LightGlueConfig(descriptor_dim=96, num_hidden_layers=N_LAYERS, num_attention_heads=1, depth_confidence=-1.0,
                          width_confidence=-1.0, filter_threshold=0.1,
                          keypoint_detector_config={"model_type": "superpoint", "descriptor_decoder_dim": 64},
                          attn_implementation="eager")
    model = LightGlueForKeypointMatching(cfg).eval()
    res = model.load_state_dict(transformers_state(sd), strict=False)
    missing = [k for k in res.missing_keys if not k.startswith("keypoint_detector.")]
    assert not missing and not res.unexpected_keys, (missing, res.unexpected_keys)
    return model.float()


def quantize(d):
    """Descriptors -> int8 q; the test input is q / 128."""
    return np.clip(np.round(d.astype(np.float64) * 128), -128, 127).astype(np.int8)


def save(path, k0, q0, s0, k1, q1, s1, r):
    np.savez_compressed(path, kpts0=k0, desc0_q=q0, size0=np.asarray(s0), kpts1=k1, desc1_q=q1, size1=np.asarray(s1),
                        min_conf=np.float32(0.1), **r)


def run_case(model, k0, d0, s0, k1, d1, s1, min_conf=0.1):
    import torch
    n0, n1 = len(k0), len(k1)
    n = max(n0, n1)
    W, H = s0                                       # the one size transformers normalises with

    def premap(k, s):                               # float64: (k' * max(W,H)/2 + (W,H)/2) with k' of this image's own size
        kn = (k.astype(np.float64) - np.asarray(s, np.float64) / 2) / (max(s) / 2)
        return kn * (max(W, H) / 2) + np.asarray([W, H], np.float64) / 2
    kp = np.zeros((1, 2, n, 2), np.float32)
    de = np.zeros((1, 2, n, 64), np.float32)
    mask = np.zeros((1, 2, n), np.int64)
    for s, (k, d, sz) in enumerate(((k0, d0, s0), (k1, d1, s1))):
        kp[0, s, :len(k)] = premap(k, sz)
        de[0, s, :len(k)] = d
        mask[0, s, :len(k)] = 1
    model.filter_threshold = min_conf
    hidden = {}

    def hook(_m, _i, o):
        hidden["x"] = o[0].detach().clone()
    h = model.transformer_layers[N_LAYERS - 1].register_forward_hook(hook)
    with torch.no_grad():
        matches, scores, *_ = model._match_image_pair(torch.from_numpy(kp), torch.from_numpy(de), H, W,
                                                      mask=torch.from_numpy(mask))
    h.remove()
    m0 = matches[0].numpy()
    sc0 = scores[0].numpy()
    i0 = np.nonzero((m0 >= 0) & (np.arange(n) < n0))[0]
    x = hidden["x"].numpy()                        # (2, n, 96): last-layer descriptors
    return {"idx0": i0.astype(np.int64), "idx1": m0[i0].astype(np.int64), "scores": sc0[i0].astype(np.float32),
            "x0_sum": np.float64(x[0, :n0].astype(np.float64).sum()), "x1_sum": np.float64(x[1, :n1].astype(np.float64).sum()),
            "x0_probe": x[0, :n0:97].copy(), "x1_probe": x[1, :n1:97].copy()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--python", default=DEFAULT_PY, help="interpreter of an environment with transformers")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    a = ap.parse_args()
    try:
        import transformers  # noqa: F401
    except ImportError:
        sys.exit(subprocess.call([a.python, os.path.abspath(__file__), "--python", a.python, "--out", a.out]))
    import cv2
    import torch
    sys.path.insert(0, ROOT)
    from accelerated_features_b200 import weights as W
    from oracle import xfeat_oracle as orc
    sd = W.load_lighterglue_state(os.path.join(REF, "weights", "xfeat-lighterglue.pt"))
    model = build_model(sd)
    xsd = orc.load_state()
    ref, tgt = cv2.imread(f"{REF}/assets/ref.png"), cv2.imread(f"{REF}/assets/tgt.png")
    for top_k in (4096, 1024):
        with torch.inference_mode():
            f0 = orc.detect_and_compute(xsd, ref, top_k)[0]
            f1 = orc.detect_and_compute(xsd, tgt, top_k)[0]
        k0, q0 = f0["keypoints"].numpy(), quantize(f0["descriptors"].numpy())
        k1, q1 = f1["keypoints"].numpy(), quantize(f1["descriptors"].numpy())
        s0, s1 = (ref.shape[1], ref.shape[0]), (tgt.shape[1], tgt.shape[0])
        r = run_case(model, k0, q0.astype(np.float32) / 128, s0, k1, q1.astype(np.float32) / 128, s1)
        save(os.path.join(a.out, f"lg_assets_{top_k}.npz"), k0, q0, s0, k1, q1, s1, r)
        print(f"lg_assets_{top_k}: {len(k0)} / {len(k1)} points, {len(r['idx0'])} matches")
        if top_k == 4096:
            full = (k0, q0, s0, k1, q1, s1)
    # ragged: a seeded subset of the 4096-point asset features, 700 vs 1900 points, the second image at 0.8x its size
    k0, q0, s0, k1, q1, s1 = full
    rs = np.random.RandomState(11)
    i0 = np.sort(rs.choice(len(k0), 700, replace=False))
    i1 = np.sort(rs.choice(len(k1), 1900, replace=False))
    k0, q0 = k0[i0], q0[i0]
    k1, q1 = (k1[i1] * np.float32(0.8)).astype(np.float32), q1[i1]
    s1 = (int(s1[0] * 0.8), int(s1[1] * 0.8))
    r = run_case(model, k0, q0.astype(np.float32) / 128, s0, k1, q1.astype(np.float32) / 128, s1)
    save(os.path.join(a.out, "lg_ragged.npz"), k0, q0, s0, k1, q1, s1, r)
    print(f"lg_ragged: 700 / 1900 points, {len(r['idx0'])} matches")


if __name__ == "__main__":
    main()
