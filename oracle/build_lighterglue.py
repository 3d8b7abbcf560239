"""Recipe for oracle/_ref/lighterglue_state.npz: the published LighterGlue matcher weights (weights/xfeat-lighterglue.pt of the
reference checkout), `matcher.*` part renamed and re-saved as .npz by accelerated_features_b200.weights.save_lighterglue_state.

Test / measurement infrastructure: the repository does not carry the matcher weights.  oracle/_ref/ is git-ignored; the file is a
build output that travels with the working tree to machines without the reference, where the LighterGlue tests and
tools/bench_lighterglue.py read it (and the package reads it through XFeat(lighterglue_weights=...)).

    python oracle/build_lighterglue.py     # needs the reference checkout; prints the output path
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("XFEAT_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref", "lighterglue_state.npz")


def build(force: bool = False) -> str | None:
    """Write OUT from the reference's xfeat-lighterglue.pt.  Returns OUT, or None when neither the reference nor a previously
    built file is present."""
    src = os.path.join(REF_ROOT, "weights", "xfeat-lighterglue.pt")
    if not os.path.exists(src):
        return OUT if os.path.exists(OUT) else None
    if force or not os.path.exists(OUT) or os.path.getmtime(OUT) < os.path.getmtime(src):
        sys.path.insert(0, os.path.dirname(HERE))
        from accelerated_features_b200 import weights
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        weights.save_lighterglue_state(src, OUT)
    return OUT


def path() -> str:
    """OUT; raises when it has not been built."""
    if not os.path.exists(OUT):
        raise RuntimeError(f"{OUT} is not built: run `python oracle/build_lighterglue.py` where the reference checkout "
                           "(weights/xfeat-lighterglue.pt) is available")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
