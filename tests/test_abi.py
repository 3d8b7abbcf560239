"""CPU-side checks of the C-ABI boundary: the library builds for sm_90a, loads, and exports exactly the symbols
include/xfeat_b200.h declares (no compute calls: there is no GPU here)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    from accelerated_features_b200.build import build_library
    return build_library()


def header_symbols():
    src = open(os.path.join(ROOT, "include", "xfeat_b200.h")).read()
    return sorted(set(re.findall(r"XF_API [\w\s\*]+?\b(xfeat_\w+)\s*\(", src)))


def test_header_matches_binding_table():
    from accelerated_features_b200 import _lib
    assert header_symbols() == sorted(_lib.SIGNATURES)


def test_library_exports_every_declared_symbol(lib_path):
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    for s in header_symbols():
        assert s in exported, s
    assert {e for e in exported if e.startswith("xfeat_")} == set(header_symbols())   # nothing undeclared leaks out


def test_library_loads_and_reports(lib_path):
    from accelerated_features_b200 import _lib, weights
    lib = _lib.load()
    assert lib.xfeat_abi_version() == _lib.ABI_VERSION == 2
    blob = weights.pack_weights(weights.load_state_dict(weights.DEFAULT_WEIGHTS))
    assert blob.dtype == np.float32 and blob.size == lib.xfeat_packed_weight_floats()
    assert lib.xfeat_launch_count() == 0


def test_sass_is_sm90a_only(lib_path):
    out = subprocess.run(["cuobjdump", "--list-elf", lib_path], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_product_never_imports_oracle():
    """The shipped package must not reach into oracle/ (parity claims depend on it)."""
    pkg = os.path.join(ROOT, "accelerated_features_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                assert "oracle" not in open(os.path.join(dp, f)).read(), f


def test_missing_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from accelerated_features_b200 import XFeat
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        XFeat()
