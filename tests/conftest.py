import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name)) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def golden():
    return load_golden


@pytest.fixture(scope="session")
def oracle_state():
    from oracle import xfeat_oracle as orc
    return orc.load_state()


@pytest.fixture(scope="session")
def assets_vga():
    g = load_golden("inputs_assets_vga.npz")
    return g["ref"], g["tgt"]
