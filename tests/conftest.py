import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def load_golden(name):
    """Return (arrays, state_dict) of one fixture made by tests/golden/make_golden.py."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    arrays = {k: z[k] for k in z.files if not k.startswith("sd::")}
    sd = {k[4:]: z[k] for k in z.files if k.startswith("sd::")}
    return arrays, sd


@pytest.fixture(scope="session")
def golden():
    return load_golden
