import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


def rel_l2(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    m = np.isfinite(a) & np.isfinite(b)
    return float(np.linalg.norm(a[m] - b[m]) / max(np.linalg.norm(b[m]), 1e-30))


@pytest.fixture(scope="session")
def golden():
    return load_golden
