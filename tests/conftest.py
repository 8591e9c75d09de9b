import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def rel_err(a, b):
    """relative norm ||a-b|| / (||a|| + ||b||), as testing/eigen_utils.hpp:104-108 of the reference"""
    import numpy as np
    a = np.asarray(a, dtype=np.float64).ravel()
    b = np.asarray(b, dtype=np.float64).ravel()
    den = np.linalg.norm(a) + np.linalg.norm(b)
    if den == 0:
        return 0.0
    return float(np.linalg.norm(a - b) / den)


@pytest.fixture(scope="session")
def tiny_problem():
    from rootba_b200.synthetic import synth_bal
    return synth_bal(12, 300, 4.1, seed=1)


@pytest.fixture(scope="session")
def small_problem():
    # shape of BASELINE.json configs[0] (ladybug-49-7776) shrunk to run in seconds
    from rootba_b200.synthetic import synth_bal
    return synth_bal(49, 1800, 4.1, seed=38401)
