import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100)')


@pytest.fixture(scope='session')
def golden():
    """Reference OUTPUTS recorded by tests/golden/make_golden.py (live reference, CPU torch)."""
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_outputs.npz'))


def maxabs(a, b):
    return float(np.nanmax(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))))
