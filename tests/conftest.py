import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run with -m gpu on an H100)')


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + '.npz')))


@pytest.fixture
def golden():
    return load_golden


def assert_close(actual, expected, rtol=1e-5, atol=None, what=''):
    """Tensor-level relative check: |a-e|_max <= rtol*|e|_max (+ atol)."""
    a = np.asarray(actual, dtype=np.float64)
    e = np.asarray(expected, dtype=np.float64)
    assert a.shape == e.shape, (what, a.shape, e.shape)
    scale = np.abs(e).max() if e.size else 0.0
    tol = rtol * scale + (atol or 0.0)
    err = np.abs(a - e).max() if e.size else 0.0
    assert err <= tol, '%s: max err %.3e > tol %.3e (scale %.3e)' % (what, err, tol, scale)
