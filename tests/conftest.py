import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def lib():
    from nerf_slam_b200 import _lib
    return _lib.load(require_cuda=False)


@pytest.fixture
def rng():
    return np.random.default_rng(1234)
