import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), ROOT):
    if p in sys.path:
        sys.path.remove(p)
    sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def _golden_6mrr_file():
    import numpy as np
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "6mrr.npz")))


@pytest.fixture
def golden_6mrr(_golden_6mrr_file):
    # fresh copies for every test: simulate() updates coords / velocities in place, and a System keeps references to its inputs
    return {k: v.copy() for k, v in _golden_6mrr_file.items()}
