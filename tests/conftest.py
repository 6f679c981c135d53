import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    path = os.path.join(ROOT, "tests", "golden", "reference_golden.npz")
    return dict(np.load(path))
