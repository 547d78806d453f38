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


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def load(name):
        if name not in cache:
            cache[name] = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
        return cache[name]

    return load
