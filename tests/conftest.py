import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLDEN = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def golden():
    class G(object):
        def __init__(self):
            self._c = {}

        def __getitem__(self, name):
            if name not in self._c:
                self._c[name] = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
            return self._c[name]

    return G()
