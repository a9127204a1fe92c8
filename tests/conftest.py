import os
import sys

import numpy as np
import pytest

# the library caches its environment switches at the first dispatch; the tests flip them per test
os.environ.setdefault("OSVOS_ENV_RELOAD", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    path = os.path.join(ROOT, "tests", "golden", "reference_outputs.npz")
    with np.load(path, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}
