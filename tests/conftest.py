import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "midi-model_b200")
for p in (PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def golden_tiny():
    import numpy as np
    return dict(np.load(os.path.join(GOLDEN, "tiny.npz")))


@pytest.fixture(scope="session")
def golden_medium():
    import numpy as np
    return dict(np.load(os.path.join(GOLDEN, "medium.npz")))
