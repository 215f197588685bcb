import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    path = os.path.join(ROOT, "tests", "golden", "reference_vectors.npz")
    return dict(np.load(path))
