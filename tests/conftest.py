import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name), allow_pickle=False))


@pytest.fixture(scope="session")
def golden():
    return load_golden


def matches_from(g, tag):
    return {
        "kp1": g[f"{tag}_kp1"],
        "kp2": g[f"{tag}_kp2"],
        "i12": g[f"{tag}_i12"],
        "img_shape": tuple(int(v) for v in g[f"{tag}_img_shape"]),
    }
