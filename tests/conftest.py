import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "sc-sfmlearner-release_b200")
GOLDEN = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, PKG, GOLDEN):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_warp():
    return np.load(os.path.join(GOLDEN, "warp_loss.npz"))


@pytest.fixture(scope="session")
def golden_nets():
    return np.load(os.path.join(GOLDEN, "nets.npz"))
