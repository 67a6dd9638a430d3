import os
import sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests", "support")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_golden.npz"))


@pytest.fixture(scope="session")
def track():
    from oracle.track import TrackTable
    return TrackTable(0.4)
