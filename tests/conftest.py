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


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def lego_bitfield():
    return np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"].copy()


from oracle.train_step import make_rays  # noqa: E402  (shared with bench.py's CPU arm)


@pytest.fixture(scope="session")
def rays_factory():
    return make_rays
