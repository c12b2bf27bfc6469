import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (tests only). Built on demand."""
    import oracle

    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def cb():
    """ctypes binding of the product library; fails loudly if it was not built."""
    from cilantro_b200 import capi

    capi.lib()
    return capi


@pytest.fixture(scope="session")
def ctx(cb):
    """A device context. GPU tests must NOT skip when the device is missing: they fail."""
    c = cb.Context(0)
    yield c
    c.close()


def frob(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - np.asarray(b, np.float64)))
