import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """Make sure the CUDA library and the oracle are built (cross-compiles without a GPU)."""
    import __graft_entry__ as g
    g.build()
    return True


@pytest.fixture(scope="session")
def gpu(built):
    from tuplex_b200 import backend
    if backend.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests must run on a GPU box (the backend has no CPU fallback)")
    backend.init([0])
    return 0
