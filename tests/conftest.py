import os
import sys


import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built():
    """Make sure libbnsgcn.so and the oracle's C library exist (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as ge
    ge.build()
    return True
