import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def built():
    """the CUDA library (cross-compiled; the host-side builder and the ABI tests need it without a GPU too), the
    oracle and, where the reference's sources are at hand (oracle/Makefile, REF), the reference build -- a no-op when they are up to date"""
    import __graft_entry__ as g
    return g.build()
