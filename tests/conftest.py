import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def orc():
    import oracle

    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def gb():
    """The product package; loading it requires the built C-ABI library."""
    import gorse_b200

    return gorse_b200
