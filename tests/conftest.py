import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with `-m gpu`")


@pytest.fixture(scope="session")
def built():
    """Build the in-tree shared objects once (product library + oracle)."""
    import __graft_entry__ as g
    g.build()
    return True


@pytest.fixture(scope="session")
def oracle(built):
    from oracle import oracle as O
    O.lib()
    return O
