import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def built():
    """Build the CUDA library and the oracle once per session (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as g

    g.build()
    return True


@pytest.fixture(scope="session")
def oracle(built):
    from oracle import oracle as O

    O.lib()
    return O


@pytest.fixture()
def engine(built):
    import fma_b200

    eng = fma_b200.Engine(0)
    yield eng
    eng.close()
