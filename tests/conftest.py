import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90)")


@pytest.fixture(scope="session")
def built():
    """Make sure the native libraries exist (oracle + engine)."""
    import __graft_entry__ as g
    g.build_if_needed()
    return True


@pytest.fixture(scope="session")
def gpu_ctx(built):
    from nrtsearch_b200.search import GpuContext
    ctx = GpuContext(0)
    yield ctx
    ctx.close()
