import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a box without a CUDA device (or without the built library) skips the gpu tests instead
    of failing them; on a GPU box nothing is skipped, and the product itself still raises without a device."""
    def have_gpu():
        try:
            from superlu_dist_b200 import capi
            return capi.device_count() >= 1
        except Exception:
            return False
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if gpu_items and not have_gpu():
        skip = pytest.mark.skip(reason="no CUDA device / libslu_b200.so: gpu tests need an H100")
        for it in gpu_items:
            it.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the host library and the oracle once (cheap; CUDA is built by __graft_entry__.build())."""
    import __graft_entry__ as g
    g.build_host()
    g.build_oracle()
    yield
