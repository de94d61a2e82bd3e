import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _has_gpu():
    try:
        from open3d_slam_b200 import _lib
        return _lib.lib().b2s_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def engine_factory():
    """Engines for the -m gpu tests.  Fails loudly (no skip, no fallback) when the CUDA library or the GPU is missing."""
    from open3d_slam_b200 import engine as E

    made = []

    def make(params=None):
        e = E.Engine(params or E.MapperParameters())
        made.append(e)
        return e

    yield make
    for e in made:
        e.close()
