import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


def _has_gpu():
    try:
        import gyroflow_b200 as g
        return g.load_library().gf_cuda_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU is a hard error inside the tests (no silent skip); nothing to do here.
    pass


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (tests only).  Built on demand from oracle/ with gcc."""
    from tests import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def gpu_available():
    return _has_gpu()
