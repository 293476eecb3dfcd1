import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _has_gpu():
    try:
        from omniswarm_b200 import lib
        return lib.load().osb_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu():
    """GPU tests must FAIL (not skip) when the CUDA library is missing on a GPU box; they are only deselected by -m."""
    from omniswarm_b200 import lib
    L = lib.load()
    assert L.osb_device_count() > 0, "no CUDA device visible: -m gpu tests need an H100"
    return L


GOLDEN = os.path.join(ROOT, "tests", "golden")
