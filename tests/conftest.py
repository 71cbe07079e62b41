import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
if os.path.dirname(os.path.abspath(__file__)) not in sys.path:
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _have_gpu():
    try:
        from gpy_b200 import _ffi
        return _ffi.lib().gpx_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def have_gpu():
    return _have_gpu()


def pytest_collection_modifyitems(config, items):
    """GPU-marked tests are skipped (not failed) on a box without a CUDA device or without the built library."""
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device (or libgpx.so not built)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
