import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


def _have_gpu() -> bool:
    try:
        from gslam_b200 import capi
        import ctypes
        n = ctypes.c_int(0)
        return capi.lib().gb_device_count(ctypes.byref(n)) == 0 and n.value > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a device must fail loudly, not silently pass/skip: only auto-skip when gpu tests were
    # not explicitly requested.
    if "gpu" in (config.getoption("-m") or ""):
        return
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def ctx():
    from gslam_b200.api import Context
    c = Context(0)
    yield c
    c.close()
