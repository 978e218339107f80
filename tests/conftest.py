import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


def _has_gpu():
    try:
        from blaze_b200 import native
        return native.device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def has_gpu():
    return _has_gpu()


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a device must fail loudly, not silently skip: only skip GPU tests
    # when they were not explicitly selected.
    if _has_gpu():
        return
    selected = config.getoption("-m") or ""
    if "gpu" in selected and "not gpu" not in selected:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
