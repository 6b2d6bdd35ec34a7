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
        import ctypes
        lib = ctypes.CDLL(os.path.join(ROOT, "sedumi_b200", "libsedumi_b200.so"))
        return lib.sb200_device_count() > 0
    except OSError:
        return False


@pytest.fixture(autouse=True)
def _reference_answers(request):
    """After each test: write its recorded reference answers, or check that it asked for all of them."""
    yield
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import replay
    replay.finish(request.node.nodeid)


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
