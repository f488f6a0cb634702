import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # a wedged kernel must not eat the GPU budget: every GPU test gets a hard per-test timeout
    try:
        import pytest_timeout  # noqa: F401
        for item in items:
            if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                item.add_marker(pytest.mark.timeout(300))
    except ImportError:
        pass
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
