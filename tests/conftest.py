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
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        # a wedged kernel or lock must fail the run, not hang it: the timer thread ends the process even when the
        # main thread sits inside a CUDA call (pytest-timeout, thread method)
        if config.pluginmanager.hasplugin("timeout"):
            for it in items:
                if "gpu" in it.keywords and not it.get_closest_marker("timeout"):
                    it.add_marker(pytest.mark.timeout(420, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
