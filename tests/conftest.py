"""pytest configuration: registers the `gpu` marker and puts the repo root on sys.path."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs an H100 (sm_90a); run with -m gpu")


def _cuda_ok():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


GPU_TEST_TIMEOUT_S = 300      # the whole GPU suite takes ~20 s; a hung kernel must not take the box with it


def pytest_collection_modifyitems(config, items):
    if _cuda_ok():
        # pytest-timeout, thread method: a test stuck inside a CUDA call (signals are not delivered there) is
        # reported with a stack dump and the process exits, instead of hanging until the box's own limit
        if config.pluginmanager.hasplugin("timeout"):
            for item in items:
                if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                    item.add_marker(pytest.mark.timeout(GPU_TEST_TIMEOUT_S, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
