import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


GPU_TEST_TIMEOUT_S = 180  # the longest GPU test takes seconds; a kernel that never returns must not hold the GPU


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        # watchdog (pytest-timeout, thread method: dumps the stacks and os._exit()s - a blocked cudaStreamSynchronize cannot be
        # interrupted by a signal)
        if config.pluginmanager.hasplugin("timeout"):
            for item in items:
                if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                    item.add_marker(pytest.mark.timeout(GPU_TEST_TIMEOUT_S, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
