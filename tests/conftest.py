import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with `-m gpu`)")
    # (pytest-timeout registers this itself; declared here so that the suite also collects cleanly without the plugin)
    config.addinivalue_line("markers", "timeout(seconds): per-test time limit of the launcher-level integration tests")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
