import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    has_cuda = torch.cuda.is_available()
    ngpu = torch.cuda.device_count() if has_cuda else 0
    for item in items:
        if "gpu" in item.keywords and not has_cuda:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
