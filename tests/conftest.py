import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100 box)")
    config.addinivalue_line("markers", "multigpu: needs at least 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    import torch
    has = torch.cuda.is_available()
    n = torch.cuda.device_count() if has else 0
    for item in items:
        if "gpu" in item.keywords and not has:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and n < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 CUDA devices"))
