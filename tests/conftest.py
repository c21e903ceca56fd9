import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU; run with -m gpu")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available() and torch.cuda.get_device_capability(0)[0] == 9
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no sm_90 GPU")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
