import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible and the run did
    not explicitly ask for them; with `-m gpu` on a GPU-less host they fail loudly."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    asked = "gpu" in (config.getoption("-m") or "") and "not gpu" not in (config.getoption("-m") or "")
    if asked:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
