import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `pytest -m gpu`)")


def pytest_collection_modifyitems(config, items):
    # GPU tests are skipped (not failed) on a box without CUDA unless explicitly selected.
    try:
        import torch

        has_cuda = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_cuda = False
    if has_cuda:
        # A protocol bug in a hand-written kernel (mbarrier / cluster barrier / warpgroup wgmma) hangs
        # instead of failing: every GPU test gets a watchdog that ends the process (the "thread" method works while
        # the main thread is blocked inside a CUDA call), so one hang cannot eat the whole GPU lease.
        for item in items:
            if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                item.add_marker(pytest.mark.timeout(240, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
