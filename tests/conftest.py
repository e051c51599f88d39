import os
import sys
from pathlib import Path

import pytest

# before anything creates a CUDA context (see faabric_b200/__init__.py)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def _cuda_ok():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _cuda_ok():
        # a wedged stream must cost minutes, not the whole session: the
        # thread method ends the process even while it is blocked inside CUDA
        for item in items:
            if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                item.add_marker(pytest.mark.timeout(420, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords or "multigpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def native_lib():
    from faabric_b200 import _lib

    return _lib.load()
