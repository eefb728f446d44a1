import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """Without a CUDA device the gpu-marked tests are skipped (not failed) when someone runs the whole directory."""
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _seed():
    import random

    import numpy as np
    import torch

    torch.manual_seed(0)
    np.random.seed(0)
    random.seed(0)
    yield


@pytest.fixture(scope="session")
def golden():
    from tests._golden_check import load

    return load()
