import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))  # oracle modules are test infrastructure
sys.path.insert(0, str(ROOT / "synth_weights"))  # seeded random-init weights (no checkpoints exist)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "reference: needs /root/reference (build container only)")


@pytest.fixture(scope="session")
def golden_dir():
    return ROOT / "tests" / "golden"


def cuda_available() -> bool:
    import torch

    return torch.cuda.is_available()


def pytest_collection_modifyitems(config, items):
    have_cuda = None
    for item in items:
        if "gpu" in item.keywords:
            if have_cuda is None:
                have_cuda = cuda_available()
            if not have_cuda:
                item.add_marker(pytest.mark.skip(reason="no CUDA device"))
