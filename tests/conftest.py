import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests need a CUDA device; without one they are skipped, so a plain `pytest` on a CPU machine is
    green instead of failing inside torch._C._cuda_init.  On a GPU machine nothing is skipped: a missing
    libptranking_b200.so must fail loudly there (there is no fallback path to hide behind)."""
    import torch
    if not torch.cuda.is_available():
        skip = pytest.mark.skip(reason="needs a CUDA device")
        for item in items:
            if "gpu" in item.keywords:
                item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
