import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _build_native():
    """Make sure the oracle and the CUDA library exist (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as ge

    ge.build()
    yield


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a box without a CUDA device: skip (not fail) the gpu-marked tests."""
    try:
        import torch

        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (kaminpar_b200 has no CPU fallback)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
