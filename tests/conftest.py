import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _gpu_available() -> bool:
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """Without a CUDA device the GPU tests are skipped, not failed (a plain `pytest tests` stays green on a CPU
    box; the GPU box runs them with -m gpu)."""
    if _gpu_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (the pick path has no CPU fallback)")
    for item in items:
        if "gpu" in item.keywords or os.path.basename(str(item.fspath)).startswith("test_gpu_"):
            item.add_marker(skip)


@pytest.fixture(scope="session")
def gpu_count() -> int:
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the in-tree libraries once if they are missing (CPU box: nvcc cross-compiles)."""
    import __graft_entry__ as ge

    ge.ensure_built()
