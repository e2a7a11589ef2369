import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    try:  # the oracle's small GEMMs are far slower with one thread per hardware thread on a 128-thread host
        import torch

        torch.set_num_threads(min(16, os.cpu_count() or 1))
    except Exception:  # pragma: no cover
        pass


def pytest_collection_modifyitems(config, items):
    """GPU tests fail loudly (not skip) on a GPU box; without a device they are deselected by -m 'not gpu'."""
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
