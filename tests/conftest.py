import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
WEIGHTS = os.path.join(ROOT, "weights")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100")


@pytest.fixture(scope="session")
def built_lib():
    """libnisqa_b200.so, (re)built in-tree if the sources changed."""
    from nisqa_b200 import build
    return build.build()


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # GPU tests fail loudly (never silently skip) when selected on a box without a GPU, except
    # when the whole suite is run unfiltered on the CPU box.
    if _has_cuda():
        return
    markexpr = config.getoption("-m") or ""
    if "gpu" in markexpr and "not gpu" not in markexpr:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
