import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")


def pytest_collection_modifyitems(config, items):
    """a plain `pytest tests` on a machine without CUDA skips the GPU tests instead of reporting them as failures"""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs an H100 (no CUDA device here)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def cabi():
    """The C-ABI binding with the in-tree library built (nvcc cross-compiles without a GPU)."""
    from adaptive_classifier_b200 import build as _b
    _b.build_library()
    from adaptive_classifier_b200 import _cabi
    _cabi.load_library()
    return _cabi
