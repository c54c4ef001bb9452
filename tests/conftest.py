import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    # A GPU test on a box without a GPU is a hard error when explicitly selected with -m gpu, and is
    # skipped otherwise (so `pytest tests/` on a CPU box stays green).
    import torch

    if torch.cuda.is_available():
        return
    selected_gpu = "gpu" in (config.getoption("-m") or "") and "not gpu" not in (config.getoption("-m") or "")
    if selected_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def lib_built():
    """Build the C-ABI library once per session (nvcc cross-compiles without a GPU)."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("lvb200_build", os.path.join(ROOT, "long-vita_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()
