import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gps-gaussian_b200", "dropin")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests are skipped (not failed) where there is no CUDA device -- a plain `pytest tests` on a CPU box stays green."""
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100); run with -m gpu on the GPU box")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def built_lib():
    """Build (if stale) and return the path of libgpsg_sm90.so; nvcc cross-compiles without a GPU."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_gpsg_build", os.path.join(ROOT, "gps-gaussian_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()
