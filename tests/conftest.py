import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    import torch
    # the CPU oracle scales poorly past ~32 threads on the many-core GPU hosts
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """The C-ABI library must exist for every test tier (nvcc cross-compiles without a GPU)."""
    from michigan_b200 import build
    build.build()
    yield
