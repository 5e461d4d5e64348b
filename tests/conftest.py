import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    import torch

    torch.set_num_threads(min(8, os.cpu_count() or 1))  # the oracle's small CPU ops crawl with 100+ threads
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Every test session starts from a built libgsx.so (nvcc cross-compiles on CPU-only machines)."""
    from gradslam_b200 import build

    build.build()
