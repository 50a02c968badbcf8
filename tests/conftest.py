import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def mcb():
    """the built package; builds libmcb200.so on demand (nvcc cross-compiles without a GPU)"""
    lib = os.path.join(ROOT, "open-solution-mapping-challenge_b200", "libmcb200.so")
    if not os.path.exists(lib):
        import __graft_entry__
        __graft_entry__.build()
    import mcb200
    return mcb200


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test started without a CUDA device")
    return torch.device("cuda:0")
