import os
import sys

import pytest

# virtual ranks sharing one GPU (tests/test_gpu_worker.py) need one hardware queue per stream: must be set before CUDA starts
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import oracle as o

    o.lib()
    return o
