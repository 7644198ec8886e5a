import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with `-m gpu`)")


@pytest.fixture(scope="session")
def native_lib():
    """Build (incrementally) and load libsonar_b200.so; the build cross-compiles without a GPU."""
    from sonar_b200 import _lib, build

    build.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    return torch.device("cuda:0")
