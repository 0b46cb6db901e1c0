import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "mega.pytorch_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def cuda_dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mega_core import _lib
    assert _lib.lib.mega_device_ok() == 1, "libmega_b200 kernels are built for sm_90a (H100) only"
    return torch.device("cuda:0")
