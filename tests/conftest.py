import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 GPU (run with -m gpu on the GPU box)")


@pytest.fixture(scope="session")
def cuda_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from internvideo_b200 import _lib, lowlevel
    _lib.load()
    lowlevel.device_check()
    return lowlevel
