"""Refusals through the raw C ABI with fake device addresses.  An entry point must refuse such a call before any CUDA
call; were a check missing, the call would go on to launch a kernel on the fake addresses, so the tests that pass them
run only where no CUDA device is visible (cpu_only)."""
import pytest
import torch

from internvideo_b200 import _lib

BASE = 1 << 32                               # fake, 256-byte aligned device addresses
cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="passes fake device pointers: CPU-only check")


def expect_refusal(rc, text):
    """The call returned a non-zero status and ivb_last_error() contains text."""
    assert rc != 0
    msg = _lib.load().ivb_last_error().decode()
    assert text in msg, msg
