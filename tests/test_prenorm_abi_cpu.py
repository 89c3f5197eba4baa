"""ivb_im2col_prenorm and ivb_prenorm_wgrad refuse bad operands before any CUDA call: an odd or short Kpad, a Kpad
past the register-resident row, an odd patch, misaligned pointers, a missing rstd, weight or dweight, a short dcols
pitch.  Checked through the raw C ABI with fake device addresses (tests/abi_fake.py), so these tests run only where no
CUDA device is visible."""
import pytest

from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

pytestmark = cpu_only

VIDEO, IDX, W, COLS, RSTD, DCOLS, DW = (BASE + k * 0x1000000 for k in range(7))
GEOM = dict(B=2, C=3, T=16, H=224, W=224, tubelet=1, patch=14, Kpad=592)


def _fwd(video=VIDEO, idx=IDX, weight=W, cols=COLS, rstd=RSTD, **kw):
    g = dict(GEOM, **kw)
    return _lib.load().ivb_im2col_prenorm(video, idx, 257, 1, 256, g["B"], g["C"], g["T"], g["H"], g["W"],
                                          g["tubelet"], g["patch"], g["Kpad"], weight, 1e-6, cols, rstd, None)


def _wgrad(video=VIDEO, idx=IDX, rstd=RSTD, dcols=DCOLS, lddc=592, dweight=DW, **kw):
    g = dict(GEOM, **kw)
    return _lib.load().ivb_prenorm_wgrad(video, idx, 257, 1, 256, g["B"], g["C"], g["T"], g["H"], g["W"],
                                         g["tubelet"], g["patch"], g["Kpad"], rstd, dcols, lddc, dweight, None)


@pytest.mark.parametrize("call", [_fwd, _wgrad], ids=["im2col_prenorm", "prenorm_wgrad"])
def test_shared_refusals(call):
    expect_refusal(call(Kpad=594), "Kpad must be a multiple of 8")
    expect_refusal(call(Kpad=584), "Kpad must be a multiple of 8, >= C*t*p*p")
    expect_refusal(call(tubelet=4, Kpad=2352), "<= 1536")
    expect_refusal(call(patch=15, Kpad=680), "patch and W even")
    expect_refusal(call(rstd=None), "video, idx and rstd must not be null")
    expect_refusal(call(rstd=RSTD + 2), "4-byte aligned")
    expect_refusal(call(video=VIDEO + 2), "4-byte aligned")


def test_im2col_prenorm_refusals():
    expect_refusal(_fwd(weight=None), "weight and cols must not be null")
    expect_refusal(_fwd(weight=W + 1), "weight 2-byte aligned")
    expect_refusal(_fwd(cols=COLS + 2), "cols must be 4-byte")


def test_prenorm_wgrad_refusals():
    expect_refusal(_wgrad(dweight=None), "dcols and dweight must not be null")
    expect_refusal(_wgrad(lddc=588), "lddc must be a multiple of 8 and >= Kpad")
    expect_refusal(_wgrad(lddc=596), "lddc must be a multiple of 8")
    expect_refusal(_wgrad(dweight=DW + 2), "dcols and dweight must be 4-byte aligned")
