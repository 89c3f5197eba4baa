"""ivb_rope_qk and the SwiGLU epilogue of ivb_gemm_bf16 refuse bad operands before any CUDA call.  Checked through the
raw C ABI with fake device addresses (tests/abi_fake.py), so these tests run only where no CUDA device is visible."""
import pytest

from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll

pytestmark = cpu_only

Q, K, COS, SIN, A, B, OUT, BIAS = (BASE + k * 0x10000000 for k in range(8))


def _rope(q=Q, ldq=3 * 4096, k=K, ldk=3 * 4096, B=2, L=32, H=32, d=128, cos=COS, sin=SIN):
    return _lib.load().ivb_rope_qk(q, ldq, k, ldk, B, L, H, d, cos, sin, None)


def test_rope_refusals():
    expect_refusal(_rope(q=None), "q, k, cos and sin are required")
    expect_refusal(_rope(sin=None), "q, k, cos and sin are required")
    for d in (8, 72, 144):
        expect_refusal(_rope(d=d, H=4), "d a multiple of 16 in [16, 128]")
    expect_refusal(_rope(H=0), "H > 0")
    expect_refusal(_rope(ldq=4100), "ldq and ldk must be multiples of 8")
    expect_refusal(_rope(ldk=4088), ">= H*d")
    expect_refusal(_rope(q=Q + 8), "16-byte aligned")
    expect_refusal(_rope(cos=COS + 4), "16-byte aligned")
    assert _rope(B=0) == 0 and _rope(L=0) == 0          # empty: a no-op


def _swiglu(M=256, N=2 * 344, Kd=512, b_mn=0, flags=0, out1=None, bias=None, tile_n=0, ld0=344, plan=False):
    lib = _lib.load()
    args = (A, 0, Kd, B, b_mn, Kd if not b_mn else N, M, N, Kd, ll.EPI_SWIGLU, flags, OUT, ld0, out1, 344 if out1 else 0,
            bias, None, None, 0, None, tile_n)
    if plan:
        return lib.ivb_gemm_bf16_plan(*args, BASE, None, None)
    return lib.ivb_gemm_bf16(*args, None)


def test_swiglu_refusals():
    expect_refusal(_swiglu(b_mn=1), "needs a K-major B")
    expect_refusal(_swiglu(N=2 * 340), "I a multiple of 8")
    expect_refusal(_swiglu(bias=BIAS), "no bias and no out1")
    expect_refusal(_swiglu(out1=BIAS), "no bias and no out1")
    expect_refusal(_swiglu(flags=ll.FLAG_ACCUM), "excludes IVB_FLAG_ACCUM and IVB_FLAG_2CTA")
    expect_refusal(_swiglu(flags=ll.FLAG_2CTA), "excludes IVB_FLAG_ACCUM and IVB_FLAG_2CTA")
    expect_refusal(_swiglu(plan=True), "no DropPath plan form")


def test_swiglu_is_bf16_only():
    lib = _lib.load()
    rc = lib.ivb_gemm_fp8(A, 0, 512, 0, BASE, B, 0, 512, BASE, 256, 688, 512, ll.EPI_SWIGLU, 0, OUT, 344, None, 0, None,
                          None, None, 0, None, 0, None)
    expect_refusal(rc, "IVB_EPI_SWIGLU is bf16 only")
