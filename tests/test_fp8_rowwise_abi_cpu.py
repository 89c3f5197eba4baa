"""Per-row FP8 entry points without a GPU.

1. ivb_fp8_quantize_rows, ivb_norm_fwd_fp8 and ivb_gemm_fp8 with IVB_FLAG_FP8_VECTOR_SCALES refuse a call their
   kernels cannot serve before any CUDA call.  They are called through the raw C ABI with fake device addresses, which
   must never reach a launch, so these checks run only where no CUDA device is visible.
2. The SASS of the vector-scale GEMM kernels: E4M3 x E4M3 QGMMA, no local memory, one epilogue body.
"""
import re

import pytest

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

EPI_BF16 = 0
FLAG_2CTA, FLAG_VEC = 8, 64
E4M3, E5M2 = 0, 1
M, N, K = 417, 1000, 592
SA, SB = BASE + 0x700000, BASE + 0x710000    # fake scale vectors


def _rows(x=BASE, ldx=K, m=M, k=K, out=BASE + 0x300000, ldo=608, sinv=SA):
    return _lib.load().ivb_fp8_quantize_rows(x, ldx, m, k, out, ldo, sinv, None)


def _norm(x=BASE, x_f32=1, ldx=1408, w=BASE + 0x100000, b=None, ln=1, m=M, d=1408, out=BASE + 0x300000, ldo=1408,
          sinv=SA):
    return _lib.load().ivb_norm_fwd_fp8(x, x_f32, ldx, w, b, 1e-5, ln, m, d, out, ldo, sinv, None)


def _gemm(a_fmt=E4M3, sa=SA, sb=SB, flags=FLAG_VEC):
    return _lib.load().ivb_gemm_fp8(BASE + 0x100000, 0, K, a_fmt, sa, BASE + 0x200000, 0, K, sb, M, N, K, EPI_BF16,
                                    flags, BASE, N, None, 0, None, None, None, 0, None, 0, None)


@cpu_only
def test_quantize_rows_refusals():
    expect_refusal(_rows(m=0), "ivb_fp8_quantize_rows: empty tensor")
    expect_refusal(_rows(k=0), "ivb_fp8_quantize_rows: empty tensor")
    expect_refusal(_rows(k=16392, ldx=16392, ldo=16400), "ivb_fp8_quantize_rows: K > IVB_FP8_ROWS_MAX_K")
    expect_refusal(_rows(x=None), "ivb_fp8_quantize_rows: x, out or row_scale_inv is null")
    expect_refusal(_rows(out=None), "ivb_fp8_quantize_rows: x, out or row_scale_inv is null")
    expect_refusal(_rows(sinv=None), "ivb_fp8_quantize_rows: x, out or row_scale_inv is null")
    expect_refusal(_rows(ldx=K + 4), "ivb_fp8_quantize_rows: ldx must be a multiple of 8 elements and >= K")
    expect_refusal(_rows(ldx=584), "ivb_fp8_quantize_rows: ldx must be a multiple of 8 elements and >= K")
    expect_refusal(_rows(ldo=600), "ivb_fp8_quantize_rows: ldo must be a multiple of 16 elements and >= K")
    expect_refusal(_rows(ldo=576), "ivb_fp8_quantize_rows: ldo must be a multiple of 16 elements and >= K")
    expect_refusal(_rows(x=BASE + 8), "ivb_fp8_quantize_rows: x and out must be 16-byte aligned")
    expect_refusal(_rows(out=BASE + 0x300008), "ivb_fp8_quantize_rows: x and out must be 16-byte aligned")
    expect_refusal(_rows(sinv=SA + 2), "ivb_fp8_quantize_rows: row_scale_inv must be 4-byte aligned")


@cpu_only
def test_norm_fwd_fp8_refusals():
    expect_refusal(_norm(m=0), "ivb_norm_fwd_fp8: empty tensor")
    for d in (0, 1404, 4104):
        expect_refusal(_norm(d=d, ldx=4104, ldo=4112),
                       "ivb_norm_fwd_fp8: D must be a multiple of 8 in [8, IVB_NORM_FP8_MAX_D]")
    expect_refusal(_norm(ldx=1412), "ivb_norm_fwd_fp8: ldx must be a multiple of 8 elements and >= D")
    expect_refusal(_norm(ldx=1400), "ivb_norm_fwd_fp8: ldx must be a multiple of 8 elements and >= D")
    expect_refusal(_norm(ldo=1416), "ivb_norm_fwd_fp8: ldo must be a multiple of 16 elements and >= D")
    expect_refusal(_norm(ldo=1392), "ivb_norm_fwd_fp8: ldo must be a multiple of 16 elements and >= D")
    for kw in (dict(x=None), dict(w=None), dict(out=None), dict(sinv=None)):
        expect_refusal(_norm(**kw), "ivb_norm_fwd_fp8: x, weight, out or row_scale_inv is null")
    for kw in (dict(x=BASE + 8), dict(w=BASE + 0x100008), dict(b=BASE + 0x200008), dict(out=BASE + 0x300008)):
        expect_refusal(_norm(**kw), "ivb_norm_fwd_fp8: x, weight, bias and out must be 16-byte aligned")
    expect_refusal(_norm(sinv=SA + 2), "ivb_norm_fwd_fp8: row_scale_inv must be 4-byte aligned")


@cpu_only
def test_gemm_vector_scale_refusals():
    expect_refusal(_gemm(a_fmt=E5M2), "ivb_gemm_fp8: vector scales need an E4M3 A operand")
    expect_refusal(_gemm(sa=None), "ivb_gemm_fp8: scale_inv pointers are null")
    expect_refusal(_gemm(sb=None), "ivb_gemm_fp8: scale_inv pointers are null")
    expect_refusal(_gemm(flags=FLAG_VEC | FLAG_2CTA), "ivb_gemm_fp8: no CTA-pair kernel")
    expect_refusal(_gemm(sa=SA + 4), "ivb_gemm_fp8: scale vectors must be 8-byte aligned")
    expect_refusal(_gemm(sb=SB + 4), "ivb_gemm_fp8: scale vectors must be 8-byte aligned")


# ------------------------------------------------------------------------------------------------ SASS
@pytest.fixture(scope="module")
def vec_kernels():
    """{kernel name: [SASS instruction lines]} of the vector-scale FP8 GEMM kernels (Op = OpVecFp8) in ivb_gemm.o."""
    out = {k: v for k, v in sass.functions("ivb_gemm.o").items() if "OpVecFp8" in k}
    assert len(out) == 3, sorted(out)     # ping-pong, cooperative BN 128 and 192
    return out


def test_vector_scale_kernels_sass(vec_kernels):
    for name, lines in vec_kernels.items():
        q = [l for l in lines if re.search(r"\bQGMMA\.", l)]
        assert q and not any(re.search(r"\bHGMMA\b", l) for l in lines), name
        assert all(re.search(r"QGMMA\.64x\d+x32\.F32\.E4M3\.E4M3\b", l) for l in q), name
        assert not any(re.search(r"\b(LDL|STL)\b", l) for l in lines), name
        assert 0 < sum(1 for l in lines if "MUFU.TANH" in l) <= 64, name
