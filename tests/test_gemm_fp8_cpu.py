"""FP8 GEMM and quantisation without a GPU.

1. ivb_gemm_fp8 and ivb_fp8_quantize refuse a call their kernels cannot serve (an MN-major operand, an operand pitch
   that is not a multiple of 16 elements, null scale pointers, misaligned outputs) before any CUDA call.  They are
   called through the raw C ABI with fake device addresses, which must never reach a launch, so these checks run only
   where no CUDA device is visible.
2. The SASS of the FP8 GEMM kernels: QGMMA with the expected formats and no HGMMA, no local memory, one epilogue body.
"""
import re

import pytest

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

EPI_BF16, EPI_F32, EPI_BIAS_GELU, EPI_RESID, EPI_GELU_BWD = 0, 1, 2, 3, 4
FLAG_1CTA, FLAG_2CTA, FLAG_PINGPONG = 4, 8, 32
E4M3, E5M2 = 0, 1
M, N, K = 417, 1000, 592
SA, SB = BASE + 0x700000, BASE + 0x700010    # fake scale_inv scalars


def _gemm(a_mn=0, lda=K, a_fmt=E4M3, sa=SA, b_mn=0, ldb=K, sb=SB, epi=EPI_BF16, flags=0, out0=BASE, ld0=N,
          out1=None, ld1=0, bias=None, gamma=None, aux=None, ldaux=0, tile_n=0):
    lib = _lib.load()
    return lib.ivb_gemm_fp8(BASE + 0x100000, a_mn, lda, a_fmt, sa, BASE + 0x200000, b_mn, ldb, sb, M, N, K, epi, flags,
                            out0, ld0, out1, ld1, bias, gamma, aux, ldaux, None, tile_n, None)


def _quant(ldx=K, fmt=E4M3, out=BASE + 0x300000, ldo=608, out_t=None, ldt=0, amax=SA, scale_inv=SB, x=BASE):
    lib = _lib.load()
    return lib.ivb_fp8_quantize(x, ldx, M, K, fmt, out, ldo, out_t, ldt, amax, scale_inv, None)


@cpu_only
@pytest.mark.parametrize("a_mn,b_mn", [(1, 0), (0, 1), (1, 1)])
def test_gemm_fp8_mn_major_refused(a_mn, b_mn):
    expect_refusal(_gemm(a_mn=a_mn, b_mn=b_mn), "ivb_gemm_fp8: both operands must be K-major")


@cpu_only
@pytest.mark.parametrize("lda,ldb", [(K + 8, K), (K, K + 8), (600, 600), (K + 1, K)])
def test_gemm_fp8_operand_pitch_refused(lda, ldb):
    expect_refusal(_gemm(lda=lda, ldb=ldb), "ivb_gemm_fp8: lda and ldb must be multiples of 16 elements")


@cpu_only
@pytest.mark.parametrize("sa,sb", [(None, SB), (SA, None), (None, None)])
def test_gemm_fp8_null_scale_refused(sa, sb):
    expect_refusal(_gemm(sa=sa, sb=sb), "ivb_gemm_fp8: scale_inv pointers are null")


@cpu_only
@pytest.mark.parametrize("slot", ["out0", "out1", "aux", "bias", "gamma"])
def test_gemm_fp8_epilogue_pointer_alignment_refused(slot):
    ptrs = dict(out0=BASE, out1=BASE + 0x300000, aux=BASE + 0x500000, bias=BASE + 0x400000, gamma=BASE + 0x600000)
    ptrs[slot] += 8
    expect_refusal(_gemm(epi=EPI_RESID, out0=ptrs["out0"], out1=ptrs["out1"], ld1=N, bias=ptrs["bias"],
                         gamma=ptrs["gamma"], aux=ptrs["aux"], ldaux=N),
                   f"ivb_gemm_fp8: {slot} must be 16-byte aligned")


@cpu_only
def test_gemm_fp8_other_refusals():
    expect_refusal(_gemm(ld0=N + 4), "ivb_gemm_fp8: N and ld0 must be multiples of 8 elements")
    expect_refusal(_gemm(a_fmt=2), "ivb_gemm_fp8: unknown a_format")
    expect_refusal(_gemm(epi=EPI_GELU_BWD), "ivb_gemm_fp8: epilogue needs aux")
    expect_refusal(_gemm(epi=EPI_BIAS_GELU, out1=BASE + 0x300000, ld1=N + 2),
                   "ivb_gemm_fp8: ld1 must be a multiple of 8")
    expect_refusal(_gemm(flags=FLAG_2CTA), "ivb_gemm_fp8: no CTA-pair kernel")
    expect_refusal(_gemm(flags=FLAG_1CTA | FLAG_PINGPONG), "exclude each other")
    expect_refusal(_gemm(tile_n=256), "ivb_gemm_fp8: tile_n must be 0, 128 or 192")
    expect_refusal(_gemm(flags=FLAG_PINGPONG, tile_n=192), "ivb_gemm_fp8: the ping-pong kernel has tile_n 128")


@cpu_only
def test_fp8_quantize_refusals():
    expect_refusal(_quant(ldo=600), "ivb_fp8_quantize: ldo must be a multiple of 16 elements and >= K")
    expect_refusal(_quant(ldo=576), "ivb_fp8_quantize: ldo must be a multiple of 16 elements and >= K")
    expect_refusal(_quant(out_t=BASE + 0x400000, ldt=424),
                   "ivb_fp8_quantize: ldt must be a multiple of 16 elements and >= M")
    expect_refusal(_quant(out_t=BASE + 0x400000, ldt=400),
                   "ivb_fp8_quantize: ldt must be a multiple of 16 elements and >= M")
    expect_refusal(_quant(ldx=K + 4), "ivb_fp8_quantize: ldx must be a multiple of 8 elements and >= K")
    expect_refusal(_quant(amax=None), "ivb_fp8_quantize: amax or scale_inv is null")
    expect_refusal(_quant(scale_inv=None), "ivb_fp8_quantize: amax or scale_inv is null")
    expect_refusal(_quant(fmt=2), "ivb_fp8_quantize: unknown format")
    for kw in (dict(out=BASE + 0x300008), dict(out_t=BASE + 0x400008, ldt=432), dict(x=BASE + 8)):
        expect_refusal(_quant(**kw), "ivb_fp8_quantize: x, out and out_t must be 16-byte aligned")
    expect_refusal(_quant(amax=SA + 2), "ivb_fp8_quantize: amax and scale_inv must be 4-byte aligned")


# ------------------------------------------------------------------------------------------------ SASS
@pytest.fixture(scope="module")
def fp8_kernels():
    """{kernel name: [SASS instruction lines]} of every FP8 GEMM kernel in ivb_gemm.o."""
    # OpFp8<A_E5M2> in the mangled template arguments: "OpFp8ILb0E" (E4M3 x E4M3) or "OpFp8ILb1E" (E5M2 x E4M3)
    out = {k: v for k, v in sass.functions("ivb_gemm.o").items() if "OpFp8" in k}
    # both formats, ping-pong and the promoting cooperative kernel at BN 128 and 192
    assert len(out) == 6, sorted(out)
    return out


def test_fp8_kernels_issue_qgmma_of_their_formats(fp8_kernels):
    for name, lines in fp8_kernels.items():
        a = "E5M2" if "OpFp8ILb1E" in name else "E4M3"
        assert sass.count(lines, r"\bHGMMA\b") == 0, name
        q = [l for l in lines if re.search(r"\bQGMMA\.", l)]
        assert q, name
        for l in q:
            assert re.search(rf"QGMMA\.64x\d+x32\.F32\.{a}\.E4M3\b", l), (name, l)


def test_fp8_kernels_use_no_local_memory(fp8_kernels):
    for name, lines in fp8_kernels.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, name


def test_fp8_kernels_hold_one_epilogue_body(fp8_kernels):
    for name, lines in fp8_kernels.items():
        assert 0 < sass.count(lines, r"MUFU\.TANH") <= 64, name
