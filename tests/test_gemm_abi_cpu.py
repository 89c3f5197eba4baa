"""ivb_gemm_bf16 refuses an epilogue operand the 16-byte vector accesses of its epilogue cannot serve: a row pitch of
out1 or aux that is not a multiple of the vector width, or a base pointer of out0 / out1 / aux / bias / gamma that is
not 16-byte aligned.  The refusal comes before any CUDA call, so it is checked here through the raw C ABI with fake
device addresses.  Those addresses must never reach a launch: if a refusal regressed, the call would go on to the
device, so these tests run only where no CUDA device is visible."""
import pytest

from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

pytestmark = cpu_only

EPI_BF16, EPI_F32, EPI_BIAS_GELU, EPI_RESID, EPI_GELU_BWD = 0, 1, 2, 3, 4
M, N, K = 417, 1000, 592


def _call(epi=EPI_BF16, out0=BASE, ld0=N, out1=None, ld1=0, bias=None, gamma=None, aux=None, ldaux=0):
    lib = _lib.load()
    return lib.ivb_gemm_bf16(BASE + 0x100000, 0, K, BASE + 0x200000, 0, K, M, N, K, epi, 0, out0, ld0, out1, ld1,
                             bias, gamma, aux, ldaux, None, 0, None)


@pytest.mark.parametrize("ld1", [N + 4, N + 2, 1001])
def test_gemm_out1_pitch_refused(ld1):
    expect_refusal(_call(EPI_BIAS_GELU, out1=BASE + 0x300000, ld1=ld1, bias=BASE + 0x400000),
                   "ivb_gemm_bf16: ld1 must be a multiple of 8 elements")
    expect_refusal(_call(EPI_RESID, out1=BASE + 0x300000, ld1=ld1, aux=BASE + 0x500000, ldaux=N),
                   "ivb_gemm_bf16: ld1 must be a multiple of 8 elements")


@pytest.mark.parametrize("epi,ldaux", [(EPI_GELU_BWD, N + 4), (EPI_GELU_BWD, N + 2), (EPI_RESID, N + 2),
                                       (EPI_RESID, N + 1)])
def test_gemm_aux_pitch_refused(epi, ldaux):
    """8 bf16 elements (GELU_BWD's h or saved gelu'), 4 fp32 elements (RESID's residual stream)."""
    out0 = BASE
    expect_refusal(_call(epi, out0=out0, aux=BASE + 0x500000, ldaux=ldaux),
                   "ivb_gemm_bf16: ldaux must be a multiple of 8 bf16 or 4 fp32 elements")


@pytest.mark.parametrize("slot", ["out0", "out1", "aux", "bias", "gamma"])
@pytest.mark.parametrize("offset", [2, 4, 8])
def test_gemm_epilogue_pointer_alignment_refused(slot, offset):
    ptrs = dict(out0=BASE, out1=BASE + 0x300000, aux=BASE + 0x500000, bias=BASE + 0x400000, gamma=BASE + 0x600000)
    ptrs[slot] += offset
    expect_refusal(_call(EPI_RESID, out0=ptrs["out0"], out1=ptrs["out1"], ld1=N, bias=ptrs["bias"], gamma=ptrs["gamma"],
                         aux=ptrs["aux"], ldaux=N),
                   f"ivb_gemm_bf16: {slot} must be 16-byte aligned")


def test_gemm_out1_and_aux_pitch_unchecked_when_absent():
    """ld1 / ldaux mean nothing without out1 / aux (lowlevel.gemm passes 0): only the alignment rule applies then."""
    expect_refusal(_call(EPI_BF16, ld1=3, ldaux=5, out0=BASE + 8), "ivb_gemm_bf16: out0 must be 16-byte aligned")


def test_gemm_fp32_aux_pitch_of_four_is_accepted_by_the_checks():
    """RESID's fp32 aux at a pitch of 4 (mod 8) passes the epilogue checks; the misaligned gamma after it is what is
    refused, so the call still never reaches the device."""
    expect_refusal(_call(EPI_RESID, aux=BASE + 0x500000, ldaux=N + 4, gamma=BASE + 0x600000 + 8),
                   "ivb_gemm_bf16: gamma must be 16-byte aligned")
