"""ivb_gemm_bf16 and ivb_gemm_fp8 refuse IVB_FLAG_GELU_TANH together with IVB_FLAG_GELU_QUICK (two GELU forms at
once) before any CUDA call; checked through the raw C ABI with fake device addresses (tests/abi_fake.py), so these
tests run only where no CUDA device is visible."""
import pytest

from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll

pytestmark = cpu_only

M, N, K = 417, 1024, 592


def _bf16(epi, flags, aux=None):
    return _lib.load().ivb_gemm_bf16(BASE + 0x100000, 0, K, BASE + 0x200000, 0, K, M, N, K, epi, flags, BASE, N,
                                     BASE + 0x300000 if epi == ll.EPI_BIAS_GELU else None, N,
                                     BASE + 0x400000 if epi == ll.EPI_BIAS_GELU else None, None, aux,
                                     N if aux else 0, None, 0, None)


def _fp8(epi, flags, aux=None):
    return _lib.load().ivb_gemm_fp8(BASE + 0x100000, 0, K, ll.FP8_E4M3, BASE + 0x600000, BASE + 0x200000, 0, K,
                                    BASE + 0x700000, M, N, K, epi, flags, BASE, N,
                                    BASE + 0x300000 if epi == ll.EPI_BIAS_GELU else None, N,
                                    BASE + 0x400000 if epi == ll.EPI_BIAS_GELU else None, None, aux,
                                    N if aux else 0, None, 0, None)


@pytest.mark.parametrize("save", [0, ll.FLAG_GELU_SAVE_GRAD], ids=["h", "save"])
@pytest.mark.parametrize("epi", [ll.EPI_BIAS_GELU, ll.EPI_GELU_BWD], ids=["bias_gelu", "gelu_bwd"])
def test_tanh_with_quick_refused(epi, save):
    flags = ll.FLAG_GELU_TANH | ll.FLAG_GELU_QUICK | save
    aux = BASE + 0x500000 if epi == ll.EPI_GELU_BWD else None
    expect_refusal(_bf16(epi, flags, aux), "ivb_gemm_bf16: IVB_FLAG_GELU_TANH and IVB_FLAG_GELU_QUICK exclude each other")
    expect_refusal(_fp8(epi, flags, aux), "IVB_FLAG_GELU_TANH and IVB_FLAG_GELU_QUICK exclude each other")


def test_flag_value():
    """IVB_FLAG_GELU_QUICK takes the bit after IVB_FLAG_FP8_VECTOR_SCALES (64)."""
    assert ll.FLAG_GELU_QUICK == 128 and ll.FLAG_FP8_VECTOR_SCALES == 64
