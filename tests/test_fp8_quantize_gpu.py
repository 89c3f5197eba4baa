"""ivb_fp8_quantize (lowlevel.fp8_quantize) against torch (gpu).

amax is exact, the scale is the power of two 2^floor(log2(fmax / amax)), the cast is bit-exact against torch's
round-to-nearest-even conversion at that scale, the transposed output is the row-major output transposed bit for bit,
and two runs give the same bits.  Ragged shapes (M and K not multiples of 64 or 128), pitches wider than K, an all-zero
tensor (scale 1) and non-finite input (scale_inv NaN) are covered.
"""
import math

import pytest
import torch

from internvideo_b200 import lowlevel as ll

pytestmark = pytest.mark.gpu

FMAX = {ll.FP8_E4M3: 448.0, ll.FP8_E5M2: 57344.0}
FORMATS = [ll.FP8_E4M3, ll.FP8_E5M2]


def _x(M, K, pitch, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = (torch.randn((M, pitch), generator=g, device="cuda") * scale).to(torch.bfloat16)
    return buf[:, :K]


def _expected_scale(amax, fmt):
    if amax == 0.0:
        return 1.0
    return 2.0 ** min(126, max(-126, math.floor(math.log2(FMAX[fmt] / amax))))


def _u8(t):
    return t.view(torch.uint8)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("M,K,pitch,scale", [(333, 200, 216, 1.0), (64, 128, 128, 3e-3), (1000, 1408, 1416, 40.0),
                                             (17, 24, 40, 1e4), (130, 72, 72, 1e-6)])
def test_cast_is_bit_exact_against_torch(cuda_lib, fmt, M, K, pitch, scale):
    x = _x(M, K, pitch, seed=M + K, scale=scale)
    q, q_t, sinv, amax = ll.fp8_quantize(x, fmt, transpose=True)
    ref_amax = x.float().abs().max().item()
    assert amax.item() == ref_amax
    s = _expected_scale(ref_amax, fmt)
    assert sinv.item() == 1.0 / s
    assert ref_amax * s <= FMAX[fmt] < 2 * ref_amax * s
    ref = (x.float() * s).to(ll.FP8_DTYPES[fmt])
    assert torch.equal(_u8(q), _u8(ref))
    assert torch.equal(_u8(q_t), _u8(q).t())
    assert q.stride(0) % 16 == 0 and q_t.stride(0) % 16 == 0


@pytest.mark.parametrize("fmt", FORMATS)
def test_all_zero_tensor_has_scale_one(cuda_lib, fmt):
    x = torch.zeros((100, 56), device="cuda", dtype=torch.bfloat16)
    q, q_t, sinv, amax = ll.fp8_quantize(x, fmt, transpose=True)
    assert amax.item() == 0.0 and sinv.item() == 1.0
    assert int(_u8(q).max()) == 0 and int(_u8(q_t).max()) == 0


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_non_finite_input_gives_nan_scale_inv(cuda_lib, fmt, bad):
    x = _x(200, 136, 136, seed=5)
    x[123, 77] = bad
    _, _, sinv, amax = ll.fp8_quantize(x, fmt)
    assert not math.isfinite(amax.item())
    assert math.isnan(sinv.item())


@pytest.mark.parametrize("fmt", FORMATS)
def test_two_runs_give_the_same_bits(cuda_lib, fmt):
    x = _x(13344 // 4, 1408, 1408, seed=9)
    a = ll.fp8_quantize(x, fmt, transpose=True)
    b = ll.fp8_quantize(x, fmt, transpose=True)
    assert torch.equal(_u8(a[0]), _u8(b[0])) and torch.equal(_u8(a[1]), _u8(b[1]))
    assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])
