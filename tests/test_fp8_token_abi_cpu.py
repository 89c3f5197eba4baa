"""Per-token FP8 training without a GPU.

1. ivb_norm_fwd_fp8_train and ivb_fp8_quantize_cols_t refuse a call their kernels cannot serve before any CUDA call.
   They are called through the raw C ABI with fake device addresses, which must never reach a launch, so these checks
   run only where no CUDA device is visible.
2. The new kernels keep nothing in local memory.
3. modules.set_fp8 takes the scaling, and block_precision resolves it.
"""
import re

import pytest

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

M, D = 417, 1408
SA, SB, SC = BASE + 0x700000, BASE + 0x710000, BASE + 0x720000    # fake per-row / per-column vectors


def _norm(x=BASE, x_f32=1, ldx=D, w=BASE + 0x100000, b=None, ln=1, m=M, d=D, out=BASE + 0x300000, ldo=D, sinv=SA,
          y=BASE + 0x400000, ldy=D, mean=SB, rstd=SC):
    return _lib.load().ivb_norm_fwd_fp8_train(x, x_f32, ldx, w, b, 1e-5, ln, m, d, out, ldo, sinv, y, ldy, mean, rstd,
                                              None)


def _cols(x=BASE, ldx=1416, m=600, k=1410, out_t=BASE + 0x300000, ldt=608, amax=SA, sinv=SB):
    return _lib.load().ivb_fp8_quantize_cols_t(x, ldx, m, k, out_t, ldt, amax, sinv, None)


@cpu_only
def test_norm_fwd_fp8_train_refusals():
    P = "ivb_norm_fwd_fp8_train: "
    expect_refusal(_norm(m=0), P + "empty tensor")
    for d in (0, 1404, 4104):
        expect_refusal(_norm(d=d, ldx=4104, ldo=4112, ldy=4104),
                       P + "D must be a multiple of 8 in [8, IVB_NORM_FP8_MAX_D]")
    expect_refusal(_norm(ldx=1412), P + "ldx must be a multiple of 8 elements and >= D")
    expect_refusal(_norm(ldx=1400), P + "ldx must be a multiple of 8 elements and >= D")
    expect_refusal(_norm(ldo=1416), P + "ldo must be a multiple of 16 elements and >= D")
    expect_refusal(_norm(ldo=1392), P + "ldo must be a multiple of 16 elements and >= D")
    expect_refusal(_norm(ldy=1412), P + "ldy must be a multiple of 8 elements and >= D")
    expect_refusal(_norm(ldy=1400), P + "ldy must be a multiple of 8 elements and >= D")
    null = P + "x, weight, out, row_scale_inv, y, rstd or (LayerNorm) mean is null"
    for kw in (dict(x=None), dict(w=None), dict(out=None), dict(sinv=None), dict(y=None), dict(rstd=None),
               dict(mean=None)):
        expect_refusal(_norm(**kw), null)
    for kw in (dict(x=BASE + 8), dict(w=BASE + 0x100008), dict(b=BASE + 0x200008), dict(out=BASE + 0x300008),
               dict(y=BASE + 0x400008)):
        expect_refusal(_norm(**kw), P + "x, weight, bias, out and y must be 16-byte aligned")
    for kw in (dict(sinv=SA + 2), dict(mean=SB + 2), dict(rstd=SC + 2)):
        expect_refusal(_norm(**kw), P + "row_scale_inv, mean and rstd must be 4-byte aligned")


@cpu_only
def test_quantize_cols_t_refusals():
    P = "ivb_fp8_quantize_cols_t: "
    expect_refusal(_cols(m=0), P + "empty tensor")
    expect_refusal(_cols(k=0), P + "empty tensor")
    for kw in (dict(x=None), dict(out_t=None), dict(amax=None), dict(sinv=None)):
        expect_refusal(_cols(**kw), P + "x, out_t, col_amax or col_scale_inv is null")
    expect_refusal(_cols(ldx=1412), P + "ldx must be a multiple of 8 elements and >= K")
    expect_refusal(_cols(ldx=1408), P + "ldx must be a multiple of 8 elements and >= K")
    expect_refusal(_cols(ldt=600), P + "ldt must be a multiple of 16 elements and >= M")
    expect_refusal(_cols(ldt=592), P + "ldt must be a multiple of 16 elements and >= M")
    expect_refusal(_cols(x=BASE + 8), P + "x and out_t must be 16-byte aligned")
    expect_refusal(_cols(out_t=BASE + 0x300008), P + "x and out_t must be 16-byte aligned")
    expect_refusal(_cols(amax=SA + 2), P + "col_amax and col_scale_inv must be 4-byte aligned")
    expect_refusal(_cols(sinv=SB + 2), P + "col_amax and col_scale_inv must be 4-byte aligned")


# norm_rows_kernel: the bf16 RMSNorm (6), the q/k pair (3), the E4M3 (16) and the E4M3 + bf16 training (16) forms
@pytest.mark.parametrize("obj, pattern, count", [("ivb_norm.o", "norm_rows_kernel", 41),
                                                 ("ivb_fp8.o", "fp8_c(ol_amax|ast_cols)_kernel", 2),
                                                 ("ivb_fp8.o", "fp8_(amax|cast|col_amax|cast_cols|rows|blocks_t)_kernel",
                                                  10)])
def test_new_kernels_keep_nothing_in_local_memory(obj, pattern, count):
    found = {k: v for k, v in sass.functions(obj).items() if re.search(pattern, k)}
    assert len(found) == count, sorted(found)
    for name, lines in found.items():
        assert not any(re.search(r"\b(LDL|STL)\b", l) for l in lines), name


def test_set_fp8_scaling_resolves_to_block_precision():
    from internvideo_b200 import ops
    from internvideo_b200.modules import Block, block_precision, set_fp8
    blk = Block(64, 2, 4.0, init_values=0.1, qk_normalization=True)
    assert block_precision(blk, True) == ops.BF16
    assert set_fp8(blk, True, scaling="token") == 1
    assert block_precision(blk, True) == ops.FP8_TOKEN and block_precision(blk, False) == ops.FP8_TOKEN
    assert set_fp8(blk) == 1
    assert block_precision(blk, True) == ops.FP8_TENSOR and block_precision(blk, False) == ops.FP8_TENSOR
    set_fp8(blk, True, scaling="token")
    assert set_fp8(blk, False) == 1
    assert block_precision(blk, True) == ops.BF16
    with pytest.raises(ValueError, match="scaling"):
        set_fp8(blk, True, scaling="row")
