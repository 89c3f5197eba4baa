"""FP8 weight gradients (modules.set_fp8(..., scaling="token", wgrad=True)) without a GPU.

1. ivb_fp8_quantize_blocks_t(_plan) and ivb_gemm_fp8_wgrad refuse a call their kernels cannot serve before any CUDA
   call.  They are called through the raw C ABI with fake device addresses, which must never reach a launch, so these
   checks run only where no CUDA device is visible.
2. The binding's prototypes of the three entry points are the header's.
3. The new kernels keep nothing in local memory and use no stack.
4. set_fp8's wgrad switch resolves to ops.FP8_TOKEN_WGRAD, and is refused with per-tensor scaling.
"""
import ctypes as C
import re

import pytest
import torch

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

SA, SB, PLAN = BASE + 0x700000, BASE + 0x710000, BASE + 0x720000


def _cast(x=BASE, ldx=1416, m=1251, c=1408, out_t=BASE + 0x300000, ldt=1264, sinv=SA, rs=None, plan=False):
    lib = _lib.load()
    if plan:
        return lib.ivb_fp8_quantize_blocks_t_plan(x, ldx, m, c, out_t, ldt, sinv, rs, None)
    return lib.ivb_fp8_quantize_blocks_t(x, ldx, m, c, out_t, ldt, sinv, None)


def _wgrad(a=BASE, lda=1264, sa=SA, b=BASE + 0x100000, ldb=1264, sb=SB, m=1408, n=4224, k=1251, epi=0, flags=0,
           out0=BASE + 0x300000, ld0=4224, k_plan=PLAN):
    return _lib.load().ivb_gemm_fp8_wgrad(a, lda, sa, b, ldb, sb, m, n, k, epi, flags, out0, ld0, k_plan, None)


@cpu_only
@pytest.mark.parametrize("plan", [False, True], ids=["plain", "plan"])
def test_quantize_blocks_t_refusals(plan):
    P = ("ivb_fp8_quantize_blocks_t_plan: " if plan else "ivb_fp8_quantize_blocks_t: ")
    kw0 = dict(plan=plan, rs=SB if plan else None)
    expect_refusal(_cast(m=0, **kw0), P + "empty tensor")
    expect_refusal(_cast(c=0, **kw0), P + "empty tensor")
    expect_refusal(_cast(c=1404, **kw0), P + "C must be a multiple of 8")
    for kw in (dict(x=None), dict(out_t=None), dict(sinv=None)):
        expect_refusal(_cast(**kw, **kw0), P + "x, out_t or scale_inv is null")
    expect_refusal(_cast(ldx=1412, **kw0), P + "ldx must be a multiple of 8 elements and >= C")
    expect_refusal(_cast(ldx=1400, **kw0), P + "ldx must be a multiple of 8 elements and >= C")
    expect_refusal(_cast(ldt=1256, **kw0), P + "ldt must be a multiple of 16 elements and >= M")
    expect_refusal(_cast(ldt=1240, **kw0), P + "ldt must be a multiple of 16 elements and >= M")
    expect_refusal(_cast(x=BASE + 8, **kw0), P + "x and out_t must be 16-byte aligned")
    expect_refusal(_cast(out_t=BASE + 0x300008, **kw0), P + "x and out_t must be 16-byte aligned")
    expect_refusal(_cast(sinv=SA + 2, **kw0), P + "scale_inv and rowscale must be 4-byte aligned")
    if plan:
        expect_refusal(_cast(plan=True, rs=SB + 2), P + "scale_inv and rowscale must be 4-byte aligned")
        expect_refusal(_cast(plan=True, rs=None), P + "rowscale is null")


@cpu_only
def test_gemm_fp8_wgrad_refusals():
    P = "ivb_gemm_fp8_wgrad: "
    for kw in (dict(m=0), dict(n=0), dict(k=0)):
        expect_refusal(_wgrad(**kw), P + "empty problem")
    for kw in (dict(a=None), dict(b=None)):
        expect_refusal(_wgrad(**kw), P + "A_t or B_t is null")
    for kw in (dict(lda=1256), dict(ldb=1256), dict(lda=1240), dict(ldb=1272)):
        expect_refusal(_wgrad(**kw), P + "lda and ldb must be multiples of 16 elements and >= K")
    for kw in (dict(m=1404), dict(n=4220, ld0=4224)):
        expect_refusal(_wgrad(**kw), P + "M and N must be multiples of 8")
    for kw in (dict(ld0=4228), dict(ld0=4216)):
        expect_refusal(_wgrad(**kw), P + "ld0 must be a multiple of 8 elements and >= N")
    for kw in (dict(sa=None), dict(sb=None)):
        expect_refusal(_wgrad(**kw), P + "scale_inv pointers are null")
    for kw in (dict(sa=SA + 8), dict(sb=SB + 4)):
        expect_refusal(_wgrad(**kw), P + "scale vectors must be 16-byte aligned")
    for epi in (2, 3, 4, 7):
        expect_refusal(_wgrad(epi=epi), P + "epilogue must be IVB_EPI_BF16 or IVB_EPI_F32")
    # ping-pong, CTA pair, forced cooperative, GELU flags, vector scales: one kernel form, and no other epilogue input
    for flags in (32, 8, 4, 1, 16, 64, 2 | 32):
        expect_refusal(_wgrad(flags=flags), P + "the only flag is IVB_FLAG_ACCUM")
    expect_refusal(_wgrad(out0=None), P + "out0 is null")
    expect_refusal(_wgrad(out0=BASE + 0x300008), P + "out0 must be 16-byte aligned")


def test_prototypes_match_the_header():
    text = _lib.HEADER.read_text()
    P = _lib.parse_prototypes(text)
    V, I, L = C.c_void_p, C.c_int, C.c_long
    assert P["ivb_fp8_quantize_blocks_t"] == (C.c_int, [V, L, I, I, V, L, V, V])
    assert P["ivb_fp8_quantize_blocks_t_plan"] == (C.c_int, [V, L, I, I, V, L, V, V, V])
    assert P["ivb_gemm_fp8_wgrad"] == (C.c_int, [V, L, V, V, L, V, I, I, I, I, I, V, L, V, V])
    lib = _lib.load()
    for name in ("ivb_fp8_quantize_blocks_t", "ivb_fp8_quantize_blocks_t_plan", "ivb_gemm_fp8_wgrad"):
        fn = getattr(lib, name)
        assert (fn.restype, fn.argtypes) == (P[name][0], P[name][1]), name
    # the pinned FP8 GEMM signature is untouched
    assert len(P["ivb_gemm_fp8"][1]) == 25


@pytest.mark.parametrize("obj, pattern", [("ivb_fp8.o", r"fp8_blocks_t_kernel"), ("ivb_gemm.o", r"OpBlockFp8")])
def test_new_kernels_use_no_local_memory_and_no_stack(obj, pattern):
    found = {k: v for k, v in sass.resources(obj).items() if re.search(pattern, k)}
    assert len(found) == 1, sorted(found)
    for name, (regs, stack, local) in found.items():
        assert stack == 0 and local == 0, (name, regs, stack, local)
        if obj == "ivb_gemm.o":
            assert regs == 168, (name, regs)      # 384 threads, one CTA per SM


def test_block_fp8_gemm_issues_e4m3_qgmma_and_no_local_memory():
    (name, lines), = [(k, v) for k, v in sass.functions("ivb_gemm.o").items() if "OpBlockFp8" in k]
    q = [l for l in lines if re.search(r"\bQGMMA\.", l)]
    assert q and all(re.search(r"QGMMA\.64x128x32\.F32\.E4M3\.E4M3\b", l) for l in q), name
    assert not any(re.search(r"\b(LDL|STL|HGMMA)\b", l) for l in lines), name


def test_set_fp8_wgrad_resolves_to_block_precision():
    from internvideo_b200 import ops
    from internvideo_b200.modules import Block, block_precision, set_fp8
    blk = Block(64, 2, 4.0, init_values=0.1, qk_normalization=True)
    assert block_precision(blk, True) == ops.BF16
    assert set_fp8(blk, True, scaling="token", wgrad=True) == 1
    assert blk.fp8_wgrad and block_precision(blk, True) == ops.FP8_TOKEN_WGRAD
    assert set_fp8(blk, True, scaling="token") == 1              # the default switches it off again
    assert block_precision(blk, True) == ops.FP8_TOKEN
    set_fp8(blk, True, scaling="token", wgrad=True)
    assert set_fp8(blk, False) == 1 and block_precision(blk, True) == ops.BF16
    for scaling in ("tensor",):
        with pytest.raises(ValueError, match="wgrad=True needs scaling='token'"):
            set_fp8(blk, True, scaling=scaling, wgrad=True)
    with pytest.raises(ValueError, match="wgrad=True needs scaling='token'"):
        set_fp8(blk, True, wgrad=True)
    assert block_precision(blk, True) == ops.BF16                # a refused call changes nothing
    set_fp8(blk, True, scaling="tensor")
    assert block_precision(blk, True) == ops.FP8_TENSOR


def test_branch_plans_of_the_new_precision():
    """FP8 weight gradients take the M plan (128-row tiles) as their K plan; the other precisions keep theirs."""
    from internvideo_b200 import ops
    M = 1251
    nm, nk = (M + 127) // 128, (M + 63) // 64
    plan = torch.arange(nm + 1 + nk + 1, dtype=torch.int32)
    m_plan, k_plan = ops._branch_plans(plan, M, ops.FP8_TOKEN_WGRAD)
    assert torch.equal(m_plan, plan[:nm + 1]) and torch.equal(k_plan, plan[:nm + 1])
    m_plan, k_plan = ops._branch_plans(plan, M, ops.FP8_TOKEN)
    assert torch.equal(m_plan, plan[:nm + 1]) and torch.equal(k_plan, plan[nm + 1:])
    assert ops._branch_plans(plan, M, ops.FP8_TENSOR) == (None, None)
    assert ops._branch_plans(None, M, ops.FP8_TOKEN_WGRAD) == (None, None)
