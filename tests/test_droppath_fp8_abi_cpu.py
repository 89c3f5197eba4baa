"""DropPath skipping in per-token FP8 and in attention, without a GPU: the prototypes of ivb_gemm_fp8_plan,
ivb_attn_fwd_plan and ivb_attn_bwd_plan extend the plain calls by one pointer, the bindings take the plan, each entry
point refuses a call it cannot run before any CUDA call, and the new kernels keep their accumulators in registers."""
import ctypes as C
import inspect
import re

import pytest
import torch

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll

P = _lib.PROTOTYPES

EPI_BF16, EPI_RESID = 0, 3
FLAG_ACCUM, FLAG_1CTA, FLAG_2CTA, FLAG_PINGPONG, FLAG_VEC = 2, 4, 8, 32, 64


@pytest.mark.parametrize("plain, planned", [("ivb_gemm_fp8", "ivb_gemm_fp8_plan"), ("ivb_attn_fwd", "ivb_attn_fwd_plan"),
                                            ("ivb_attn_bwd", "ivb_attn_bwd_plan")])
def test_plan_prototypes_extend_the_plain_call(plain, planned):
    """The planned call is the plain one with one pointer (the plan or the factors) before the stream."""
    (r0, a0), (r1, a1) = P[plain], P[planned]
    assert r0 == r1
    assert a1 == a0[:-1] + [C.c_void_p, a0[-1]]


def test_ivb_gemm_fp8_keeps_its_prototype():
    assert len(P["ivb_gemm_fp8"][1]) == 25


def test_bindings_take_the_plan():
    assert "m_plan" in inspect.signature(ll._gemm_fp8_plan).parameters
    assert "m_plan" not in inspect.signature(ll.gemm_fp8).parameters
    assert "rowscale" in inspect.signature(ll.attn_fwd).parameters
    assert "rowscale" in inspect.signature(ll.attn_bwd).parameters


# ---- refusals through the raw C ABI with fake device addresses (never reach a launch)
def _fp8(flags=FLAG_VEC, fmt=0, lda=1024, ldb=1024, ld0=512, tile_n=0, m_plan=BASE + 0x300000, epi=EPI_BF16, aux=None,
         a_s=BASE + 0x500000, b_s=BASE + 0x510000):
    M, N, K = 1024, 512, 1024
    return _lib.load().ivb_gemm_fp8_plan(BASE + 0x100000, 0, lda, fmt, a_s, BASE + 0x200000, 0, ldb, b_s, M, N, K, epi,
                                         flags, BASE, ld0, None, 0, None, None, aux, N if aux else 0, None, tile_n,
                                         m_plan, None)


@cpu_only
@pytest.mark.parametrize("kw, text", [
    (dict(flags=FLAG_VEC | FLAG_2CTA), "ivb_gemm_fp8_plan: no CTA-pair kernel"),
    (dict(flags=FLAG_VEC | FLAG_2CTA, m_plan=None), "ivb_gemm_fp8_plan: no CTA-pair kernel"),
    (dict(flags=0), "ivb_gemm_fp8_plan: a DropPath plan needs IVB_FLAG_FP8_VECTOR_SCALES"),
    (dict(flags=FLAG_VEC | FLAG_ACCUM), "ivb_gemm_fp8_plan: an M plan excludes IVB_FLAG_ACCUM"),
    (dict(tile_n=192), "ivb_gemm_fp8_plan: a DropPath plan runs the FP8 GEMM at tile_n 128"),
    (dict(flags=FLAG_VEC | FLAG_1CTA | FLAG_PINGPONG), "ivb_gemm_fp8_plan: IVB_FLAG_1CTA and IVB_FLAG_PINGPONG exclude"),
    (dict(lda=1000), "ivb_gemm_fp8_plan: lda and ldb must be multiples of 16 elements"),
    (dict(ldb=1032), "ivb_gemm_fp8_plan: lda and ldb must be multiples of 16 elements"),
    (dict(ld0=516), "ivb_gemm_fp8_plan: N and ld0 must be multiples of 8 elements"),
    (dict(fmt=1), "ivb_gemm_fp8_plan: vector scales need an E4M3 A operand"),
    (dict(a_s=None), "ivb_gemm_fp8_plan: scale_inv pointers are null"),
    (dict(a_s=BASE + 0x500004), "ivb_gemm_fp8_plan: scale vectors must be 8-byte aligned"),
    (dict(epi=EPI_RESID), "ivb_gemm_fp8_plan: epilogue needs aux"),
])
def test_gemm_fp8_plan_refuses(kw, text):
    expect_refusal(_fp8(**kw), text)


D16 = 16 * 88
LD_BWD = (3 * D16,) * 3 + (D16,) * 2 + (3 * D16,) * 3


def _attn_fwd(rs=BASE + 0x900000, d=88, ld=(3 * D16, 3 * D16, 3 * D16, D16)):
    return _lib.load().ivb_attn_fwd_plan(None, ld[0], None, ld[1], None, ld[2], None, ld[3], None, 2, 417, 16, d, 0.1,
                                         rs, None)


def _attn_bwd(rs=BASE + 0x900000, d=88, ld=LD_BWD, ws=1024):
    return _lib.load().ivb_attn_bwd_plan(None, ld[0], None, ld[1], None, ld[2], None, ld[3], None, ld[4], 1, ws, None,
                                         ld[5], None, ld[6], None, ld[7], 2, 417, 16, d, 0.1, rs, None)


def test_attn_plan_needs_the_factors():
    expect_refusal(_attn_fwd(rs=None), "ivb_attn_fwd_plan: rowscale is null")
    expect_refusal(_attn_bwd(rs=None), "ivb_attn_bwd_plan: rowscale is null")


@pytest.mark.parametrize("slot", range(8))
def test_attn_plan_pitch_refused(slot):
    ld = list(LD_BWD)
    ld[slot] += 4
    expect_refusal(_attn_bwd(ld=ld), "ivb_attn_bwd_plan: pitches must be multiples of 8")
    if slot < 4:
        expect_refusal(_attn_fwd(ld=ld[:4]), "ivb_attn_fwd_plan: pitches must be multiples of 8")


def test_attn_plan_head_dim_and_workspace_refused():
    expect_refusal(_attn_fwd(d=136), "ivb_attn_fwd_plan: head_dim must be a multiple of 8 in [16,128]")
    expect_refusal(_attn_bwd(d=12), "ivb_attn_bwd_plan: head_dim must be a multiple of 8 in [16,128]")
    expect_refusal(_attn_bwd(ws=1032), "ivb_attn_bwd_plan: workspace must be 16-byte aligned")


def test_bindings_refuse_a_bad_rowscale():
    """The attention plan reads rowscale[b n] for every clip: the binding wants a contiguous [B*n] vector (checked
    before any device call, with meta tensors standing in for CUDA ones)."""
    with pytest.raises(_lib.IvbError):
        ll._chk_rowscale("attn_fwd", torch.empty((2, 417), device="meta"), 2 * 417)
    with pytest.raises(_lib.IvbError):
        ll._chk_rowscale("attn_bwd", torch.empty((2 * 417 * 2,), device="meta")[::2], 2 * 417)
    ll._chk_rowscale("attn_fwd", torch.empty((2 * 417,), device="meta"), 2 * 417)


# ---- the new kernels, from the objects build.py compiled
def test_planned_kernels_do_not_spill():
    """Every GEMM instantiation with the plan code (bf16 single-CTA, OpPlannedFp8) and every attention plan kernel:
    168 registers (384 threads, one CTA per SM), no stack and no local memory."""
    res = {**sass.resources("ivb_gemm.o"), **sass.resources("ivb_attn.o"), **sass.resources("ivb_attn_bwd.o")}
    planned = {k: v for k, v in res.items() if "OpPlannedFp8" in k or re.search(r"attn_\w+_plan_kernelI", k)
               or ("OpBf16" in k and ("pingpong" in k or "Li1EEEv" in k))}
    assert sum("OpPlannedFp8" in k for k in planned) == 2, sorted(planned)          # ping-pong, cooperative at BN 128
    assert sum("attn_fwd_plan_kernel" in k for k in planned) == 8
    assert sum("attn_bwd_plan_kernel" in k for k in planned) == 16
    for k, v in planned.items():
        assert v == (168, 0, 0), k


@pytest.mark.parametrize("obj, plain, planned", [("ivb_attn.o", "15attn_fwd_kernelI", "20attn_fwd_plan_kernelI"),
                                                 ("ivb_attn_bwd.o", "15attn_bwd_kernelI", "20attn_bwd_plan_kernelI")])
def test_attn_plan_kernels_keep_the_mma_pipeline(obj, plain, planned):
    """A plan kernel runs its live CTAs as the plain kernel of the same head dim: the same wgmmas, the same waits on
    them (WARPGROUP.DEPBAR), no local memory; the dead CTA's exit only adds instructions in front."""
    k = sass.functions(obj)
    plans = {n: v for n, v in k.items() if planned in n}
    assert len(plans) == len([n for n in k if plain in n]) > 0
    for n, lines in plans.items():
        twin = k[n.replace(planned, plain).replace("EPKf", "E")]
        for pat in (r"HGMMA", r"WARPGROUP\.DEPBAR", r"\b(LDL|STL)\b"):
            assert sum(bool(re.search(pat, l)) for l in lines) == sum(bool(re.search(pat, l)) for l in twin), (n, pat)
