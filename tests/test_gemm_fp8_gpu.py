"""The FP8 GEMM (lowlevel.gemm_fp8) on the H100 (gpu), in two parts.

(a) Epilogues, with the accumulation taken out of the question: K <= 256 and operands whose dequantised values are
    small integers (|a|, |b| <= 4) times power-of-two scales, so every partial sum is an integer below 2^13 (times a
    power of two) and exact even in the tensor core's reduced-precision fp8 accumulator, and the dequantising multiply
    by a power of two is exact too.  Every epilogue and flag, both format pairs (E4M3 x E4M3, E5M2 x E4M3), every kernel
    form the FP8 path can select (ping-pong, the promoting cooperative kernel at tile_n 128 and 192, the default), with
    ragged M, N and K tails, element by element against tests/gemm_ref.py on the dequantised operands, with the bounds
    the bf16 epilogue tests use.
(b) Accumulation, at the eight step shapes of the cfg-2 block (M = 13 344 tokens: forward qkv / proj / fc1 / fc2,
    dgrad dh / dn2 / da / dn1) with Gaussian operands and the library's default kernel: the error the kernel adds must
    stay below the error the quantisation already carries,
        ||C_kernel - C64(deq)||_F <= 0.25 ||C64(deq) - C64(bf16)||_F,
    C64 the float64 product of the dequantised FP8 operands or of the original bf16 operands.  The measured ratios are
    in DESIGN.md 4.1 (FP8).
"""
import pytest
import torch

from gemm_ref import elem_errors, gemm_ref, worst
from internvideo_b200 import lowlevel as ll

pytestmark = pytest.mark.gpu

bf, f32 = torch.bfloat16, torch.float32
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
FL_1CTA, FL_PP = ll.FLAG_1CTA, ll.FLAG_PINGPONG
LIMIT_BF16, LIMIT_F32 = 1.9, 1.4     # the limits of the bf16 epilogue tests (test_gemm_epilogue_gpu.LIMITS)
KERNELS = [("pingpong", FL_PP, 0), ("coop128", FL_1CTA, 128), ("coop192", FL_1CTA, 192), ("default", 0, 0)]


def _operand(rows, K, pitch, seed, dtype, exp):
    """Integers v in [-4, 4]: (fp8 [rows, K] view of a [rows, pitch] buffer holding v * 2^exp, scale_inv 2^-exp, the
    dequantised operand v in fp32).  Every such value is exact in E4M3 and E5M2."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randint(-4, 5, (rows, pitch), generator=g, device="cuda").float()
    q = (v * 2.0 ** exp).to(dtype)[:, :K]
    return q, torch.tensor([2.0 ** -exp], device="cuda", dtype=f32), v[:, :K]


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(bf)


def _epilogues(M, N, seed):
    """(name, epilogue kwargs of gemm_fp8 / gemm_ref, out0's old values or None) for every epilogue and flag."""
    out = []
    for fl, nm in ((0, "bf16"), (ll.FLAG_ACCUM, "bf16+accum")):
        o = _mk((M, N), seed)
        out.append((nm, dict(epi=ll.EPI_BF16, flags=fl, bias=_mk((N,), seed + 1)), o))
    for fl, nm in ((0, "f32"), (ll.FLAG_ACCUM, "f32+accum")):
        o = _mk((M, N), seed + 2).float()
        out.append((nm, dict(epi=ll.EPI_F32, flags=fl), o))
    for tanh in (0, ll.FLAG_GELU_TANH):
        for save in (0, ll.FLAG_GELU_SAVE_GRAD):
            out.append((f"gelu tanh={tanh} save={save}",
                        dict(epi=ll.EPI_BIAS_GELU, flags=tanh | save, bias=_mk((N,), seed + 3),
                             out1=torch.empty((M, N), device="cuda", dtype=bf)), None))
    out.append(("gelu no out1", dict(epi=ll.EPI_BIAS_GELU, bias=_mk((N,), seed + 3)), None))
    g = torch.Generator(device="cuda").manual_seed(seed + 4)
    rs = (torch.rand((M,), generator=g, device="cuda") * 2).float()
    out.append(("resid", dict(epi=ll.EPI_RESID, bias=_mk((N,), seed + 5), gamma=_mk((N,), seed + 6, 0.1),
                              aux=torch.randn((M, N), device="cuda"), rowscale=rs,
                              out1=torch.empty((M, N), device="cuda", dtype=bf)), None))
    out.append(("resid plain", dict(epi=ll.EPI_RESID, aux=torch.randn((M, N), device="cuda")), None))
    h = _mk((M, N), seed + 7, 2.0)
    for fl in (0, ll.FLAG_GELU_TANH, ll.FLAG_GELU_SAVE_GRAD):
        out.append((f"gelu_bwd flags={fl}", dict(epi=ll.EPI_GELU_BWD, flags=fl, aux=h), None))
    return out


@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
@pytest.mark.parametrize("a_fmt", [E4, E5], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("M,N,K", [(333, 392, 200), (128, 200, 256), (517, 136, 40)])
def test_every_epilogue_exact_accumulation(cuda_lib, kernel, a_fmt, M, N, K):
    name, flag, tile_n = kernel
    pitch = (K + 15) // 16 * 16 + 16          # operand pitches wider than K, multiples of 16
    a8, sa, a = _operand(M, K, pitch, M + K, a_fmt, 3)
    b8, sb, b = _operand(N, K, pitch, N + K, E4, -2)
    for ename, kw, old in _epilogues(M, N, seed=M + N):
        kw = dict(kw)
        out_dtype = f32 if kw["epi"] in (ll.EPI_F32, ll.EPI_RESID) else bf
        out0 = old.clone() if old is not None else torch.full((M, N), float("nan"), device="cuda", dtype=out_dtype)
        flags = kw.pop("flags", 0)
        got = ll.gemm_fp8(a8, sa, b8, sb, out0=out0, flags=flags | flag, tile_n=tile_n, **kw)
        refs = gemm_ref(a, b, out0=old, flags=flags, **kw)
        outs = [(got, "out0")] + ([(kw["out1"], "out1")] if len(refs) > 1 else [])
        for (ref, scale), (t, slot) in zip(refs, outs):
            e, where = worst(elem_errors(t, ref, scale))
            lim = LIMIT_F32 if t.dtype == f32 else LIMIT_BF16
            assert e <= lim, (name, ename, slot, e, where)


STEP = [  # (name, N, K, A format): M = 13 344 tokens (B = 32 clips of 417)
    ("qkv", 4224, 1408, E4), ("proj", 1408, 1408, E4), ("fc1", 6144, 1408, E4), ("fc2", 1408, 6144, E4),
    ("dh", 6144, 1408, E5), ("dn2", 1408, 6144, E5), ("da", 1408, 1408, E5), ("dn1", 1408, 4224, E5),
]
M_STEP = 13344


def accumulation_ratio(N, K, a_fmt, flags=0, seed=0):
    """||C_kernel - C64(deq)||_F / ||C64(deq) - C64(bf16)||_F for Gaussian operands at [M_STEP, N, K]."""
    a = _mk((M_STEP, K), seed)
    b = _mk((N, K), seed + 1, 0.02)
    fa = ll.FP8_E5M2 if a_fmt == E5 else ll.FP8_E4M3
    qa, _, sa, _ = ll.fp8_quantize(a, fa)
    qb, _, sb, _ = ll.fp8_quantize(b, ll.FP8_E4M3)
    c = ll.gemm_fp8(qa, sa, qb, sb, epi=ll.EPI_F32, flags=flags)
    num = den = 0.0
    bd = (qb.double() * sb.double()).t()
    b64 = b.double().t()
    for r in range(0, M_STEP, 2048):
        rows = slice(r, min(r + 2048, M_STEP))
        c_deq = (qa[rows].double() * sa.double()) @ bd
        c_bf = a[rows].double() @ b64
        num += float(((c[rows].double() - c_deq) ** 2).sum())
        den += float(((c_deq - c_bf) ** 2).sum())
    return (num / den) ** 0.5


@pytest.mark.parametrize("name,N,K,a_fmt", STEP, ids=[s[0] for s in STEP])
def test_accumulation_error_at_step_shapes(cuda_lib, name, N, K, a_fmt):
    r = accumulation_ratio(N, K, a_fmt)
    assert r <= 0.25, (name, r)
