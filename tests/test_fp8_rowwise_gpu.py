"""Per-row FP8 kernels on the H100 (gpu): lowlevel.fp8_quantize_rows, lowlevel.norm_fwd_fp8 and lowlevel.gemm_fp8 with
per-row / per-column scale vectors (the FP8 inference path of the frozen towers).

- The row cast is bit-exact against torch with each row's scale recomputed on the host from the row's amax, and its
  dequantisation is never further from x than the per-tensor cast's, element by element (a row's power-of-two grid
  refines the tensor's).
- The fused norm -> E4M3 rows is within the E4M3 rounding of the fp64 norm (u = 2^-4 relative, plus half the subnormal
  spacing 2^-10 * scale_inv, times 1 + 2^-10 for the fp32 row statistics), and differs from norm_fwd's bf16 output cast
  row by row only where the bf16 rounding moved an element onto or across an E4M3 rounding boundary.
- The vector-scale GEMM: bit-identical to the scalar-scale GEMM for constant vectors; the teachers' epilogues element by
  element against tests/gemm_ref.py with exact accumulation on both kernel forms; the accumulation-error ratio of
  tests/test_gemm_fp8_gpu.py (0.25) at the teachers' eight forward shapes.
- Every new kernel gives the same bits on two runs.
"""
import pytest
import torch

from gemm_ref import elem_errors, gemm_ref, worst
from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll

pytestmark = pytest.mark.gpu

bf, f32, E4 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
LIMIT_BF16, LIMIT_F32 = 1.9, 1.4     # the limits of the bf16 epilogue tests (test_gemm_epilogue_gpu.LIMITS)
KERNELS = [("pingpong", ll.FLAG_PINGPONG, 0), ("coop128", ll.FLAG_1CTA, 128), ("coop192", ll.FLAG_1CTA, 192),
           ("default", 0, 0)]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def host_scale(amax):
    """fp8_scale on the host: the largest power of two 2^e with amax * 2^e <= 448, e in [-126, 126]; 1 for amax = 0."""
    a = amax.double()
    e = torch.floor(torch.log2(448.0 / a.clamp_min(1e-300)))
    e = torch.where(a * torch.exp2(e + 1) <= 448.0, e + 1, e)
    e = torch.where(a * torch.exp2(e) > 448.0, e - 1, e)
    e = e.clamp(-126, 126)
    return torch.where(a == 0, torch.ones_like(a), torch.exp2(e)).float()


def _rows_input(M, K, pitch, seed):
    """bf16 [M, K] view of a [M, pitch] buffer: Gaussian rows times 2^[-20, 20], a zero row, a row of tiny values and
    rows mixing magnitudes 2^-12 .. 2^12."""
    g = _gen(seed)
    x = torch.randn((M, pitch), generator=g, device="cuda")
    x *= torch.exp2(torch.randint(-20, 21, (M, 1), generator=g, device="cuda").float())
    x[0] = 0
    x[1] *= 2.0 ** -100
    x[2:6] *= torch.exp2(torch.randint(-12, 13, (4, pitch), generator=g, device="cuda").float())
    return x.to(bf)[:, :K]


@pytest.mark.parametrize("M,K,pitch", [(64, 128, 128), (300, 1408, 1416), (77, 593, 600), (130, 3200, 3208),
                                       (33, 12800, 12800), (9, 5, 8)])
def test_quantize_rows_bit_exact(cuda_lib, M, K, pitch):
    x = _rows_input(M, K, pitch, M + K)
    q, sinv = ll.fp8_quantize_rows(x)
    scale = host_scale(x.float().abs().amax(1))
    ref = (x.float() * scale[:, None]).to(E4)
    assert torch.equal(q.view(torch.uint8), ref.view(torch.uint8))
    assert torch.equal(sinv, 1.0 / scale)
    q2, s2 = ll.fp8_quantize_rows(x)
    assert torch.equal(q.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(sinv, s2)


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_quantize_rows_non_finite_row(cuda_lib, bad):
    x = _rows_input(40, 600, 600, 7).contiguous()
    x[5, 17] = bad
    q, sinv = ll.fp8_quantize_rows(x)
    assert torch.isnan(sinv[5]) and torch.isfinite(torch.cat([sinv[:5], sinv[6:]])).all()
    ok = torch.ones(40, dtype=torch.bool, device="cuda"); ok[5] = False
    scale = host_scale(x[ok].float().abs().amax(1))
    assert torch.equal(q[ok].view(torch.uint8), (x[ok].float() * scale[:, None]).to(E4).view(torch.uint8))


@pytest.mark.parametrize("M,K", [(500, 1408), (257, 3200), (64, 12800)])
def test_row_cast_refines_tensor_cast(cuda_lib, M, K):
    x = _rows_input(M, K, K, 3 * M + K)
    x[1] = 0.0          # keep the tensor's amax within reach of every row (a 2^-100 row would flush to zero)
    q, sinv = ll.fp8_quantize_rows(x)
    qt, _, st, _ = ll.fp8_quantize(x, ll.FP8_E4M3)
    xd = x.double()
    err_row = (q.double() * sinv.double()[:, None] - xd).abs()
    err_tensor = (qt.double() * st.double() - xd).abs()
    assert bool((err_row <= err_tensor).all())
    assert float(err_row.sum()) < float(err_tensor.sum())


def _norm64(x, w, b, eps, layernorm):
    xd = x.double()
    if layernorm:
        xd = xd - xd.mean(1, keepdim=True)
    y = xd * torch.rsqrt((xd * xd).mean(1, keepdim=True) + eps) * w.double()
    return y + b.double() if b is not None else y


@pytest.mark.parametrize("D", [384, 1408, 3200])
@pytest.mark.parametrize("layernorm", [False, True], ids=["rms", "ln"])
@pytest.mark.parametrize("xdt", [f32, bf], ids=["x32", "x16"])
def test_norm_fwd_fp8_within_e4m3_rounding(cuda_lib, D, layernorm, xdt):
    M = 777
    g = _gen(D + 2 * layernorm)
    x = (torch.randn((M, D + 8), generator=g, device="cuda") * 3 + 0.5).to(xdt)[:, :D]
    w = (1 + 0.3 * torch.randn(D, generator=g, device="cuda")).to(bf)
    b = (0.2 * torch.randn(D, generator=g, device="cuda")).to(bf) if layernorm else None
    eps = 1e-5 if layernorm else 1e-6
    q, sinv = ll.norm_fwd_fp8(x, w, b, eps=eps, layernorm=layernorm)
    y = _norm64(x, w, b, eps, layernorm)
    deq = q.double() * sinv.double()[:, None]
    bound = (1 + 2.0 ** -10) * (2.0 ** -4 * y.abs() + 2.0 ** -10 * sinv.double()[:, None])
    assert bool(((deq - y).abs() <= bound).all()), float(((deq - y).abs() / bound).max())
    q2, s2 = ll.norm_fwd_fp8(x, w, b, eps=eps, layernorm=layernorm)
    assert torch.equal(q.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(sinv, s2)
    # against norm_fwd's bf16 row, cast row by row.  A row's scale differs only when bf16 rounding moves its amax across
    # a power-of-two boundary of 448 / amax.  Within a row of equal scale, an element differs only where the bf16 value
    # landed on or across an E4M3 rounding midpoint: a midpoint is one of the ~16 bf16 values per E4M3 step, so about
    # 1/16 of the elements can be affected and about half of those round the other way; and then by one E4M3 step.
    y16, _, _ = ll.norm_fwd(x, w, b, eps=eps, layernorm=layernorm)
    q16, s16 = ll.fp8_quantize_rows(y16)
    same = sinv == s16
    assert float((~same).float().mean()) <= 0.02
    a, c = q[same].float(), q16[same].float()
    differ = a != c
    frac = float(differ.float().mean())
    print(f"norm_fwd_fp8 D={D} {'ln' if layernorm else 'rms'} x={xdt}: {frac:.4f} of the elements differ from the "
          f"bf16 path, {int((~same).sum())} rows with another scale")
    assert frac <= 1 / 16
    step = 2.0 ** (torch.floor(torch.log2(torch.maximum(a.abs(), c.abs()).clamp_min(2.0 ** -6))) - 3)
    assert bool(((a - c).abs()[differ] <= step[differ]).all())


# ------------------------------------------------------------------------------------------------ vector-scale GEMM
def _operand(rows, K, pitch, seed):
    """Integers v in [-4, 4] stored as v * 2^e_r with a per-row exponent e_r in [-2, 3]: (E4M3 [rows, K] view of a
    [rows, pitch] buffer, scale_inv 2^-e_r [rows], v fp32).  Dequantised, the operand is v exactly."""
    g = _gen(seed)
    v = torch.randint(-4, 5, (rows, pitch), generator=g, device="cuda").float()
    e = torch.randint(-2, 4, (rows,), generator=g, device="cuda").float()
    q = (v * torch.exp2(e)[:, None]).to(E4)[:, :K]
    return q, torch.exp2(-e).contiguous(), v[:, :K]


def _mk(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=_gen(seed), device="cuda") * scale).to(bf)


def _teacher_epilogues(M, N, seed):
    rs = (torch.rand((M,), generator=_gen(seed + 4), device="cuda") * 2).float()
    return [
        ("qkv bias", dict(epi=ll.EPI_BF16, bias=_mk((N,), seed + 1))),
        ("qkv", dict(epi=ll.EPI_BF16)),
        ("fc1 gelu erf", dict(epi=ll.EPI_BIAS_GELU, bias=_mk((N,), seed + 3))),
        ("fc1 gelu tanh", dict(epi=ll.EPI_BIAS_GELU, flags=ll.FLAG_GELU_TANH, bias=_mk((N,), seed + 3))),
        ("proj resid gamma", dict(epi=ll.EPI_RESID, bias=_mk((N,), seed + 5), gamma=_mk((N,), seed + 6, 0.1),
                                  aux=torch.randn((M, N), device="cuda"), rowscale=rs)),
        ("fc2 resid", dict(epi=ll.EPI_RESID, bias=_mk((N,), seed + 5), aux=torch.randn((M, N), device="cuda"))),
    ]


@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
@pytest.mark.parametrize("M,N,K", [(333, 392, 200), (517, 136, 256)])
def test_vector_scales_every_teacher_epilogue(cuda_lib, kernel, M, N, K):
    name, flag, tile_n = kernel
    pitch = (K + 15) // 16 * 16 + 16
    a8, sa, a = _operand(M, K, pitch, M + K)
    b8, sb, b = _operand(N, K, pitch, N + K + 1)
    for ename, kw in _teacher_epilogues(M, N, seed=M + N):
        kw = dict(kw)
        flags = kw.pop("flags", 0)
        out_dtype = f32 if kw["epi"] == ll.EPI_RESID else bf
        out0 = torch.full((M, N), float("nan"), device="cuda", dtype=out_dtype)
        got = ll.gemm_fp8(a8, sa, b8, sb, out0=out0, flags=flags | flag, tile_n=tile_n, **kw)
        (ref, scale), = gemm_ref(a, b, flags=flags, **kw)[:1]
        e, where = worst(elem_errors(got, ref, scale))
        assert e <= (LIMIT_F32 if got.dtype == f32 else LIMIT_BF16), (name, ename, e, where)
        again = ll.gemm_fp8(a8, sa, b8, sb, out0=out0.clone(), flags=flags | flag, tile_n=tile_n, **kw)
        assert torch.equal(got, again), (name, ename)


@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
def test_constant_vectors_match_scalar_scales(cuda_lib, kernel):
    name, flag, tile_n = kernel
    M, N, K = 1000, 648, 1408
    g = _gen(11)
    a8 = (torch.randn((M, K), generator=g, device="cuda") * 40).to(E4)
    b8 = (torch.randn((N, K), generator=g, device="cuda") * 40).to(E4)
    sa, sb = torch.tensor([2.0 ** -7], device="cuda"), torch.tensor([2.0 ** -9], device="cuda")
    va, vb = sa.expand(M).contiguous(), sb.expand(N).contiguous()
    for ename, kw in _teacher_epilogues(M, N, seed=5):
        kw = dict(kw)
        flags = kw.pop("flags", 0) | flag
        s = ll.gemm_fp8(a8, sa, b8, sb, flags=flags, tile_n=tile_n, **kw)
        v = ll.gemm_fp8(a8, va, b8, vb, flags=flags, tile_n=tile_n, **kw)
        assert torch.equal(s, v), (name, ename)


def test_gemm_fp8_refuses_mismatched_vectors(cuda_lib):
    a = torch.zeros((64, 128), device="cuda", dtype=E4)
    b = torch.zeros((32, 128), device="cuda", dtype=E4)
    with pytest.raises(_lib.IvbError, match="vector scales"):
        ll.gemm_fp8(a, torch.ones(63, device="cuda"), b, torch.ones(32, device="cuda"))
    with pytest.raises(_lib.IvbError, match="vector scales"):
        ll.gemm_fp8(a, torch.ones(64, device="cuda"), b, torch.ones(1, device="cuda"))


TEACHER_GEMMS = [  # (name, M, N, K): InternVL-6B (B = 32 clips x 8 frames x 257 tokens), VideoMAEv2-g (32 x 2048)
    ("ivl qkv", 65792, 9600, 3200), ("ivl proj", 65792, 3200, 3200), ("ivl fc1", 65792, 12800, 3200),
    ("ivl fc2", 65792, 3200, 12800), ("mae qkv", 65536, 4224, 1408), ("mae proj", 65536, 1408, 1408),
    ("mae fc1", 65536, 6144, 1408), ("mae fc2", 65536, 1408, 6144),
]


def rowwise_accumulation_ratio(M, N, K, seed=0):
    """||C_kernel - C64(deq)||_F / ||C64(deq) - C64(bf16)||_F for Gaussian operands cast row by row (a) and per output
    channel (b), on the library's default kernel."""
    a = _mk((M, K), seed)
    b = _mk((N, K), seed + 1, 0.02)
    qa, sa = ll.fp8_quantize_rows(a)
    qb, sb = ll.fp8_quantize_rows(b)
    c = ll.gemm_fp8(qa, sa, qb, sb, epi=ll.EPI_F32)
    num = den = 0.0
    bd = (qb.double() * sb.double()[:, None]).t()
    b64 = b.double().t()
    for r in range(0, M, 2048):
        rows = slice(r, min(r + 2048, M))
        c_deq = (qa[rows].double() * sa[rows].double()[:, None]) @ bd
        c_bf = a[rows].double() @ b64
        num += float(((c[rows].double() - c_deq) ** 2).sum())
        den += float(((c_deq - c_bf) ** 2).sum())
    return (num / den) ** 0.5


@pytest.mark.parametrize("name,M,N,K", TEACHER_GEMMS, ids=[s[0] for s in TEACHER_GEMMS])
def test_accumulation_error_at_teacher_shapes(cuda_lib, name, M, N, K):
    r = rowwise_accumulation_ratio(M, N, K)
    print(f"{name}: accumulation ratio {r:.4f}")
    assert r <= 0.25, (name, r)
