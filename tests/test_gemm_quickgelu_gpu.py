"""QuickGELU (IVB_FLAG_GELU_QUICK, x * sigmoid(1.702 x)) in the fused GEMM epilogues, element by element against
float64 (gpu), on every kernel the library can select: the cooperative kernel at tile_n 128 and 192, the ping-pong
kernel, the CTA pair, the default choice, the DropPath-planned bf16 GEMM, and the per-token FP8 GEMM (vector scales)
on its kernel forms and in its planned form.

Four epilogue forms: EPI_BIAS_GELU writing out1 = h, EPI_BIAS_GELU writing out1 = gelu'(h) (FLAG_GELU_SAVE_GRAD),
EPI_GELU_BWD from h, and EPI_GELU_BWD from the saved gelu'.  The accumulator's float64 reference and its error bound
come from tests/gemm_ref.py (an EPI_F32 call with the same operands and bias); the QuickGELU value, derivative and
the error of their fp32 evaluation (one MUFU.EX2, one MUFU.RCP and a few roundings) are stated here.  The FP8 operands
are tests/fp8_exact.py's exact ones, so the FP8 accumulation is exact and the same reference applies.

Each error is the largest |got - ref| over (bound + half an ulp of the output), and must stay below 1.9, the limit
test_gemm_epilogue_gpu.py holds the erf and tanh forms to.
"""
import pytest
import torch

import fp8_exact as fx
from gemm_ref import U24, elem_errors, gemm_ref, worst
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu

bf, f32 = torch.bfloat16, torch.float32
LIMIT = 1.9
EVAL = 2.0 ** -21          # fp32 evaluation of sigmoid(1.702 x) (as gemm_ref.EVAL for the other GELU forms)
C = 1.702
QUICK, SAVE = ll.FLAG_GELU_QUICK, ll.FLAG_GELU_SAVE_GRAD
M, N, K = 333, 264, 136    # ragged in M and N (tile edges inside the last tiles)
K8 = 16                    # the FP8 tests' K: exact integer sums of at most 16 unit products


def quick64(h):
    """QuickGELU in float64: value, first and second derivative, and the bounds of the kernel's fp32 evaluation of the
    value and of the derivative (an error ds <= EVAL s in s moves h s by |h| ds and s + C h s (1 - s) by at most
    (1 + C |h|) ds, plus the roundings of the products)."""
    s = torch.sigmoid(C * h)
    f = h * s
    d1 = s + C * h * s * (1 - s)
    d2 = C * s * (1 - s) * (2 + C * h * (1 - 2 * s))
    e0 = EVAL * (f.abs() + h.abs() * d1.abs())
    e1 = EVAL * (s * (2 + 2 * C * h.abs()) + h.abs() * d2.abs())
    return f, d1, d2, e0, e1


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(bf)


def _operands(seed=7):
    a, b = _mk((M, K), seed), _mk((N, K), seed + 1, 0.15)
    bias = _mk((N,), seed + 2, 0.3)
    return a, b, bias


def _fp8_operands(seed):
    """Exact FP8 operands (tests/fp8_exact.py): E4M3 values v 2^e with v in {-1, 0, 1} and one exponent per row, so the
    tensor core's FP8 accumulation and the dequantisation are exact; the pre-activation is an integer in [-K8, K8]
    plus a bias on a 2^-8 grid in (-4, 4), which spans QuickGELU's curved range.  Returns the E4M3 operands with
    their scale vectors, the dequantised operands (exact in bf16) and the bias."""
    a8, sa, va = fx.vec_operand(M, K8, K8, seed, 1)
    b8, sb, vb = fx.vec_operand(N, K8, K8, seed + 1, 1)
    bias = fx.grid_values((N,), seed + 2, limit=4.0).to(bf)
    return (a8, sa, b8, sb), va.to(bf), vb.to(bf), bias


def _refs(form, a, b, bias, aux):
    """[(ref, bound) of out0, (of out1)] of one epilogue form over operands a, b (bf16, exact)."""
    if form.startswith("fwd"):
        ((v, acc),) = gemm_ref(a, b, epi=ll.EPI_F32, bias=bias)
        f, d1, d2, e0, e1 = quick64(v)
        out1 = (d1, d2.abs() * acc + e1) if form == "fwd_save" else (v, acc)
        return [(f, d1.abs() * acc + e0), out1]
    ((v, acc),) = gemm_ref(a, b, epi=ll.EPI_F32)
    h = aux.double()
    if form == "bwd_save":
        d, e = h, torch.zeros_like(h)
    else:
        _, d, _, _, e = quick64(h)
    return [(v * d, d.abs() * acc + v.abs() * e + U24 * (v * d).abs())]


def _aux(form, seed=11):
    h = _mk((M, N), seed, 1.5)
    if form == "bwd_save":
        return quick64(h.double())[1].to(bf)
    return h


FORMS = ["fwd", "fwd_save", "bwd", "bwd_save"]


def _epi(form):
    if form.startswith("fwd"):
        return ll.EPI_BIAS_GELU, QUICK | (SAVE if form == "fwd_save" else 0)
    return ll.EPI_GELU_BWD, QUICK | (SAVE if form == "bwd_save" else 0)


def _check(outs, refs, live_rows, what):
    for i, (got, (ref, bound)) in enumerate(zip(outs, refs)):
        e = elem_errors(got[live_rows], ref[live_rows], bound[live_rows])
        val, where = worst(e)
        assert val <= LIMIT, f"{what}: out{i} error {val:.3g} x tol at {where}"


BF16_KERNELS = [("coop128", ll.FLAG_1CTA, 128), ("coop192", ll.FLAG_1CTA, 192), ("pingpong", ll.FLAG_PINGPONG, 0),
                ("pair128", ll.FLAG_2CTA, 128), ("default", 0, 0)]


def _dead_first_tile():
    """DropPath factors whose first 128-row tile is dropped, and their plan (ops.droppath_plan)."""
    rs = torch.ones(M, device="cuda", dtype=f32)
    rs[:128] = 0
    return rs, ops.droppath_plan(rs[None].contiguous())[0]


def _run(fn, form, with_out1):
    out0 = torch.full((M, N), float("nan"), device="cuda", dtype=bf)
    out1 = torch.full((M, N), float("nan"), device="cuda", dtype=bf) if with_out1 else None
    try:
        fn(out0, out1)
    except ll._lib.IvbError as e:
        pytest.skip(f"refused by the library: {e}")
    torch.cuda.synchronize()
    return [out0] + ([out1] if with_out1 else [])


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kern", BF16_KERNELS + [("plan", 0, 0)], ids=lambda k: k[0])
def test_quickgelu_bf16(cuda_lib, kern, form):
    name, flag, tile_n = kern
    a, b, bias = _operands()
    aux = _aux(form)
    epi, flags = _epi(form)
    fwd = form.startswith("fwd")
    m_plan = None
    live = slice(None)
    if name == "plan":
        _, plan = _dead_first_tile()
        nm = (M + 127) // 128
        m_plan, live = plan[:nm + 1], slice(128, None)

    def call(out0, out1):
        ll.gemm(a, b, epi=epi, flags=flags | flag, out0=out0, out1=out1, bias=bias if fwd else None,
                aux=None if fwd else aux, tile_n=tile_n, m_plan=m_plan)
    outs = _run(call, form, fwd)
    _check(outs, _refs(form, a, b, bias, aux), live, f"{name} {form}")
    if m_plan is not None:      # a dead tile's GELU epilogues write 0
        for o in outs:
            assert (o[:128].float() == 0).all(), f"plan {form}: the dead tile is not 0"


FP8_KERNELS = [("pingpong", ll.FLAG_PINGPONG, 0), ("coop128", ll.FLAG_1CTA, 128), ("coop192", ll.FLAG_1CTA, 192),
               ("default", 0, 0)]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kern", FP8_KERNELS + [("plan", 0, 0)], ids=lambda k: k[0])
def test_quickgelu_fp8_vector_scales(cuda_lib, kern, form):
    name, flag, tile_n = kern
    (qa, sa, qb, sb), a_dq, b_dq, bias = _fp8_operands(21)
    aux = _aux(form, seed=23)
    epi, flags = _epi(form)
    fwd = form.startswith("fwd")
    m_plan, live = None, slice(None)
    if name == "plan":
        _, plan = _dead_first_tile()
        m_plan, live = plan[:(M + 127) // 128 + 1], slice(128, None)

    def call(out0, out1):
        ll._gemm_fp8_plan(qa, sa, qb, sb, m_plan, epi=epi, flags=flags | flag, out0=out0, out1=out1,
                          bias=bias if fwd else None, aux=None if fwd else aux, tile_n=tile_n)
    outs = _run(call, form, fwd)
    _check(outs, _refs(form, a_dq, b_dq, bias, aux), live, f"fp8 {name} {form}")
    if m_plan is not None:
        for o in outs:
            assert (o[:128].float() == 0).all(), f"fp8 plan {form}: the dead tile is not 0"


def _all_bf16():
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(bf)


# The documented domain (ivb_ptx.cuh): below h = -51 the fast reciprocal of 1 + e^{-1.702 h} (above 2^126) is 0, so
# both functions return 0 where the exact values are below 1e-36; gelu_quick_grad is NaN for |h| above 2e38, where
# 1.702 h overflows.
TAIL, BIG = -50.0, 2.0 ** 127


def _sweep_checks(hd, got, ref, bound, what, deriv):
    fin = torch.isfinite(hd)
    live = fin & (hd >= TAIL) & (hd.abs() <= 2.0 ** 10)
    e = elem_errors(got[live], ref[live], bound[live])
    i = int(e.argmax())
    assert float(e[i]) <= LIMIT, (f"{what}: error {float(e[i]):.3g} x tol at h = {float(hd[live][i]):.6g} "
                                  f"(got {float(got[live][i]):.6g}, want {float(ref[live][i]):.6g})")
    tail = fin & (hd < TAIL) & (hd.abs() < BIG)
    assert (got[tail].double().abs() <= 1e-30).all(), f"{what}: the left tail is not 0"
    dom = fin & (hd.abs() < BIG) if deriv else fin
    assert torch.isfinite(got[dom]).all(), f"{what}: not finite inside its documented domain"
    if deriv:
        assert torch.isnan(got[fin & (hd.abs() > 2.0e38)]).all(), f"{what}: the documented NaN range is out of date"
    assert torch.isnan(got[torch.isnan(hd)]).all(), f"{what}: NaN does not propagate"


@pytest.mark.parametrize("kern", [("coop128", ll.FLAG_1CTA, 128), ("pingpong", ll.FLAG_PINGPONG, 0),
                                  ("default", 0, 0)], ids=lambda k: k[0])
def test_gelu_quick_every_bf16_value(cuda_lib, kern):
    """EPI_BIAS_GELU with A = 0 and bias = h (acc + bias is exactly h) over all 65536 bf16 patterns, writing gelu_quick
    and (FLAG_GELU_SAVE_GRAD) gelu_quick_grad; then EPI_GELU_BWD with acc = 1 and aux = every pattern."""
    name, flag, tile_n = kern
    h = _all_bf16()
    Nn, Mm, Kk = h.numel(), 2, 8
    a = torch.zeros((Mm, Kk), device="cuda", dtype=bf)
    b = torch.zeros((Nn, Kk), device="cuda", dtype=bf)
    g = torch.empty((Mm, Nn), device="cuda", dtype=bf)
    d = torch.empty((Mm, Nn), device="cuda", dtype=bf)
    ll.gemm(a, b, epi=ll.EPI_BIAS_GELU, flags=QUICK | SAVE | flag, bias=h, out0=g, out1=d, tile_n=tile_n)
    aux = h.reshape(256, 256)
    a1 = torch.zeros((256, Kk), device="cuda", dtype=bf)
    b1 = torch.zeros((256, Kk), device="cuda", dtype=bf)
    a1[:, 0] = 1
    b1[:, 0] = 1
    gb = torch.empty((256, 256), device="cuda", dtype=bf)
    ll.gemm(a1, b1, epi=ll.EPI_GELU_BWD, flags=QUICK | flag, aux=aux, out0=gb, tile_n=tile_n)
    torch.cuda.synchronize()
    hd = h.double()
    f, d1, _, e0, e1 = quick64(torch.nan_to_num(hd, nan=0.0, posinf=0.0, neginf=0.0))
    _sweep_checks(hd, g[0], f, e0, f"{name} gelu_quick", False)
    _sweep_checks(hd, d[0], d1, e1, f"{name} gelu_quick_grad (saved)", True)
    _sweep_checks(hd, gb.reshape(-1), d1, e1 + U24 * d1.abs(), f"{name} gelu_quick_grad (GELU_BWD)", True)


def test_tanh_and_quick_refused(cuda_lib):
    a, b, bias = _operands()
    out = torch.empty((M, N), device="cuda", dtype=bf)
    with pytest.raises(ll._lib.IvbError, match="exclude each other"):
        ll.gemm(a, b, epi=ll.EPI_BIAS_GELU, flags=QUICK | ll.FLAG_GELU_TANH, bias=bias, out0=out)


def test_block_quickgelu_against_float64(cuda_lib):
    """One fused LayerNorm block with gelu_quick against a float64 restatement (nn.MultiheadAttention semantics), forward
    and the fc1 / fc2 weight gradients, whose only QuickGELU-specific inputs are the epilogues under test."""
    torch.manual_seed(0)
    B, n, D, H = 2, 70, 128, 2
    lin = lambda o, i, s=0.05: (torch.randn(o, i) * s).to(bf).cuda().requires_grad_(True)  # noqa: E731
    vec = lambda k, m=0.0, s=0.05: (m + torch.randn(k) * s).to(bf).cuda().requires_grad_(True)  # noqa: E731
    P = ops.BlockParams(n1w=vec(D, 1.0), n1b=vec(D), qkvw=lin(3 * D, D), qkvb=vec(3 * D), qnw=None, knw=None,
                        projw=lin(D, D), projb=vec(D), g1=None, n2w=vec(D, 1.0), n2b=vec(D), fc1w=lin(4 * D, D),
                        fc1b=vec(4 * D), fc2w=lin(D, 4 * D), fc2b=vec(D), g2=None)
    x = torch.randn(B * n, D, device="cuda")
    spec = ops.BlockSpec(B, n, H, layernorm=True, gelu_quick=True, eps1=1e-5, eps2=1e-5)
    y = ops.BlockFn.apply(x, spec, None, None, *P)
    w = torch.randn_like(y)
    (y * w).sum().backward()

    p64 = {k: v.detach().double().requires_grad_(True) for k, v in P._asdict().items() if v is not None}
    x64 = x.double()
    ln = lambda t, a, c: torch.nn.functional.layer_norm(t, (D,), p64[a], p64[c], 1e-5)  # noqa: E731
    h = ln(x64, "n1w", "n1b")
    q, k, v = (h @ p64["qkvw"].t() + p64["qkvb"]).reshape(B, n, 3, H, D // H).permute(2, 0, 3, 1, 4)
    att = torch.softmax(q @ k.transpose(-1, -2) * (D // H) ** -0.5, -1) @ v
    x1 = x64 + att.transpose(1, 2).reshape(B * n, D) @ p64["projw"].t() + p64["projb"]
    hh = ln(x1, "n2w", "n2b") @ p64["fc1w"].t() + p64["fc1b"]
    y64 = x1 + (hh * torch.sigmoid(C * hh)) @ p64["fc2w"].t() + p64["fc2b"]
    (y64 * w.double()).sum().backward()
    rel = lambda g, r: float((g.double() - r).norm() / r.norm())  # noqa: E731
    assert rel(y, y64.detach()) < 1e-2
    for name in ("fc1w", "fc1b", "fc2w", "qkvw"):
        assert rel(getattr(P, name).grad, p64[name].grad) < 3e-2, name
