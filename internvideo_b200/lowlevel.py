"""Thin tensor-level wrappers over the C ABI (no autograd): pointer/shape plumbing only.

Every function checks its tensor operands with _chk (a required operand must not be None; each given one must be a
CUDA tensor of the expected dtype) and raises otherwise; nothing here computes on the CPU.  Every entry point that
takes a stream is called through _call.
"""
from __future__ import annotations

import torch

from . import _lib

EPI_BF16, EPI_F32, EPI_BIAS_GELU, EPI_RESID, EPI_GELU_BWD = 0, 1, 2, 3, 4
EPI_SWIGLU = 5             # silu(x gate^T) * (x up^T) from one [gate; up] weight [2I, K]; out0 is [M, I]
FLAG_GELU_TANH, FLAG_ACCUM, FLAG_1CTA, FLAG_2CTA, FLAG_GELU_SAVE_GRAD, FLAG_PINGPONG = 1, 2, 4, 8, 16, 32
FLAG_GELU_QUICK = 128      # QuickGELU x * sigmoid(1.702 x) in the GELU epilogues (excludes FLAG_GELU_TANH)
FLAG_FP8_VECTOR_SCALES = 64

bf16 = torch.bfloat16
f32 = torch.float32
i32 = torch.int32


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _chk(*operands):
    """The one operand check.  Each operand is (name, tensor, dtype or tuple of dtypes); a name ending in "?" marks an
    operand the entry point accepts as NULL, which may be None.  Every missing required operand is refused before any
    device or dtype check."""
    for name, t, _ in operands:
        if t is None and not name.endswith("?"):
            raise _lib.IvbError(f"{name}: required operand is None")
    for name, t, dtype in operands:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.IvbError(f"{name.rstrip('?')}: expected a CUDA tensor (ivb200 has no CPU path)")
        if t.dtype not in (dtype if isinstance(dtype, tuple) else (dtype,)):
            raise _lib.IvbError(f"{name.rstrip('?')}: expected dtype {dtype}, got {t.dtype}")


def _rows2d(t, name):
    """Row pitch (elements) of a 2-D tensor with unit inner stride; 0 for an absent operand."""
    if t is None:
        return 0
    if t.dim() != 2:
        raise _lib.IvbError(f"{name}: expected 2-D tensor, got {tuple(t.shape)}")
    if t.stride(1) != 1:
        raise _lib.IvbError(f"{name}: inner stride must be 1")
    return t.stride(0)


_PROFILERS = []     # the enabled OpProfiler / GemmProfiler objects


def _call(name, *args, kind=None, flops=0.0):
    """The one call path into the library: ivb_<name>(*args, current stream), with a tensor passed as its data_ptr() and
    None as NULL.  Raises IvbError naming the entry point on a non-zero status.  Each enabled profiler that records
    `kind` (default: `name`) gets one (name, kind, flops, start event, end event) record."""
    fn = getattr(_lib.load(), "ivb_" + name)
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    args.append(_stream())
    kind = kind or name
    profs = [p for p in _PROFILERS if p.kinds is None or kind in p.kinds] if _PROFILERS else None
    if profs:
        e0 = torch.cuda.Event(enable_timing=True); e0.record()
    _lib.check(fn(*args), "ivb_" + name)
    if profs:
        e1 = torch.cuda.Event(enable_timing=True); e1.record()
        rec = (_gemm_name(*args) if name.startswith("gemm_bf16") else name, kind, flops, e0, e1)
        for p in profs:
            p.records.append(rec)


def _gemm_name(a, a_t, lda, b, b_t, ldb, M, N, K, epi, *_):
    return f"gemm[{'T' if a_t else 'N'}{'T' if b_t else 'N'} epi{epi}] {M}x{N}x{K}"


class OpProfiler:
    """CUDA-event timing of every library call, in situ (warm caches, real overlap): records holds one
    (name, kind, flops, start, stop) per call, in call order; a bf16 GEMM is named by its layout, epilogue and shape."""
    kinds = None

    def __init__(self):
        self.records = []

    def enable(self):
        if self not in _PROFILERS:
            _PROFILERS.append(self)

    def disable(self):
        if self in _PROFILERS:
            _PROFILERS.remove(self)

    def summary(self):
        torch.cuda.synchronize()
        agg = {}
        for name, _, _, e0, e1 in self.records:
            c, t = agg.get(name, (0, 0.0))
            agg[name] = (c + 1, t + e0.elapsed_time(e1))
        return sorted(agg.items(), key=lambda kv: -kv[1][1])


class GemmProfiler(OpProfiler):
    """CUDA-event timing of every tensor-core launch (GEMMs, bf16 and fp8: kind "gemm"; attention forward / backward)
    and of the fp8 casts that feed the fp8 GEMMs and the fp8 attention (kind "fp8_quantize", no flops) and the norms that
    write FP8 rows (kind "norm_fwd_fp8", no flops) on the launching stream (bench.py roofline).  Records only those
    calls."""
    kinds = frozenset(("gemm", "attn_fwd", "attn_bwd", "fp8_quantize", "norm_fwd_fp8"))

    def __init__(self):
        super().__init__()
        self.count = 0

    def totals(self, kind="gemm"):
        """(total algorithmic FLOPs, total milliseconds) over the recorded launches of `kind`."""
        torch.cuda.synchronize()
        fl = ms = 0.0
        cnt = 0
        for _, k, f, e0, e1 in self.records:
            if k != kind:
                continue
            fl += f
            ms += e0.elapsed_time(e1)
            cnt += 1
        if kind == "gemm":
            self.count = cnt
        return fl, ms


def launch_count() -> int:
    return int(_lib.load().ivb_launch_count())


def reset_launch_count() -> None:
    _lib.load().ivb_reset_launch_count()


def set_default_2cta(enable: bool) -> None:
    _lib.load().ivb_set_default_2cta(int(bool(enable)))


def device_check() -> None:
    _lib.check(_lib.load().ivb_device_check(), "ivb_device_check")


# ----------------------------------------------------------------------------------------- GEMM
def gemm(a, b, *, a_t=False, b_t=False, epi=EPI_BF16, flags=0, out0=None, out1=None, bias=None,
         gamma=None, aux=None, rowscale=None, tile_n=0, m_plan=None, k_plan=None):
    """D[M,N] = epi(sum_k A(m,k) B(n,k)).

    a_t=False: `a` is [M,K]; a_t=True: `a` is [K,M] (MN-major operand).
    b_t=False: `b` is [N,K]; b_t=True: `b` is [K,N].
    m_plan / k_plan: the M and K plans of a DropPath plan over the GEMM's M rows / its K (ops.droppath_plan); with
    either the call goes to ivb_gemm_bf16_plan, which skips the work of the dropped rows.
    epi=EPI_SWIGLU: `b` is [gate; up], [N = 2I, K] (K-major), and out0 is [M, I] = silu(x gate^T) * (x up^T).
    """
    _chk(("a", a, bf16), ("b", b, bf16), ("m_plan?", m_plan, i32), ("k_plan?", k_plan, i32))
    lda = _rows2d(a, "a"); ldb = _rows2d(b, "b")
    if a_t:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_t:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    if K != Kb:
        raise _lib.IvbError(f"gemm: contraction mismatch {K} vs {Kb}")
    out0 = _epilogue_operands(M, N, epi, out0, out1, bias, gamma, aux, rowscale, a.device)
    plan = () if m_plan is None and k_plan is None else (m_plan, k_plan)
    _call("gemm_bf16_plan" if plan else "gemm_bf16", a, int(a_t), lda, b, int(b_t), ldb, M, N, K, epi, flags, out0,
          _rows2d(out0, "out0"), out1, _rows2d(out1, "out1"), bias, gamma, aux, _rows2d(aux, "aux"), rowscale, tile_n,
          *plan, kind="gemm", flops=2.0 * M * N * K)
    return out0



def _epilogue_operands(M, N, epi, out0, out1, bias, gamma, aux, rowscale, device):
    """Checks the fused epilogue's operands of an [M, N] GEMM, allocating out0 if it is None.  Returns out0."""
    out_dtype = f32 if epi in (EPI_F32, EPI_RESID) else bf16
    if out0 is None:
        out0 = torch.empty((M, N // 2 if epi == EPI_SWIGLU else N), device=device, dtype=out_dtype)
    _chk(("out0", out0, out_dtype), ("out1?", out1, bf16), ("bias?", bias, bf16), ("gamma?", gamma, bf16),
         ("aux?", aux, f32 if epi == EPI_RESID else bf16), ("rowscale?", rowscale, f32))
    return out0


# ----------------------------------------------------------------------------------------- FP8
FP8_E4M3, FP8_E5M2 = 0, 1
FP8_DTYPES = {FP8_E4M3: torch.float8_e4m3fn, FP8_E5M2: torch.float8_e5m2}


def _pad16(n):
    return (n + 15) // 16 * 16


def _fp8_rows(rows, cols, device, dtype=torch.float8_e4m3fn):
    """An uninitialised FP8 [rows, cols] view of a buffer whose row pitch is cols rounded up to 16 elements (the fp8
    GEMM's operand rule)."""
    return torch.empty((rows, _pad16(cols)), device=device, dtype=dtype)[:, :cols]


def fp8_quantize(x, fmt=FP8_E4M3, transpose=False):
    """Per-tensor current-scaling cast of a bf16 [M, K] tensor (any row pitch) to FP8 (ivb_fp8_quantize).

    Returns (q [M, K], q_t [K, M] = q^T or None, scale_inv fp32 [1], amax fp32 [1]): x ~ q * scale_inv, with a
    power-of-two scale.  q and q_t are views of buffers whose row pitch is rounded up to 16 elements (the fp8 GEMM's
    operand rule)."""
    _chk(("x", x, bf16))
    ldx = _rows2d(x, "x")
    M, K = x.shape
    dt = FP8_DTYPES[fmt]
    q = _fp8_rows(M, K, x.device, dt)
    q_t = _fp8_rows(K, M, x.device, dt) if transpose else None
    stats = torch.empty((2,), device=x.device, dtype=f32)
    amax, scale_inv = stats[0:1], stats[1:2]
    _call("fp8_quantize", x, ldx, M, K, fmt, q, q.stride(0), q_t, q_t.stride(0) if transpose else 0, amax, scale_inv)
    return q, q_t, scale_inv, amax


def fp8_quantize_rows(x, transposed=False):
    """Per-row current-scaling cast of a bf16 [M, K] tensor (any row pitch) to E4M3 (ivb_fp8_quantize_rows).

    Returns (q [M, K], row_scale_inv fp32 [M]): x[m] ~ q[m] * row_scale_inv[m], each row with its own power-of-two
    scale.  A weight [N, K] quantised this way has one scale per output channel.  q is a view of a buffer whose row
    pitch is rounded up to 16 elements (the fp8 GEMM's operand rule).

    transposed=True casts the rows of x^T instead, reading x once (ivb_fp8_quantize_cols_t): (q_t [K, M], col_scale_inv
    fp32 [K]) with x[:, k] ~ q_t[k] * col_scale_inv[k].  For a weight [N, K] that is the B operand of the input-gradient
    GEMM dx = dy W, with one scale per input channel of the weight."""
    _chk(("x", x, bf16))
    ldx = _rows2d(x, "x")
    M, K = x.shape
    if transposed:
        q_t = _fp8_rows(K, M, x.device)
        amax = torch.empty((K,), device=x.device, dtype=f32)
        sinv = torch.empty((K,), device=x.device, dtype=f32)
        _call("fp8_quantize_cols_t", x, ldx, M, K, q_t, q_t.stride(0), amax, sinv, kind="fp8_quantize")
        return q_t, sinv
    q = _fp8_rows(M, K, x.device)
    sinv = torch.empty((M,), device=x.device, dtype=f32)
    _call("fp8_quantize_rows", x, ldx, M, K, q, q.stride(0), sinv, kind="fp8_quantize")
    return q, sinv


def norm_fwd_fp8(x, weight, bias=None, eps=1e-6, layernorm=False, save=False):
    """RMSNorm / LayerNorm of x [M, D] (fp32 or bf16, any row pitch) written only as E4M3 rows with per-row scales
    (ivb_norm_fwd_fp8).  Returns (q [M, D] float8_e4m3fn, row_scale_inv fp32 [M]): q[m] * row_scale_inv[m] is the
    row norm_fwd would round to bf16, rounded to E4M3 instead.

    save=True also writes what a backward needs, from the same read of each row (ivb_norm_fwd_fp8_train), and returns
    (q, row_scale_inv, y, mean | None, rstd): q and row_scale_inv the same bits, y (bf16 [M, D]), mean (LayerNorm only)
    and rstd norm_fwd's bits."""
    _chk(("x", x, (f32, bf16)), ("weight", weight, bf16), ("bias?", bias, bf16))
    ldx = _rows2d(x, "x")
    M, D = x.shape
    q = _fp8_rows(M, D, x.device)
    sinv = torch.empty((M,), device=x.device, dtype=f32)
    if not save:
        _call("norm_fwd_fp8", x, int(x.dtype == f32), ldx, weight, bias, float(eps), int(layernorm), M, D, q,
              q.stride(0), sinv)
        return q, sinv
    y = torch.empty((M, D), device=x.device, dtype=bf16)
    rstd = torch.empty((M,), device=x.device, dtype=f32)
    mean = torch.empty((M,), device=x.device, dtype=f32) if layernorm else None
    _call("norm_fwd_fp8_train", x, int(x.dtype == f32), ldx, weight, bias, float(eps), int(layernorm), M, D, q,
          q.stride(0), sinv, y, y.stride(0), mean, rstd, kind="norm_fwd_fp8")
    return q, sinv, y, mean, rstd


def gemm_fp8(a, a_scale_inv, b, b_scale_inv, *, epi=EPI_BF16, flags=0, out0=None, out1=None, bias=None, gamma=None,
             aux=None, rowscale=None, tile_n=0):
    """D[M,N] = epi(a_scale_inv * b_scale_inv * sum_k A(m,k) B(n,k)) on the FP8 tensor cores (ivb_gemm_fp8).

    a: [M,K] float8_e4m3fn or float8_e5m2; b: [N,K] float8_e4m3fn; both K-major (fp8_quantize's q, or q_t for a
    transposed operand).  a_scale_inv / b_scale_inv: fp32 [1] CUDA tensors (per-tensor scales), or fp32 [M] and [N]
    vectors (per-row scales of a, per-output-channel scales of b, as fp8_quantize_rows / norm_fwd_fp8 give them; a
    must then be E4M3), which sets FLAG_FP8_VECTOR_SCALES.  Epilogue arguments as for gemm()."""
    return _gemm_fp8_plan(a, a_scale_inv, b, b_scale_inv, None, epi=epi, flags=flags, out0=out0, out1=out1, bias=bias,
                          gamma=gamma, aux=aux, rowscale=rowscale, tile_n=tile_n)


def _gemm_fp8_plan(a, a_scale_inv, b, b_scale_inv, m_plan, *, epi=EPI_BF16, flags=0, out0=None, out1=None, bias=None,
                   gamma=None, aux=None, rowscale=None, tile_n=0):
    """gemm_fp8 with the M plan of a DropPath plan over its M rows (as for gemm(); vector scales only), through
    ivb_gemm_fp8_plan, which skips the row tiles of the dropped rows; m_plan None: gemm_fp8 itself.  The block's
    per-token FP8 path (ops.block_forward / block_backward) is its caller, as ops.droppath_plan is the plans' maker:
    gemm_fp8, the public FP8 GEMM, stays the unplanned call."""
    _chk(("a", a, tuple(FP8_DTYPES.values())), ("a_scale_inv", a_scale_inv, f32), ("b", b, torch.float8_e4m3fn),
         ("b_scale_inv", b_scale_inv, f32), ("m_plan?", m_plan, i32))
    lda = _rows2d(a, "a"); ldb = _rows2d(b, "b")
    M, K = a.shape
    N, Kb = b.shape
    if K != Kb:
        raise _lib.IvbError(f"gemm_fp8: contraction mismatch {K} vs {Kb}")
    out0 = _epilogue_operands(M, N, epi, out0, out1, bias, gamma, aux, rowscale, a.device)
    fmt = FP8_E5M2 if a.dtype == torch.float8_e5m2 else FP8_E4M3
    if a_scale_inv.numel() != 1 or b_scale_inv.numel() != 1:
        if (a_scale_inv.shape != (M,) or b_scale_inv.shape != (N,) or not a_scale_inv.is_contiguous()
                or not b_scale_inv.is_contiguous()):
            raise _lib.IvbError(f"gemm_fp8: vector scales must be contiguous [M] = [{M}] and [N] = [{N}], got "
                                f"{tuple(a_scale_inv.shape)} and {tuple(b_scale_inv.shape)}")
        flags |= FLAG_FP8_VECTOR_SCALES
    plan = () if m_plan is None else (m_plan,)
    _call("gemm_fp8_plan" if plan else "gemm_fp8", a, 0, lda, fmt, a_scale_inv, b, 0, ldb, b_scale_inv, M, N, K, epi,
          flags, out0, _rows2d(out0, "out0"), out1, _rows2d(out1, "out1"), bias, gamma, aux, _rows2d(aux, "aux"),
          rowscale, tile_n, *plan, kind="gemm", flops=2.0 * M * N * K)
    return out0


def _fp8_quantize_blocks_t(x, rowscale=None):
    """Transposing cast of a bf16 [M, C] tensor of M tokens (any row pitch) to E4M3 with one power-of-two scale per
    channel per 128-token block (ivb_fp8_quantize_blocks_t): the operands of the FP8 weight gradient, _gemm_fp8_wgrad.

    Returns (q_t [C, M] float8_e4m3fn, scale_inv fp32 [ceil(M/128), C]): x[128b + i, c] ~ q_t[c, 128b + i] *
    scale_inv[b, c].  q_t is a view of a buffer whose row pitch is rounded up to 16 elements.  rowscale: optional fp32
    [M] DropPath factors (ivb_fp8_quantize_blocks_t_plan): tokens whose factor is 0 are cast as zeros.  Private, as
    _gemm_fp8_plan: the block backward's FP8 weight gradients (ops.block_backward) are its caller."""
    _chk(("x", x, bf16), ("rowscale?", rowscale, f32))
    ldx = _rows2d(x, "x")
    M, C = x.shape
    _chk_rowscale("fp8_quantize_blocks_t", rowscale, M)
    q_t = _fp8_rows(C, M, x.device)
    sinv = torch.empty(((M + 127) // 128, C), device=x.device, dtype=f32)
    plan = () if rowscale is None else (rowscale,)
    _call("fp8_quantize_blocks_t_plan" if plan else "fp8_quantize_blocks_t", x, ldx, M, C, q_t, q_t.stride(0), sinv,
          *plan, kind="fp8_quantize")
    return q_t, sinv


def _gemm_fp8_wgrad(a_t, a_scale_inv, b_t, b_scale_inv, *, epi=EPI_BF16, flags=0, out0=None, k_plan=None):
    """The weight gradient D[M, N] = sum over tokens k of dy[k, m] act[k, n] on the FP8 tensor cores from the
    block-scaled transposed copies _fp8_quantize_blocks_t makes (ivb_gemm_fp8_wgrad): a_t = dy^T [M, K] with a_scale_inv
    [ceil(K/128), M], b_t = act^T [N, K] with b_scale_inv [ceil(K/128), N].  epi EPI_BF16 or EPI_F32; flags 0 or
    FLAG_ACCUM (accumulate into out0).  k_plan: optional list of the 128-token k-blocks to sum, in the format of a
    DropPath plan's M plan over the tokens (ops._branch_plans)."""
    _chk(("a_t", a_t, torch.float8_e4m3fn), ("a_scale_inv", a_scale_inv, f32), ("b_t", b_t, torch.float8_e4m3fn),
         ("b_scale_inv", b_scale_inv, f32), ("k_plan?", k_plan, i32))
    M, K = a_t.shape
    N, Kb = b_t.shape
    if K != Kb:
        raise _lib.IvbError(f"gemm_fp8_wgrad: contraction mismatch {K} vs {Kb}")
    nkb = (K + 127) // 128
    for nm, sc, n in (("a_scale_inv", a_scale_inv, M), ("b_scale_inv", b_scale_inv, N)):
        if sc.shape != (nkb, n) or not sc.is_contiguous():
            raise _lib.IvbError(f"gemm_fp8_wgrad: {nm} must be a contiguous [{nkb}, {n}], got {tuple(sc.shape)}")
    out0 = _epilogue_operands(M, N, epi, out0, None, None, None, None, None, a_t.device)
    _call("gemm_fp8_wgrad", a_t, _rows2d(a_t, "a_t"), a_scale_inv, b_t, _rows2d(b_t, "b_t"), b_scale_inv, M, N, K, epi,
          flags, out0, _rows2d(out0, "out0"), k_plan, kind="gemm", flops=2.0 * M * N * K)
    return out0


# ----------------------------------------------------------------------------------------- norms
def norm_fwd(x, weight, bias=None, eps=1e-6, layernorm=False, out=None, want_stats=True):
    """x: [M,D] fp32 or bf16 (row stride arbitrary). Returns (y bf16, mean|None, rstd)."""
    _chk(("x", x, (f32, bf16)), ("weight", weight, bf16), ("bias?", bias, bf16), ("out?", out, bf16))
    ldx = _rows2d(x, "x")
    M, D = x.shape
    if out is None:
        out = torch.empty((M, D), device=x.device, dtype=bf16)
    rstd = torch.empty((M,), device=x.device, dtype=f32) if want_stats else None
    mean = torch.empty((M,), device=x.device, dtype=f32) if (want_stats and layernorm) else None
    _call("norm_fwd", x, int(x.dtype == f32), ldx, weight, bias, float(eps), int(layernorm), M, D, out,
          _rows2d(out, "out"), mean, rstd)
    return out, mean, rstd


def rmsnorm_pair_fwd(qkv, D, w0, w1, out, eps=1e-6, want_stats=True):
    """RMSNorm of the q and k column slices ([:, :D] and [:, D:2D]) of a bf16 [M, >=2D] projection buffer in one
    launch -> out[:, :D], out[:, D:2D] (bf16 [M, >=2D]).  Returns rstd fp32 [M, 2] (or None)."""
    _chk(("qkv", qkv, bf16), ("w0", w0, bf16), ("w1", w1, bf16), ("out", out, bf16))
    M = qkv.shape[0]
    rstd = torch.empty((M, 2), device=qkv.device, dtype=f32) if want_stats else None
    _call("rmsnorm_pair_fwd", qkv, _rows2d(qkv, "qkv"), D, w0, w1, float(eps), M, D, out, _rows2d(out, "out"), D, rstd)
    return rstd


def rmsnorm_pair_bwd(dqk, qkv, D, w0, w1, rstd, dw0=None, dw1=None):
    """Backward of rmsnorm_pair_fwd, IN PLACE on the gradient buffer: dqk[:, :D] / dqk[:, D:2D] hold d(normed q/k) on
    entry and d(q/k) on return.  dw0/dw1: optional fp32 [D] accumulators."""
    _chk(("dqk", dqk, bf16), ("qkv", qkv, bf16), ("w0", w0, bf16), ("w1", w1, bf16), ("rstd", rstd, f32),
         ("dw0?", dw0, f32), ("dw1?", dw1, f32))
    M = qkv.shape[0]
    ld = _rows2d(dqk, "dqk")
    _call("rmsnorm_pair_bwd", dqk, ld, D, qkv, _rows2d(qkv, "qkv"), D, w0, w1, rstd, M, D, dqk, ld, D, dw0, dw1)
    return dqk


def norm_bwd(dy, x, weight, mean, rstd, layernorm=False, dx_in=None, dx_out=None,
             dx_dtype=f32, dweight=None, dbias=None):
    _chk(("dy", dy, bf16), ("x", x, (f32, bf16)), ("weight", weight, bf16), ("mean?", mean, f32), ("rstd", rstd, f32),
         ("dx_in?", dx_in, f32), ("dx_out?", dx_out, (f32, bf16)), ("dweight?", dweight, f32), ("dbias?", dbias, f32))
    M, D = x.shape
    lddy = _rows2d(dy, "dy"); ldx = _rows2d(x, "x")
    if dx_out is None:
        dx_out = torch.empty((M, D), device=x.device, dtype=dx_dtype)
    _call("norm_bwd", dy, lddy, x, int(x.dtype == f32), ldx, weight, mean, rstd, int(layernorm), M, D, dx_in,
          _rows2d(dx_in, "dx_in"), dx_out, int(dx_out.dtype == f32), _rows2d(dx_out, "dx_out"), dweight, dbias)
    return dx_out


def rmsnorm_bwd_layerscale(dy, x, weight, rstd, dx_in, ybr, gamma, dweight, dgamma, dcolsum, rowscale=None):
    """RMSNorm backward on the fp32 stream fused with the LayerScale backward of the preceding branch (one pass over the
    rows).  Returns (dx fp32 [M,D], dyb bf16 [M,D])."""
    _chk(("dy", dy, bf16), ("x", x, f32), ("weight", weight, bf16), ("rstd", rstd, f32), ("dx_in?", dx_in, f32),
         ("ybr", ybr, bf16), ("gamma", gamma, bf16), ("dweight?", dweight, f32), ("dgamma?", dgamma, f32),
         ("dcolsum?", dcolsum, f32), ("rowscale?", rowscale, f32))
    M, D = x.shape
    dx = torch.empty((M, D), device=x.device, dtype=f32)
    dyb = torch.empty((M, D), device=x.device, dtype=bf16)
    _call("rmsnorm_bwd_layerscale", dy, _rows2d(dy, "dy"), x, _rows2d(x, "x"), weight, rstd, M, D, dx_in,
          _rows2d(dx_in, "dx_in"), dx, D, dweight, ybr, _rows2d(ybr, "ybr"), gamma, rowscale, dyb, D, dgamma, dcolsum)
    return dx, dyb


def layerscale_bwd(dx, y, gamma, dgamma=None, dcolsum=None, out=None, rowscale=None):
    _chk(("dx", dx, f32), ("y?", y, bf16), ("gamma?", gamma, bf16), ("dgamma?", dgamma, f32),
         ("dcolsum?", dcolsum, f32), ("out?", out, bf16), ("rowscale?", rowscale, f32))
    M, D = dx.shape
    if out is None:
        out = torch.empty((M, D), device=dx.device, dtype=bf16)
    _call("layerscale_bwd", dx, _rows2d(dx, "dx"), y, _rows2d(y, "y"), gamma, M, D, out, _rows2d(out, "out"), dgamma,
          dcolsum, rowscale)
    return out


def colsum(x, out=None):
    _chk(("x", x, bf16), ("out?", out, f32))
    M, N = x.shape
    if out is None:
        out = torch.zeros((N,), device=x.device, dtype=f32)
    _call("colsum_bf16", x, _rows2d(x, "x"), M, N, out)
    return out


# ----------------------------------------------------------------------------------------- attention
def _chk_causal(fn, causal, rowscale):
    if causal and rowscale is not None:
        raise _lib.IvbError(f"{fn}: causal attention has no DropPath plan form (rowscale must be None)")


def attn_fwd(q, k, v, B, n, H, d, scale, out=None, want_lse=True, rowscale=None, causal=False, kv_len=None):
    """q/k/v: 2-D views [B*n, H*d] (any row pitch) of the projection buffers.  rowscale: optional fp32 [B*n] DropPath
    factors of the attention branch (one per clip): the call goes to ivb_attn_fwd_plan, which skips the clips whose
    factor is 0 and writes zeros to their rows.  causal: key index > query index is masked (ivb_attn_fwd_causal; not
    with rowscale).  kv_len: optional contiguous int32 [B], the keys each clip keeps (ivb_attn_fwd_keylen: keys >=
    kv_len[b] are masked for every query of clip b; an entry outside [1, n] makes the clip's rows NaN; not with
    rowscale or causal)."""
    _chk(("q", q, bf16), ("k", k, bf16), ("v", v, bf16), ("out?", out, bf16), ("rowscale?", rowscale, f32),
         ("kv_len?", kv_len, i32))
    _chk_rowscale("attn_fwd", rowscale, B * n)
    _chk_causal("attn_fwd", causal, rowscale)
    if kv_len is not None and (causal or rowscale is not None):
        raise _lib.IvbError("attn_fwd: key lengths (kv_len) have no causal or DropPath plan form")
    if kv_len is not None and (kv_len.shape != (B,) or not kv_len.is_contiguous()):
        raise _lib.IvbError(f"attn_fwd: kv_len must be a contiguous [B] = [{B}], got {tuple(kv_len.shape)}")
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if t.shape != (B * n, H * d):
            raise _lib.IvbError(f"attn_fwd: {nm} must be [B*n, H*d], got {tuple(t.shape)}")
    if out is None:
        out = torch.empty((B * n, H * d), device=q.device, dtype=bf16)
    lse = torch.empty((B, H, n), device=q.device, dtype=f32) if want_lse else None
    extra = (rowscale,) if rowscale is not None else (kv_len,) if kv_len is not None else ()
    name = ("attn_fwd_causal" if causal else "attn_fwd_plan" if rowscale is not None
            else "attn_fwd_keylen" if kv_len is not None else "attn_fwd")
    # QK^T + PV; causal: about half.  With kv_len the host does not know the lengths: n is the upper bound.
    _call(name, q, _rows2d(q, "q"), k, _rows2d(k, "k"), v, _rows2d(v, "v"), out, _rows2d(out, "out"), lse, B, n, H, d,
          float(scale), *extra, kind="attn_fwd", flops=(2.0 if causal else 4.0) * B * H * n * n * d)
    return out, lse


def _rope_qk(q, k, B, L, H, d, cos, sin):
    """Rotary position embedding of the heads of q and k, in place (ivb_rope_qk): q, k bf16 2-D views [B*L, H*d] (any
    row pitch; e.g. two column slots of one qkv buffer), cos and sin contiguous fp32 [L, d/2], row l for position l of
    each clip (LLaMA's rotate_half pairing: column j with column j + d/2).  Private, as _token_embed_fwd: the LLaMA
    layer (llama_modules.LlamaDecoderLayer) is its caller."""
    _chk(("q", q, bf16), ("k", k, bf16), ("cos", cos, f32), ("sin", sin, f32))
    for t, nm in ((q, "q"), (k, "k")):
        if t.shape != (B * L, H * d):
            raise _lib.IvbError(f"rope_qk: {nm} must be [B*L, H*d], got {tuple(t.shape)}")
    for t, nm in ((cos, "cos"), (sin, "sin")):
        if t.shape != (L, d // 2) or not t.is_contiguous():
            raise _lib.IvbError(f"rope_qk: {nm} must be a contiguous [L, d/2] = [{L}, {d // 2}], got {tuple(t.shape)}")
    _call("rope_qk", q, _rows2d(q, "q"), k, _rows2d(k, "k"), B, L, H, d, cos, sin)


def _dpe_ln_fwd(x, conv_w, conv_b, ln_w, ln_b, eps, N, T, H, W, out=None):
    """InternVideo-MM's extractor position conv + key LayerNorm (ivb_dpe_ln_fwd): x fp32 or bf16 [N*T*(1+H*W), C] (any
    row pitch), conv_w bf16 [C, 1, 3, 3, 3], conv_b / ln_w / ln_b bf16 [C] -> bf16 [N*T*(1+H*W), C]: each patch row
    LN(x + dpe(x)), each frame's cls row LN(x).  out (optional, any row pitch) must not overlap x: the kernel reads
    the neighbour rows that other CTAs write.  Private, as _rope_qk: InternVideo-MM's extractor
    (internvideo_mm.Transformer) is its caller."""
    _chk(("x", x, (f32, bf16)), ("conv_w", conv_w, bf16), ("conv_b", conv_b, bf16), ("ln_w", ln_w, bf16),
         ("ln_b", ln_b, bf16), ("out?", out, bf16))
    M, C = x.shape
    if M != N * T * (1 + H * W) or conv_w.shape != (C, 1, 3, 3, 3) or not conv_w.is_contiguous():
        raise _lib.IvbError(f"dpe_ln_fwd: x must be [N*T*(1+H*W), C] = [{N * T * (1 + H * W)}, C] and conv_w a "
                            f"contiguous [C, 1, 3, 3, 3], got {tuple(x.shape)}, {tuple(conv_w.shape)}")
    for t, nm in ((conv_b, "conv_b"), (ln_w, "ln_w"), (ln_b, "ln_b")):
        if t.shape != (C,) or not t.is_contiguous():
            raise _lib.IvbError(f"dpe_ln_fwd: {nm} must be a contiguous [C] = [{C}], got {tuple(t.shape)}")
    if out is None:
        out = torch.empty((M, C), device=x.device, dtype=bf16)
    elif out.shape != (M, C):
        raise _lib.IvbError(f"dpe_ln_fwd: out must be [{M}, {C}], got {tuple(out.shape)}")
    else:
        xs, xe = x.data_ptr(), x.data_ptr() + ((M - 1) * x.stride(0) + C) * x.element_size()
        os_, oe = out.data_ptr(), out.data_ptr() + ((M - 1) * out.stride(0) + C) * out.element_size()
        if xs < oe and os_ < xe:
            raise _lib.IvbError("dpe_ln_fwd: out must not overlap x (the kernel reads rows other CTAs write)")
    _call("dpe_ln_fwd", x, int(x.dtype == f32), _rows2d(x, "x"), conv_w, conv_b, ln_w, ln_b, float(eps), N, T, H, W, C,
          out, _rows2d(out, "out"))
    return out


def headaxis_attn_fwd(qkv, B, N, H, d, scale):
    """The VideoMAEv2 teacher's attention as the reference runs it (softmax over the H heads of each token, see
    include/ivb200.h).  qkv bf16 [B*N, 3*H*d] -> bf16 [B, H, N, d] contiguous."""
    _chk(("qkv", qkv, bf16))
    if qkv.shape != (B * N, 3 * H * d):
        raise _lib.IvbError(f"headaxis_attn_fwd: qkv must be [B*N, 3*H*d], got {tuple(qkv.shape)}")
    out = torch.empty((B, H, N, d), device=qkv.device, dtype=bf16)
    _call("headaxis_attn_fwd", qkv, _rows2d(qkv, "qkv"), B, N, H, d, float(scale), out)
    return out


def attn_bwd(q, k, v, out, dout, lse, B, n, H, d, scale, dq, dk, dv, rowscale=None, causal=False):
    """dq/dk/dv: preallocated bf16 2-D views [B*n, H*d] (e.g. the three slots of a [B*n, 3D] buffer).  rowscale: the
    forward's DropPath factors (attn_fwd): ivb_attn_bwd_plan writes zeros to the dropped clips' rows.  causal: the
    backward of attn_fwd(causal=True) (ivb_attn_bwd_causal; not with rowscale)."""
    rows = (("q", q), ("k", k), ("v", v), ("out", out), ("dout", dout), ("dq", dq), ("dk", dk), ("dv", dv))
    _chk(*((nm, t, bf16) for nm, t in rows), ("lse", lse, f32), ("rowscale?", rowscale, f32))
    _chk_rowscale("attn_bwd", rowscale, B * n)
    _chk_causal("attn_bwd", causal, rowscale)
    for nm, t in rows:
        if t.shape != (B * n, H * d):
            raise _lib.IvbError(f"attn_bwd: {nm} must be [B*n, H*d], got {tuple(t.shape)}")
    delta = torch.empty((int(_lib.load().ivb_attn_bwd_workspace_floats(B, n, H)),), device=q.device, dtype=f32)
    plan = () if rowscale is None else (rowscale,)
    _call("attn_bwd_causal" if causal else "attn_bwd_plan" if plan else "attn_bwd", q, _rows2d(q, "q"), k, _rows2d(k, "k"), v, _rows2d(v, "v"), out,
          _rows2d(out, "out"), dout, _rows2d(dout, "dout"), lse, delta, dq, _rows2d(dq, "dq"), dk, _rows2d(dk, "dk"), dv,
          _rows2d(dv, "dv"), B, n, H, d, float(scale), *plan, kind="attn_bwd",
          flops=(5.0 if causal else 10.0) * B * H * n * n * d)  # algorithmic: 5 GEMMs (SURVEY §8d: 2.5x forward)
    return dq, dk, dv


def _attn_fp8_pack(q, k, v, B, n, H, d):
    """Casts the attention operands to E4M3 for attn_fwd_fp8 (ivb_attn_fp8_pack); q, k, v as attn_fwd takes them.

    Returns (q8, k8, q_scale_inv, k_scale_inv, vt8, v_scale_inv): q8, k8 float8_e4m3fn [B*n, H*dp], dp = d rounded up
    to 32 (a head's columns: d values, then zeros), with one power-of-two scale per (token, head), q_scale_inv /
    k_scale_inv fp32 [B, H, ns] (ns: n rounded up to 64, the padding 0); vt8
    float8_e4m3fn [B, H, d, round_up(n, 16)] = V^T per (clip, head), keys n.. zero, with one scale per (clip, head,
    channel), v_scale_inv fp32 [B, H, d].  q8 and k8 are views of buffers whose row pitch is rounded up to 16.  Private,
    as _gemm_fp8_plan: the FP8-inference block forward (ops.block_forward with spec.attn_fp8) is its caller."""
    _chk(("q", q, bf16), ("k", k, bf16), ("v", v, bf16))
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if t.shape != (B * n, H * d):
            raise _lib.IvbError(f"attn_fp8_pack: {nm} must be [B*n, H*d], got {tuple(t.shape)}")
    dev, e4m3, dp = q.device, torch.float8_e4m3fn, (d + 31) // 32 * 32
    q8 = torch.empty((B * n, H * dp), device=dev, dtype=e4m3)
    k8 = torch.empty((B * n, H * dp), device=dev, dtype=e4m3)
    ns = int(_lib.load().ivb_attn_fp8_scale_pitch(n))
    sq = torch.empty((B, H, ns), device=dev, dtype=f32)
    sk = torch.empty((B, H, ns), device=dev, dtype=f32)
    vt8 = torch.empty((B, H, d, _pad16(n)), device=dev, dtype=e4m3)
    sv = torch.empty((B, H, d), device=dev, dtype=f32)
    _call("attn_fp8_pack", q, _rows2d(q, "q"), k, _rows2d(k, "k"), v, _rows2d(v, "v"), B, n, H, d, q8, k8,
          q8.stride(0), sq, sk, vt8, vt8.stride(2), sv, kind="fp8_quantize")
    return q8, k8, sq, sk, vt8, sv


def _attn_fwd_fp8(q8, k8, q_scale_inv, k_scale_inv, vt8, v_scale_inv, B, n, H, d, scale, out=None):
    """softmax(scale q k^T) v on the FP8 tensor cores from attn_fp8_pack's outputs (ivb_attn_fwd_fp8): bf16 [B*n, H*d]
    (out: an optional bf16 [B*n, H*d] view, any row pitch).  Inference only: no lse, no backward.  Private, as
    _attn_fp8_pack."""
    _chk(("q8", q8, torch.float8_e4m3fn), ("k8", k8, torch.float8_e4m3fn), ("q_scale_inv", q_scale_inv, f32),
         ("k_scale_inv", k_scale_inv, f32), ("vt8", vt8, torch.float8_e4m3fn), ("v_scale_inv", v_scale_inv, f32),
         ("out?", out, bf16))
    ns = int(_lib.load().ivb_attn_fp8_scale_pitch(n))
    dp = (d + 31) // 32 * 32
    if q8.shape != (B * n, H * dp) or k8.stride() != q8.stride() or k8.shape != q8.shape:
        raise _lib.IvbError(f"attn_fwd_fp8: q8 and k8 must be [B*n, H*round_up(d, 32)] with one row pitch, got "
                            f"{tuple(q8.shape)}, {tuple(k8.shape)}")
    for nm, t, shape in (("q_scale_inv", q_scale_inv, (B, H, ns)), ("k_scale_inv", k_scale_inv, (B, H, ns)),
                         ("v_scale_inv", v_scale_inv, (B, H, d))):
        if t.shape != shape or not t.is_contiguous():
            raise _lib.IvbError(f"attn_fwd_fp8: {nm} must be a contiguous {list(shape)}, got {tuple(t.shape)}")
    if vt8.shape[:3] != (B, H, d) or vt8.stride(3) != 1 or vt8.stride(1) != d * vt8.stride(2) or \
            vt8.stride(0) != H * vt8.stride(1):
        raise _lib.IvbError(f"attn_fwd_fp8: vt8 must be [B, H, d, >= n] with packed B, H, d, got {tuple(vt8.shape)}")
    if out is None:
        out = torch.empty((B * n, H * d), device=q8.device, dtype=bf16)
    _call("attn_fwd_fp8", q8, k8, _rows2d(q8, "q8"), q_scale_inv, k_scale_inv, vt8, vt8.stride(2), v_scale_inv, out,
          _rows2d(out, "out"), B, n, H, d, float(scale), kind="attn_fwd", flops=4.0 * B * H * n * n * d)
    return out


def _chk_rowscale(fn, rowscale, rows):
    """The attention plan calls read rowscale[b*n] for every clip b (the block-scaled cast every row): a contiguous fp32
    [B*n]."""
    if rowscale is not None and (rowscale.shape != (rows,) or not rowscale.is_contiguous()):
        raise _lib.IvbError(f"{fn}: rowscale must be a contiguous [B*n] = [{rows}], got {tuple(rowscale.shape)}")


# ----------------------------------------------------------------------------------------- token front-end
def visible_indices(mask, n_keep):
    """mask: bool/uint8 [B, N] on CUDA (True = masked). Returns (idx int32 [B, n_keep], err int32[1])."""
    _chk(("mask", mask, (torch.bool, torch.uint8)))
    m = mask.contiguous()
    if m.dtype == torch.bool:
        m = m.view(torch.uint8)
    B, N = m.shape
    idx = torch.empty((B, n_keep), device=m.device, dtype=i32)
    err = torch.zeros((1,), device=m.device, dtype=i32)
    _call("visible_indices", m, B, N, n_keep, idx, err)
    return idx, err


def im2col_visible(video, idx, j0, rows_per_clip, tubelet, patch, kpad):
    _chk(("video", video, bf16), ("idx", idx, i32))
    if not video.is_contiguous():
        raise _lib.IvbError("im2col_visible: video must be contiguous [B,C,T,H,W]")
    B, C, T, H, W = video.shape
    cols = torch.empty((B * rows_per_clip, kpad), device=video.device, dtype=bf16)
    _call("im2col_visible", video, idx, idx.stride(0), j0, rows_per_clip, B, C, T, H, W, tubelet, patch, kpad, cols)
    return cols


def _im2col_prenorm(video, idx, j0, rows_per_clip, tubelet, patch, kpad, weight, eps=1e-6):
    """im2col_visible's rows through the patch embed's pre-conv RMSNorm (ivb_im2col_prenorm): weight bf16 [C*t*p*p] in
    the reference's (t hp wp c) order.  Returns (cols bf16 [B*rows_per_clip, kpad], rstd fp32 [B*rows_per_clip])."""
    _chk(("video", video, bf16), ("idx", idx, i32), ("weight", weight, bf16))
    if not video.is_contiguous():
        raise _lib.IvbError("im2col_prenorm: video must be contiguous [B,C,T,H,W]")
    B, C, T, H, W = video.shape
    cols = torch.empty((B * rows_per_clip, kpad), device=video.device, dtype=bf16)
    rstd = torch.empty((B * rows_per_clip,), device=video.device, dtype=f32)
    _call("im2col_prenorm", video, idx, idx.stride(0), j0, rows_per_clip, B, C, T, H, W, tubelet, patch, kpad, weight,
          float(eps), cols, rstd)
    return cols, rstd


def _prenorm_wgrad(video, idx, j0, rows_per_clip, tubelet, patch, kpad, rstd, dcols, dweight=None):
    """Weight gradient of im2col_prenorm's RMSNorm from dcols bf16 [B*rows_per_clip, >=kpad], the gradient of its rows
    (ivb_prenorm_wgrad, fixed order).  dweight: optional fp32 [C*t*p*p] accumulator.  Returns dweight."""
    _chk(("video", video, bf16), ("idx", idx, i32), ("rstd", rstd, f32), ("dcols", dcols, bf16),
         ("dweight?", dweight, f32))
    if not video.is_contiguous():
        raise _lib.IvbError("prenorm_wgrad: video must be contiguous [B,C,T,H,W]")
    B, C, T, H, W = video.shape
    if dweight is None:
        dweight = torch.zeros((C * tubelet * patch * patch,), device=video.device, dtype=f32)
    _call("prenorm_wgrad", video, idx, idx.stride(0), j0, rows_per_clip, B, C, T, H, W, tubelet, patch, kpad, rstd,
          dcols, _rows2d(dcols, "dcols"), dweight)
    return dweight


def gather_add(src, src_bstride, table, idx, idx_bstride, idx_off, B, rows, D, out, out_bstride):
    _chk(("src?", src, f32), ("table?", table, bf16), ("idx?", idx, i32), ("out", out, (f32, bf16)))
    _call("gather_add", src, src_bstride, table, idx, idx_bstride, idx_off, B, rows, D, out, int(out.dtype == f32),
          out_bstride)
    return out


def scatter_add(g, g_bstride, idx, idx_bstride, idx_off, B, rows, D, table_grad):
    _chk(("g", g, (f32, bf16)), ("idx?", idx, i32), ("table_grad", table_grad, f32))
    _call("scatter_add", g, int(g.dtype == f32), g_bstride, idx, idx_bstride, idx_off, B, rows, D, table_grad)
    return table_grad


def _token_embed_fwd(ids, table, pos):
    """The text tower's token embedding (ivb_token_embed_fwd): ids int64 [B, L], table bf16 [V, D], pos bf16 [L, D] ->
    (fp32 residual stream [B*L, D] = table[ids] + pos, int32[1] device flag: 1 + the first row seen with an id outside
    [0, V), else 0).  Private, as _attn_fp8_pack: ops.TokenEmbedFn is its caller."""
    _chk(("ids", ids, torch.int64), ("table", table, bf16), ("pos", pos, bf16))
    B, L = ids.shape
    V, D = table.shape
    if pos.shape != (L, D) or not (ids.is_contiguous() and table.is_contiguous() and pos.is_contiguous()):
        raise _lib.IvbError(f"token_embed_fwd: contiguous ids [B, L], table [V, D] and pos [L, D] needed, got "
                            f"{tuple(ids.shape)}, {tuple(table.shape)}, {tuple(pos.shape)}")
    out = torch.empty((B * L, D), device=ids.device, dtype=f32)
    err = torch.zeros((1,), device=ids.device, dtype=i32)
    _call("token_embed_fwd", ids, B, L, table, V, pos, D, out, out.stride(0), err)
    return out, err


def _token_embed_bwd(ids, g, V):
    """Backward of _token_embed_fwd (ivb_token_embed_bwd): ids int64 [B, L], g fp32 [B*L, D] -> (dtable fp32 [V, D],
    zero in the rows of ids not present, dpos fp32 [L, D]), each summed in a fixed order.  Private, as
    _token_embed_fwd."""
    _chk(("ids", ids, torch.int64), ("g", g, f32))
    B, L = ids.shape
    D = g.shape[1]
    if g.shape[0] != B * L or not ids.is_contiguous():
        raise _lib.IvbError(f"token_embed_bwd: g must be [B*L, D] for contiguous ids [B, L], got {tuple(g.shape)}")
    dtable = torch.zeros((V, D), device=g.device, dtype=f32)
    dpos = torch.empty((L, D), device=g.device, dtype=f32)
    ws = torch.empty((int(_lib.load().ivb_token_embed_bwd_workspace_ints(V, B, L)),), device=g.device, dtype=i32)
    _call("token_embed_bwd", ids, B, L, g, _rows2d(g, "g"), V, D, dtable, dpos, ws)
    return dtable, dpos


# ----------------------------------------------------------------------------------------- heads / losses
def ln_l2_fwd(z, weight, bias, eps=1e-5, want_out=True, target=None, loss_sum=None):
    _chk(("z", z, bf16), ("weight", weight, bf16), ("bias", bias, bf16), ("target?", target, (f32, bf16)),
         ("loss_sum?", loss_sum, f32))
    M, Cc = z.shape
    out = torch.empty((M, Cc), device=z.device, dtype=bf16) if want_out else None
    stats = torch.empty((M, 3), device=z.device, dtype=f32)
    _call("ln_l2_fwd", z, _rows2d(z, "z"), weight, bias, float(eps), M, Cc, out, Cc if want_out else 0, stats, target,
          int(target is not None and target.dtype == f32), _rows2d(target, "target"), loss_sum)
    return out, stats


def ln_l2_bwd(z, weight, bias, stats, dout, gscale_host=1.0, gscale_dev=None, dweight=None, dbias=None):
    _chk(("z", z, bf16), ("weight", weight, bf16), ("bias", bias, bf16), ("stats", stats, f32),
         ("dout", dout, (f32, bf16)), ("gscale_dev?", gscale_dev, f32), ("dweight?", dweight, f32),
         ("dbias?", dbias, f32))
    M, Cc = z.shape
    dz = torch.empty((M, Cc), device=z.device, dtype=bf16)
    _call("ln_l2_bwd", z, _rows2d(z, "z"), weight, bias, stats, M, Cc, dout, int(dout.dtype == f32),
          _rows2d(dout, "dout"), float(gscale_host), gscale_dev, dz, Cc, dweight, dbias)
    return dz


def vtc_loss_fwd(cosm, idx, temp, temp_dev=None):
    """temp_dev: optional CUDA fp32[1] temperature (overrides the host float `temp`)."""
    _chk(("cosm", cosm, f32), ("idx", idx, torch.int64), ("temp_dev?", temp_dev, f32))
    G = cosm.shape[0]
    lse_r = torch.empty((G,), device=cosm.device, dtype=f32)
    lse_c = torch.empty((G,), device=cosm.device, dtype=f32)
    loss = torch.zeros((1,), device=cosm.device, dtype=f32)
    _call("vtc_loss_fwd", cosm, idx, G, float(temp), temp_dev, lse_r, lse_c, loss)
    return loss, lse_r, lse_c


def vtc_loss_bwd(cosm, idx, temp, lse_r, lse_c, gscale_host=1.0, gscale_dev=None, temp_dev=None):
    _chk(("cosm", cosm, f32), ("idx", idx, torch.int64), ("lse_r", lse_r, f32), ("lse_c", lse_c, f32),
         ("gscale_dev?", gscale_dev, f32), ("temp_dev?", temp_dev, f32))
    G = cosm.shape[0]
    dcos = torch.empty((G, G), device=cosm.device, dtype=bf16)
    dtemp = torch.zeros((1,), device=cosm.device, dtype=f32)
    _call("vtc_loss_bwd", cosm, idx, G, float(temp), temp_dev, lse_r, lse_c, float(gscale_host), gscale_dev, dcos, dtemp)
    return dcos, dtemp


def l2norm_rows_fwd(x):
    _chk(("x", x, (f32, bf16)))
    M, Cc = x.shape
    out = torch.empty((M, Cc), device=x.device, dtype=bf16)
    inv = torch.empty((M,), device=x.device, dtype=f32)
    _call("l2norm_rows_fwd", x, int(x.dtype == f32), _rows2d(x, "x"), M, Cc, out, Cc, inv)
    return out, inv


def l2norm_rows_bwd(dy, xn, inv):
    _chk(("dy", dy, f32), ("xn", xn, bf16), ("inv", inv, f32))
    M, Cc = dy.shape
    dx = torch.empty((M, Cc), device=dy.device, dtype=f32)
    _call("l2norm_rows_bwd", dy, _rows2d(dy, "dy"), xn, _rows2d(xn, "xn"), inv, M, Cc, dx, Cc)
    return dx


def pixel_targets(video, masked_idx, n_mask, tubelet, patch, normalize, mean3, std3):
    _chk(("video", video, bf16), ("masked_idx", masked_idx, i32), ("mean3", mean3, f32), ("std3", std3, f32))
    B, C, T, H, W = video.shape
    labels = torch.empty((B * n_mask, tubelet * patch * patch * C), device=video.device, dtype=f32)
    _call("pixel_targets", video.contiguous(), masked_idx, n_mask, B, C, T, H, W, tubelet, patch, int(normalize),
          mean3, std3, labels)
    return labels


def mse_loss(pred, label, loss_sum, gscale_host=0.0, gscale_dev=None, dpred=None):
    _chk(("pred", pred, bf16), ("label", label, f32), ("loss_sum?", loss_sum, f32), ("gscale_dev?", gscale_dev, f32),
         ("dpred?", dpred, bf16))
    _call("mse_loss", pred, label, pred.numel(), loss_sum, float(gscale_host), gscale_dev, dpred)
    return loss_sum


def adamw_step(master, exp_avg, exp_avg_sq, grad, param_bf16, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
               grad_scale_dev=None, dyn_lr_step=None):
    _chk(("master", master, f32), ("exp_avg", exp_avg, f32), ("exp_avg_sq", exp_avg_sq, f32),
         ("grad", grad, (f32, bf16)), ("param_bf16", param_bf16, bf16), ("grad_scale_dev?", grad_scale_dev, f32),
         ("dyn_lr_step?", dyn_lr_step, f32))
    _call("adamw_step", master, exp_avg, exp_avg_sq, grad, int(grad.dtype == f32), param_bf16, master.numel(),
          float(lr), float(beta1), float(beta2), float(eps), float(wd), int(step), float(grad_scale), grad_scale_dev,
          dyn_lr_step)


def pool_attn_fwd(q, k, v, B, n, H, d, scale):
    """q: [B, H*d]; k, v: [B*n, H*d] 2-D views. Returns (out bf16 [B, H*d], probs fp32 [B,H,n])."""
    _chk(("q", q, bf16), ("k", k, bf16), ("v", v, bf16))
    out = torch.empty((B, H * d), device=q.device, dtype=bf16)
    probs = torch.empty((B, H, n), device=q.device, dtype=f32)
    _call("pool_attn_fwd", q, k, _rows2d(k, "k"), v, _rows2d(v, "v"), B, n, H, d, float(scale), out, probs)
    return out, probs


def pool_attn_bwd(q, k, v, probs, dout, B, n, H, d, scale):
    _chk(("q", q, bf16), ("k", k, bf16), ("v", v, bf16), ("probs", probs, f32), ("dout", dout, bf16))
    dq = torch.empty((B, H * d), device=q.device, dtype=bf16)
    dk = torch.empty((B * n, H * d), device=q.device, dtype=bf16)
    dv = torch.empty((B * n, H * d), device=q.device, dtype=bf16)
    _call("pool_attn_bwd", q, k, _rows2d(k, "k"), v, _rows2d(v, "v"), probs, dout, B, n, H, d, float(scale), dq, dk,
          H * d, dv, H * d)
    return dq, dk, dv
