"""float64 reference of ivb_gemm_bf16 (every fused epilogue and flag) and the per-element error metric the GEMM tests
use.

gemm_ref takes the arguments of lowlevel.gemm and returns, for every output the call writes, the float64 reference
and a per-element tolerance `scale`: the error the kernel may make before the output is rounded to its storage
format.  elem_errors adds half an ulp of that format and divides, so a value of 1 is the edge of what a correct
kernel can produce.  `scale` is built from the pieces of the computation:
  - the fp32 accumulation and epilogue adds: 2^-24 * (sqrt(ceil(K / 16)) sum_k |A(m,k)| |B(n,k)| + |bias| + |old out0|),
    times the epilogue's sensitivity to its input (|gelu'(h)| for GELU, |rowscale * gamma| for RESID, |aux| for
    GELU_BWD).  The tensor cores add one k16 step's products into the fp32 accumulator at a time; on the H100 the
    accumulation error measured up to 4x 2^-24 sum |a b| at K = 592 and 15x at K = 6144, about sqrt(K / 16) times it;
  - the documented error of the GELU form the kernel evaluates: Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7 on erf,
    7.5e-8 on Phi) for the erf form, the tanh.approx.f32 instruction (relative error about 2^-11) for the tanh form;
  - a few fp32 ulps of the transcendental evaluation and of the epilogue's own multiplies.
Everything runs in float64 on the inputs' device, in row chunks, so the full-size shapes of the training step fit.
"""
from __future__ import annotations

import math

import torch

EPI_BF16, EPI_F32, EPI_BIAS_GELU, EPI_RESID, EPI_GELU_BWD = 0, 1, 2, 3, 4
FLAG_GELU_TANH, FLAG_ACCUM, FLAG_1CTA, FLAG_2CTA, FLAG_GELU_SAVE_GRAD, FLAG_PINGPONG = 1, 2, 4, 8, 16, 32

U24 = 2.0 ** -24            # fp32 unit roundoff
EVAL = 2.0 ** -21           # fp32 evaluation of the GELU functions (MUFU.EX2 / MUFU.RCP, a handful of roundings)
AS_PHI = 7.5e-8             # Abramowitz-Stegun 7.1.26: |erf error| <= 1.5e-7, so |Phi error| <= 7.5e-8
TANH_REL = 2.0 ** -10.987   # tanh.approx.f32 (MUFU.TANH): maximum relative error
TANH_C, TANH_A = math.sqrt(2.0 / math.pi), 0.044715
ROW_CHUNK = 2048


# ---------------------------------------------------------------- GELU forms in float64
def gelu_erf(h):
    """h * Phi(h), its first and second derivative, and the absolute error of the kernel's A-S evaluation of each."""
    phi = torch.exp(-0.5 * h * h) / math.sqrt(2.0 * math.pi)
    cdf = 0.5 * torch.special.erfc(-h / math.sqrt(2.0))
    f, d1, d2 = h * cdf, cdf + h * phi, phi * (2.0 - h * h)
    e0 = AS_PHI * h.abs() + EVAL * (f.abs() + h.abs() * d1.abs())
    e1 = AS_PHI + EVAL * (d1.abs() + h.abs() * d2.abs())
    return f, d1, d2, e0, e1


def gelu_tanh(h):
    """0.5 h (1 + tanh(u)), u = sqrt(2/pi) (h + 0.044715 h^3): value, derivatives and the error bounds of the kernel's
    evaluation through tanh.approx.f32 (an error dt in t moves the value by 0.5|h| dt and the derivative by
    dt (0.5 + |h t| u'))."""
    u = TANH_C * (h + TANH_A * h * h * h)
    t = torch.tanh(u)
    s = 1.0 - t * t
    du = TANH_C * (1.0 + 3.0 * TANH_A * h * h)
    d2u = 6.0 * TANH_A * TANH_C * h
    f = 0.5 * h * (1.0 + t)
    d1 = 0.5 * (1.0 + t) + 0.5 * h * s * du
    d2 = s * du - h * t * s * du * du + 0.5 * h * s * d2u
    dt = TANH_REL * t.abs()
    e0 = 0.5 * h.abs() * dt + EVAL * (f.abs() + h.abs() * d1.abs())
    e1 = dt * (0.5 + (h * t).abs() * du) + EVAL * (d1.abs() + h.abs() * d2.abs())
    return f, d1, d2, e0, e1


def gelu_form(flags):
    return gelu_tanh if flags & FLAG_GELU_TANH else gelu_erf


# ---------------------------------------------------------------- the reference
def _operand_rows(a, a_t, rows):
    """float64 [len(rows), K] rows of the A operand."""
    return (a[:, rows].t() if a_t else a[rows]).double()


def gemm_ref(a, b, *, a_t=False, b_t=False, epi=EPI_BF16, flags=0, out0=None, out1=None, bias=None, gamma=None,
             aux=None, rowscale=None, rows=None):
    """float64 reference of lowlevel.gemm with the same arguments.  `out0` is only read (its values BEFORE the call)
    under FLAG_ACCUM; `out1` only says whether the call writes it.  rows: a slice of output rows (default all).
    Returns a list of (ref, scale) pairs, float64 [rows, N]: out0, then out1 when the call writes it."""
    M = a.shape[1] if a_t else a.shape[0]
    N = b.shape[1] if b_t else b.shape[0]
    r0, r1, _ = (rows or slice(None)).indices(M)
    bm = (b if b_t else b.t()).double()                                    # [K, N]
    bm_abs = bm.abs()
    with_out1 = out1 is not None and epi in (EPI_BIAS_GELU, EPI_RESID)
    res = [torch.empty((r1 - r0, N), dtype=torch.float64, device=a.device) for _ in range(2 if with_out1 else 1)]
    scl = [torch.empty_like(r) for r in res]
    bias64 = bias.double() if bias is not None else None
    for c0 in range(r0, r1, ROW_CHUNK):
        c1 = min(c0 + ROW_CHUNK, r1)
        rs = slice(c0, c1)
        am = _operand_rows(a, a_t, rs)
        v = am @ bm                                                        # exact-ish: bf16 products, fp64 sums
        base = (am.abs() @ bm_abs) * math.sqrt(math.ceil(am.shape[1] / 16))
        if bias64 is not None:
            v = v + bias64
            base = base + bias64.abs()
        outs = _epilogue(v, base * U24, epi, flags, out0, bias64, gamma, aux, rowscale, rs, with_out1)
        for i, (r, s) in enumerate(outs):
            res[i][c0 - r0:c1 - r0] = r
            scl[i][c0 - r0:c1 - r0] = s
    return list(zip(res, scl))


def _epilogue(v, acc_err, epi, flags, out0, bias, gamma, aux, rowscale, rs, with_out1):
    """v = acc + bias (float64) and its fp32 error bound for rows rs -> [(ref, scale) of out0, (of out1)]."""
    if epi in (EPI_BF16, EPI_F32):
        if flags & FLAG_ACCUM:
            old = out0[rs].double()
            return [(v + old, acc_err + U24 * old.abs())]
        return [(v, acc_err)]
    if epi == EPI_BIAS_GELU:
        f, d1, d2, e0, e1 = gelu_form(flags)(v)
        out = [(f, d1.abs() * acc_err + e0)]
        if with_out1:
            out.append((d1, d2.abs() * acc_err + e1) if flags & FLAG_GELU_SAVE_GRAD else (v, acc_err))
        return out
    if epi == EPI_RESID:
        res = aux[rs].double()
        g = gamma.double() if gamma is not None else torch.ones_like(v[0])
        r = rowscale[rs].double()[:, None] if rowscale is not None else torch.ones_like(v[:, :1])
        branch = r * g * v
        # the kernel forms (gamma * rs) and y in fp32, then one fma with the residual
        out = [(res + branch, (r * g).abs() * acc_err + 2 * U24 * branch.abs())]
        if with_out1:
            out.append((v, acc_err))
        return out
    if epi == EPI_GELU_BWD:
        h = aux[rs].double()
        if flags & FLAG_GELU_SAVE_GRAD:
            d, e = h, torch.zeros_like(h)
        else:
            _, d, d2, _, e = gelu_form(flags)(h)
        return [(v * d, d.abs() * acc_err + v.abs() * e + U24 * (v * d).abs())]
    raise ValueError(f"unknown epilogue {epi}")


# ---------------------------------------------------------------- the metric
def half_ulp(dtype, ref):
    """Half an ulp of `dtype` (bfloat16 or float32) at |ref|; flush-to-zero below the smallest normal."""
    mant = {torch.bfloat16: 8, torch.float32: 24}[dtype]
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - mant) + 2.0 ** -126


def elem_errors(got, ref, scale):
    """|got - ref| / tol per element, tol = scale + half an ulp of got's format at |ref|.  NaN in got reads as inf."""
    err = (got.double() - ref).abs() / (scale + half_ulp(got.dtype, ref))
    return torch.nan_to_num(err, nan=math.inf)


def binned_bias(got, ref, scale, h, width=0.25, lo=-8.0, hi=8.0, min_count=256):
    """Mean signed distance of got from the correctly rounded reference, in units of elem_errors' tolerance and signed
    like ref, over the elements whose pre-activation h lies in each `width`-wide bin of [lo, hi).  A correct kernel
    returns the rounded reference or, near a rounding tie, a neighbour on either side, so a bin's mean stays near 0;
    an error of the GELU evaluation that is systematic in h tips the ties one way, however far inside the per-element
    tolerance each element stays.  Bins with fewer than min_count elements are left out.
    Returns (largest |bin mean|, the bin's lower edge)."""
    tol = scale + half_ulp(got.dtype, ref)
    s = ((got.double() - ref.to(got.dtype).double()) * torch.sign(ref) / tol).reshape(-1)
    nb = int(round((hi - lo) / width))
    idx = torch.floor((h.double().reshape(-1) - lo) / width)
    keep = (idx >= 0) & (idx < nb) & torch.isfinite(s)
    idx = idx[keep].long()
    sums = torch.zeros(nb, dtype=torch.float64, device=s.device).index_add_(0, idx, s[keep])
    cnt = torch.zeros(nb, dtype=torch.float64, device=s.device).index_add_(0, idx, torch.ones_like(s[keep]))
    mean = torch.where(cnt >= min_count, sums / cnt.clamp_min(1), torch.zeros_like(sums)).abs()
    i = int(mean.argmax())
    return float(mean[i]), lo + i * width


def worst(errs, bm=128, bn=128, row0=0):
    """The largest error of an [M, N] error tensor and where it lies in the kernel's tiling: bm x bn tiles (256 x bn
    for the CTA pair), 64-row warpgroup bands and 16-column epilogue chunks.  row0: first row of `errs` in the
    output (for row-chunked checks).  Returns (value, description)."""
    M, N = errs.shape
    flat = int(errs.argmax())
    m, n = flat // N + row0, flat % N
    Mt = row0 + M
    tm, tn = m // bm, n // bn
    ragged = []
    if Mt % bm and tm == (Mt - 1) // bm:
        ragged.append(f"last row tile ({Mt % bm} rows)")
    if N % bn and tn == (N - 1) // bn:
        ragged.append(f"last column tile ({N % bn} cols)")
    where = (f"element ({m}, {n}): tile ({tm}, {tn}) of {bm}x{bn}, warpgroup band {(m % bm) // 64} "
             f"(rows {m // 64 * 64}..{m // 64 * 64 + 63}), epilogue chunk {(n % bn) // 16} "
             f"(cols {n // 16 * 16}..{n // 16 * 16 + 15})" + (", " + ", ".join(ragged) if ragged else ""))
    return float(errs.reshape(-1)[flat]), where
