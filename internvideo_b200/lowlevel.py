"""Thin tensor-level wrappers over the C ABI (no autograd): pointer/shape plumbing only.

Every function checks that its tensors are CUDA tensors of the expected dtype and raises otherwise;
nothing here computes on the CPU.
"""
from __future__ import annotations

import torch

from . import _lib

EPI_BF16, EPI_F32, EPI_BIAS_GELU, EPI_RESID, EPI_GELU_BWD = 0, 1, 2, 3, 4
FLAG_GELU_TANH, FLAG_ACCUM, FLAG_1CTA, FLAG_2CTA, FLAG_GELU_SAVE_GRAD = 1, 2, 4, 8, 16

bf16 = torch.bfloat16
f32 = torch.float32


def _lib_():
    return _lib.load()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _chk(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise _lib.IvbError(f"{name}: expected a CUDA tensor (ivb200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.IvbError(f"{name}: expected dtype {dtype}, got {t.dtype}")


def _rows2d(t, name):
    """View as 2-D [rows, cols] with unit inner stride; returns (tensor, ld)."""
    if t.dim() != 2:
        raise _lib.IvbError(f"{name}: expected 2-D tensor, got {tuple(t.shape)}")
    if t.stride(1) != 1:
        raise _lib.IvbError(f"{name}: inner stride must be 1")
    return t.stride(0)


def launch_count() -> int:
    return int(_lib_().ivb_launch_count())


def reset_launch_count() -> None:
    _lib_().ivb_reset_launch_count()


def set_default_2cta(enable: bool) -> None:
    _lib_().ivb_set_default_2cta(int(bool(enable)))


def device_check() -> None:
    _lib.check(_lib_().ivb_device_check(), "ivb_device_check")


# ----------------------------------------------------------------------------------------- GEMM
def gemm(a, b, *, a_t=False, b_t=False, epi=EPI_BF16, flags=0, out0=None, out1=None, bias=None,
         gamma=None, aux=None, rowscale=None, tile_n=0):
    """D[M,N] = epi(sum_k A(m,k) B(n,k)).

    a_t=False: `a` is [M,K]; a_t=True: `a` is [K,M] (MN-major operand).
    b_t=False: `b` is [N,K]; b_t=True: `b` is [K,N].
    """
    _chk(a, bf16, "a"); _chk(b, bf16, "b")
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
    out_dtype = f32 if epi in (EPI_F32, EPI_RESID) else bf16
    if out0 is None:
        out0 = torch.empty((M, N), device=a.device, dtype=out_dtype)
    _chk(out0, out_dtype, "out0")
    ld0 = _rows2d(out0, "out0")
    ld1 = 0
    if out1 is not None:
        _chk(out1, bf16, "out1"); ld1 = _rows2d(out1, "out1")
    _chk(bias, bf16, "bias"); _chk(gamma, bf16, "gamma")
    ldaux = 0
    if aux is not None:
        _chk(aux, f32 if epi == EPI_RESID else bf16, "aux")
        ldaux = _rows2d(aux, "aux")
    prof = _PROF[0]
    if prof is not None:
        ev0 = torch.cuda.Event(enable_timing=True); ev0.record()
    rc = _lib_().ivb_gemm_bf16(_p(a), int(a_t), lda, _p(b), int(b_t), ldb, M, N, K, epi, flags,
                               _p(out0), ld0, _p(out1), ld1, _p(bias), _p(gamma), _p(aux), ldaux,
                               _p(rowscale), tile_n, _stream())
    _lib.check(rc, "ivb_gemm_bf16")
    if prof is not None:
        ev1 = torch.cuda.Event(enable_timing=True); ev1.record()
        prof.records.append((ev0, ev1, 2.0 * M * N * K, "gemm"))
    return out0


_PROF = [None]


class GemmProfiler:
    """CUDA-event timing of every tensor-core launch (GEMMs, attention forward / backward) on the launching stream
    (bench.py roofline).  Records (start, stop, algorithmic flops, kind)."""

    def __init__(self):
        self.records = []
        self.count = 0

    def enable(self):
        _PROF[0] = self

    def disable(self):
        _PROF[0] = None

    def totals(self, kind="gemm"):
        """(total algorithmic FLOPs, total milliseconds) over the recorded launches of `kind`."""
        torch.cuda.synchronize()
        fl = ms = 0.0
        cnt = 0
        for e0, e1, f, k in self.records:
            if k != kind:
                continue
            fl += f
            ms += e0.elapsed_time(e1)
            cnt += 1
        if kind == "gemm":
            self.count = cnt
        return fl, ms


def _prof_begin():
    prof = _PROF[0]
    if prof is None:
        return None
    ev0 = torch.cuda.Event(enable_timing=True); ev0.record()
    return ev0


def _prof_end(ev0, flops, kind):
    if ev0 is not None and _PROF[0] is not None:
        ev1 = torch.cuda.Event(enable_timing=True); ev1.record()
        _PROF[0].records.append((ev0, ev1, flops, kind))


# ----------------------------------------------------------------------------------------- norms
def norm_fwd(x, weight, bias=None, eps=1e-6, layernorm=False, out=None, want_stats=True):
    """x: [M,D] fp32 or bf16 (row stride arbitrary). Returns (y bf16, mean|None, rstd)."""
    if x.dtype not in (f32, bf16):
        raise _lib.IvbError("norm_fwd: x must be fp32 or bf16")
    _chk(x, x.dtype, "x"); _chk(weight, bf16, "weight"); _chk(bias, bf16, "bias")
    ldx = _rows2d(x, "x")
    M, D = x.shape
    if out is None:
        out = torch.empty((M, D), device=x.device, dtype=bf16)
    _chk(out, bf16, "out")
    ldy = _rows2d(out, "out")
    rstd = torch.empty((M,), device=x.device, dtype=f32) if want_stats else None
    mean = torch.empty((M,), device=x.device, dtype=f32) if (want_stats and layernorm) else None
    rc = _lib_().ivb_norm_fwd(_p(x), int(x.dtype == f32), ldx, _p(weight), _p(bias), float(eps),
                              int(layernorm), M, D, _p(out), ldy, _p(mean), _p(rstd), _stream())
    _lib.check(rc, "ivb_norm_fwd")
    return out, mean, rstd


def rmsnorm_pair_fwd(qkv, D, w0, w1, out, eps=1e-6, want_stats=True):
    """RMSNorm of the q and k column slices ([:, :D] and [:, D:2D]) of a bf16 [M, >=2D] projection buffer in one
    launch -> out[:, :D], out[:, D:2D] (bf16 [M, >=2D]).  Returns rstd fp32 [M, 2] (or None)."""
    _chk(qkv, bf16, "qkv"); _chk(w0, bf16, "w0"); _chk(w1, bf16, "w1"); _chk(out, bf16, "out")
    M = qkv.shape[0]
    rstd = torch.empty((M, 2), device=qkv.device, dtype=f32) if want_stats else None
    rc = _lib_().ivb_rmsnorm_pair_fwd(_p(qkv), _rows2d(qkv, "qkv"), D, _p(w0), _p(w1), float(eps), M, D,
                                      _p(out), _rows2d(out, "out"), D, _p(rstd), _stream())
    _lib.check(rc, "ivb_rmsnorm_pair_fwd")
    return rstd


def rmsnorm_pair_bwd(dqk, qkv, D, w0, w1, rstd, dw0=None, dw1=None):
    """Backward of rmsnorm_pair_fwd, IN PLACE on the gradient buffer: dqk[:, :D] / dqk[:, D:2D] hold d(normed q/k) on
    entry and d(q/k) on return.  dw0/dw1: optional fp32 [D] accumulators."""
    _chk(dqk, bf16, "dqk"); _chk(qkv, bf16, "qkv"); _chk(rstd, f32, "rstd"); _chk(dw0, f32, "dw0"); _chk(dw1, f32, "dw1")
    M = qkv.shape[0]
    rc = _lib_().ivb_rmsnorm_pair_bwd(_p(dqk), _rows2d(dqk, "dqk"), D, _p(qkv), _rows2d(qkv, "qkv"), D, _p(w0), _p(w1),
                                      _p(rstd), M, D, _p(dqk), _rows2d(dqk, "dqk"), D, _p(dw0), _p(dw1), _stream())
    _lib.check(rc, "ivb_rmsnorm_pair_bwd")
    return dqk


def norm_bwd(dy, x, weight, mean, rstd, layernorm=False, dx_in=None, dx_out=None,
             dx_dtype=f32, dweight=None, dbias=None):
    _chk(dy, bf16, "dy"); _chk(weight, bf16, "weight")
    _chk(rstd, f32, "rstd"); _chk(mean, f32, "mean")
    _chk(dweight, f32, "dweight"); _chk(dbias, f32, "dbias"); _chk(dx_in, f32, "dx_in")
    M, D = x.shape
    lddy = _rows2d(dy, "dy"); ldx = _rows2d(x, "x")
    if dx_out is None:
        dx_out = torch.empty((M, D), device=x.device, dtype=dx_dtype)
    lddx = _rows2d(dx_out, "dx_out")
    lddx_in = _rows2d(dx_in, "dx_in") if dx_in is not None else 0
    rc = _lib_().ivb_norm_bwd(_p(dy), lddy, _p(x), int(x.dtype == f32), ldx, _p(weight), _p(mean),
                              _p(rstd), int(layernorm), M, D, _p(dx_in), lddx_in, _p(dx_out),
                              int(dx_out.dtype == f32), lddx, _p(dweight), _p(dbias), _stream())
    _lib.check(rc, "ivb_norm_bwd")
    return dx_out


def rmsnorm_bwd_layerscale(dy, x, weight, rstd, dx_in, ybr, gamma, dweight, dgamma, dcolsum, rowscale=None):
    """RMSNorm backward on the fp32 stream fused with the LayerScale backward of the preceding branch (one pass over the
    rows).  Returns (dx fp32 [M,D], dyb bf16 [M,D])."""
    _chk(dy, bf16, "dy"); _chk(x, f32, "x"); _chk(weight, bf16, "weight"); _chk(rstd, f32, "rstd"); _chk(dx_in, f32, "dx_in")
    _chk(ybr, bf16, "ybr"); _chk(gamma, bf16, "gamma"); _chk(dweight, f32, "dweight"); _chk(dgamma, f32, "dgamma")
    _chk(dcolsum, f32, "dcolsum"); _chk(rowscale, f32, "rowscale")
    M, D = x.shape
    dx = torch.empty((M, D), device=x.device, dtype=f32)
    dyb = torch.empty((M, D), device=x.device, dtype=bf16)
    rc = _lib_().ivb_rmsnorm_bwd_layerscale(_p(dy), _rows2d(dy, "dy"), _p(x), _rows2d(x, "x"), _p(weight), _p(rstd), M, D,
                                            _p(dx_in), _rows2d(dx_in, "dx_in") if dx_in is not None else 0, _p(dx), D,
                                            _p(dweight), _p(ybr), _rows2d(ybr, "ybr"), _p(gamma), _p(rowscale), _p(dyb), D,
                                            _p(dgamma), _p(dcolsum), _stream())
    _lib.check(rc, "ivb_rmsnorm_bwd_layerscale")
    return dx, dyb


def layerscale_bwd(dx, y, gamma, dgamma=None, dcolsum=None, out=None, rowscale=None):
    _chk(dx, f32, "dx"); _chk(y, bf16, "y"); _chk(gamma, bf16, "gamma")
    _chk(dgamma, f32, "dgamma"); _chk(dcolsum, f32, "dcolsum")
    M, D = dx.shape
    if out is None:
        out = torch.empty((M, D), device=dx.device, dtype=bf16)
    rc = _lib_().ivb_layerscale_bwd(_p(dx), _rows2d(dx, "dx"), _p(y),
                                    _rows2d(y, "y") if y is not None else 0, _p(gamma), M, D,
                                    _p(out), _rows2d(out, "out"), _p(dgamma), _p(dcolsum), _p(rowscale), _stream())
    _lib.check(rc, "ivb_layerscale_bwd")
    return out


def colsum(x, out=None):
    _chk(x, bf16, "x")
    M, N = x.shape
    if out is None:
        out = torch.zeros((N,), device=x.device, dtype=f32)
    _chk(out, f32, "out")
    rc = _lib_().ivb_colsum_bf16(_p(x), _rows2d(x, "x"), M, N, _p(out), _stream())
    _lib.check(rc, "ivb_colsum_bf16")
    return out


# ----------------------------------------------------------------------------------------- attention
def attn_fwd(q, k, v, B, n, H, d, scale, out=None, want_lse=True):
    """q/k/v: 2-D views [B*n, H*d] (any row pitch) of the projection buffers."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _chk(t, bf16, nm)
        if t.shape != (B * n, H * d):
            raise _lib.IvbError(f"attn_fwd: {nm} must be [B*n, H*d], got {tuple(t.shape)}")
    if out is None:
        out = torch.empty((B * n, H * d), device=q.device, dtype=bf16)
    lse = torch.empty((B, H, n), device=q.device, dtype=f32) if want_lse else None
    ev0 = _prof_begin()
    rc = _lib_().ivb_attn_fwd(_p(q), _rows2d(q, "q"), _p(k), _rows2d(k, "k"), _p(v), _rows2d(v, "v"),
                              _p(out), _rows2d(out, "out"), _p(lse), B, n, H, d, float(scale), _stream())
    _lib.check(rc, "ivb_attn_fwd")
    _prof_end(ev0, 4.0 * B * H * n * n * d, "attn_fwd")          # QK^T + PV
    return out, lse


def headaxis_attn_fwd(qkv, B, N, H, d, scale):
    """The VideoMAEv2 teacher's attention as the reference runs it (softmax over the H heads of each token, see
    include/ivb200.h).  qkv bf16 [B*N, 3*H*d] -> bf16 [B, H, N, d] contiguous."""
    _chk(qkv, bf16, "qkv")
    if qkv.shape != (B * N, 3 * H * d):
        raise _lib.IvbError(f"headaxis_attn_fwd: qkv must be [B*N, 3*H*d], got {tuple(qkv.shape)}")
    out = torch.empty((B, H, N, d), device=qkv.device, dtype=bf16)
    rc = _lib_().ivb_headaxis_attn_fwd(_p(qkv), _rows2d(qkv, "qkv"), B, N, H, d, float(scale), _p(out), _stream())
    _lib.check(rc, "ivb_headaxis_attn_fwd")
    return out


def attn_bwd(q, k, v, out, dout, lse, B, n, H, d, scale, dq, dk, dv):
    """dq/dk/dv: preallocated bf16 2-D views [B*n, H*d] (e.g. the three slots of a [B*n, 3D] buffer)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (dout, "dout"), (dq, "dq"), (dk, "dk"), (dv, "dv")):
        _chk(t, bf16, nm)
        if t.shape != (B * n, H * d):
            raise _lib.IvbError(f"attn_bwd: {nm} must be [B*n, H*d], got {tuple(t.shape)}")
    _chk(lse, f32, "lse")
    delta = torch.empty((int(_lib_().ivb_attn_bwd_workspace_floats(B, n, H)),), device=q.device, dtype=f32)
    ev0 = _prof_begin()
    rc = _lib_().ivb_attn_bwd(_p(q), _rows2d(q, "q"), _p(k), _rows2d(k, "k"), _p(v), _rows2d(v, "v"),
                              _p(out), _rows2d(out, "out"), _p(dout), _rows2d(dout, "dout"), _p(lse),
                              _p(delta), _p(dq), _rows2d(dq, "dq"), _p(dk), _rows2d(dk, "dk"),
                              _p(dv), _rows2d(dv, "dv"), B, n, H, d, float(scale), _stream())
    _lib.check(rc, "ivb_attn_bwd")
    _prof_end(ev0, 10.0 * B * H * n * n * d, "attn_bwd")         # algorithmic: 5 GEMMs (SURVEY §8d: 2.5x forward)
    return dq, dk, dv


# ----------------------------------------------------------------------------------------- token front-end
i32 = torch.int32


def visible_indices(mask, n_keep):
    """mask: bool/uint8 [B, N] on CUDA (True = masked). Returns (idx int32 [B, n_keep], err int32[1])."""
    if not mask.is_cuda:
        raise _lib.IvbError("visible_indices: mask must be a CUDA tensor")
    m = mask.contiguous()
    if m.dtype == torch.bool:
        m = m.view(torch.uint8)
    if m.dtype != torch.uint8:
        raise _lib.IvbError("visible_indices: mask must be bool or uint8")
    B, N = m.shape
    idx = torch.empty((B, n_keep), device=m.device, dtype=i32)
    err = torch.zeros((1,), device=m.device, dtype=i32)
    rc = _lib_().ivb_visible_indices(_p(m), B, N, n_keep, _p(idx), _p(err), _stream())
    _lib.check(rc, "ivb_visible_indices")
    return idx, err


def im2col_visible(video, idx, j0, rows_per_clip, tubelet, patch, kpad):
    _chk(video, bf16, "video"); _chk(idx, i32, "idx")
    if not video.is_contiguous():
        raise _lib.IvbError("im2col_visible: video must be contiguous [B,C,T,H,W]")
    B, C, T, H, W = video.shape
    cols = torch.empty((B * rows_per_clip, kpad), device=video.device, dtype=bf16)
    rc = _lib_().ivb_im2col_visible(_p(video), _p(idx), idx.stride(0), j0, rows_per_clip, B, C, T, H, W,
                                    tubelet, patch, kpad, _p(cols), _stream())
    _lib.check(rc, "ivb_im2col_visible")
    return cols


def gather_add(src, src_bstride, table, idx, idx_bstride, idx_off, B, rows, D, out, out_bstride):
    _chk(src, f32, "src"); _chk(table, bf16, "table"); _chk(idx, i32, "idx")
    if out.dtype not in (f32, bf16) or not out.is_cuda:
        raise _lib.IvbError("gather_add: out must be a CUDA fp32/bf16 tensor")
    rc = _lib_().ivb_gather_add(_p(src), src_bstride, _p(table), _p(idx), idx_bstride, idx_off, B, rows, D,
                                _p(out), int(out.dtype == f32), out_bstride, _stream())
    _lib.check(rc, "ivb_gather_add")
    return out


def scatter_add(g, g_bstride, idx, idx_bstride, idx_off, B, rows, D, table_grad):
    _chk(table_grad, f32, "table_grad"); _chk(idx, i32, "idx")
    if g.dtype not in (f32, bf16) or not g.is_cuda:
        raise _lib.IvbError("scatter_add: g must be a CUDA fp32/bf16 tensor")
    rc = _lib_().ivb_scatter_add(_p(g), int(g.dtype == f32), g_bstride, _p(idx), idx_bstride, idx_off, B,
                                 rows, D, _p(table_grad), _stream())
    _lib.check(rc, "ivb_scatter_add")
    return table_grad


# ----------------------------------------------------------------------------------------- heads / losses
def ln_l2_fwd(z, weight, bias, eps=1e-5, want_out=True, target=None, loss_sum=None):
    _chk(z, bf16, "z"); _chk(weight, bf16, "weight"); _chk(bias, bf16, "bias"); _chk(loss_sum, f32, "loss_sum")
    M, Cc = z.shape
    out = torch.empty((M, Cc), device=z.device, dtype=bf16) if want_out else None
    stats = torch.empty((M, 3), device=z.device, dtype=f32)
    tf32 = 0
    ldt = 0
    if target is not None:
        if target.dtype not in (f32, bf16):
            raise _lib.IvbError("ln_l2_fwd: target must be fp32/bf16")
        _chk(target, target.dtype, "target")
        tf32 = int(target.dtype == f32); ldt = _rows2d(target, "target")
    rc = _lib_().ivb_ln_l2_fwd(_p(z), _rows2d(z, "z"), _p(weight), _p(bias), float(eps), M, Cc, _p(out),
                               Cc if want_out else 0, _p(stats), _p(target), tf32, ldt, _p(loss_sum), _stream())
    _lib.check(rc, "ivb_ln_l2_fwd")
    return out, stats


def ln_l2_bwd(z, weight, bias, stats, dout, gscale_host=1.0, gscale_dev=None, dweight=None, dbias=None):
    _chk(z, bf16, "z"); _chk(stats, f32, "stats"); _chk(dweight, f32, "dweight"); _chk(dbias, f32, "dbias")
    _chk(gscale_dev, f32, "gscale_dev")
    if dout.dtype not in (f32, bf16) or not dout.is_cuda:
        raise _lib.IvbError("ln_l2_bwd: dout must be CUDA fp32/bf16")
    M, Cc = z.shape
    dz = torch.empty((M, Cc), device=z.device, dtype=bf16)
    rc = _lib_().ivb_ln_l2_bwd(_p(z), _rows2d(z, "z"), _p(weight), _p(bias), _p(stats), M, Cc, _p(dout),
                               int(dout.dtype == f32), _rows2d(dout, "dout"), float(gscale_host),
                               _p(gscale_dev), _p(dz), Cc, _p(dweight), _p(dbias), _stream())
    _lib.check(rc, "ivb_ln_l2_bwd")
    return dz


def vtc_loss_fwd(cosm, idx, temp, temp_dev=None):
    """temp_dev: optional CUDA fp32[1] temperature (overrides the host float `temp`)."""
    _chk(cosm, f32, "cos"); _chk(idx, torch.int64, "idx"); _chk(temp_dev, f32, "temp_dev")
    G = cosm.shape[0]
    lse_r = torch.empty((G,), device=cosm.device, dtype=f32)
    lse_c = torch.empty((G,), device=cosm.device, dtype=f32)
    loss = torch.zeros((1,), device=cosm.device, dtype=f32)
    rc = _lib_().ivb_vtc_loss_fwd(_p(cosm), _p(idx), G, float(temp), _p(temp_dev), _p(lse_r), _p(lse_c), _p(loss), _stream())
    _lib.check(rc, "ivb_vtc_loss_fwd")
    return loss, lse_r, lse_c


def vtc_loss_bwd(cosm, idx, temp, lse_r, lse_c, gscale_host=1.0, gscale_dev=None, temp_dev=None):
    _chk(temp_dev, f32, "temp_dev")
    G = cosm.shape[0]
    dcos = torch.empty((G, G), device=cosm.device, dtype=bf16)
    dtemp = torch.zeros((1,), device=cosm.device, dtype=f32)
    rc = _lib_().ivb_vtc_loss_bwd(_p(cosm), _p(idx), G, float(temp), _p(temp_dev), _p(lse_r), _p(lse_c), float(gscale_host),
                                  _p(gscale_dev), _p(dcos), _p(dtemp), _stream())
    _lib.check(rc, "ivb_vtc_loss_bwd")
    return dcos, dtemp


def l2norm_rows_fwd(x):
    if x.dtype not in (f32, bf16) or not x.is_cuda:
        raise _lib.IvbError("l2norm_rows_fwd: x must be CUDA fp32/bf16")
    M, Cc = x.shape
    out = torch.empty((M, Cc), device=x.device, dtype=bf16)
    inv = torch.empty((M,), device=x.device, dtype=f32)
    rc = _lib_().ivb_l2norm_rows_fwd(_p(x), int(x.dtype == f32), _rows2d(x, "x"), M, Cc, _p(out), Cc, _p(inv), _stream())
    _lib.check(rc, "ivb_l2norm_rows_fwd")
    return out, inv


def l2norm_rows_bwd(dy, xn, inv):
    _chk(dy, f32, "dy"); _chk(xn, bf16, "xn"); _chk(inv, f32, "inv")
    M, Cc = dy.shape
    dx = torch.empty((M, Cc), device=dy.device, dtype=f32)
    rc = _lib_().ivb_l2norm_rows_bwd(_p(dy), _rows2d(dy, "dy"), _p(xn), _rows2d(xn, "xn"), _p(inv), M, Cc, _p(dx), Cc, _stream())
    _lib.check(rc, "ivb_l2norm_rows_bwd")
    return dx


def pixel_targets(video, masked_idx, n_mask, tubelet, patch, normalize, mean3, std3):
    _chk(video, bf16, "video"); _chk(masked_idx, i32, "masked_idx"); _chk(mean3, f32, "mean3"); _chk(std3, f32, "std3")
    B, C, T, H, W = video.shape
    labels = torch.empty((B * n_mask, tubelet * patch * patch * C), device=video.device, dtype=f32)
    rc = _lib_().ivb_pixel_targets(_p(video.contiguous()), _p(masked_idx), n_mask, B, C, T, H, W, tubelet, patch,
                                   int(normalize), _p(mean3), _p(std3), _p(labels), _stream())
    _lib.check(rc, "ivb_pixel_targets")
    return labels


def mse_loss(pred, label, loss_sum, gscale_host=0.0, gscale_dev=None, dpred=None):
    _chk(pred, bf16, "pred"); _chk(label, f32, "label"); _chk(loss_sum, f32, "loss_sum"); _chk(dpred, bf16, "dpred")
    rc = _lib_().ivb_mse_loss(_p(pred), _p(label), pred.numel(), _p(loss_sum), float(gscale_host), _p(gscale_dev), _p(dpred), _stream())
    _lib.check(rc, "ivb_mse_loss")
    return loss_sum


def adamw_step(master, exp_avg, exp_avg_sq, grad, param_bf16, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
               grad_scale_dev=None, dyn_lr_step=None):
    _chk(master, f32, "master"); _chk(exp_avg, f32, "exp_avg"); _chk(exp_avg_sq, f32, "exp_avg_sq"); _chk(param_bf16, bf16, "param")
    _chk(dyn_lr_step, f32, "dyn_lr_step")
    if grad.dtype not in (f32, bf16) or not grad.is_cuda:
        raise _lib.IvbError("adamw_step: grad must be CUDA fp32/bf16")
    rc = _lib_().ivb_adamw_step(_p(master), _p(exp_avg), _p(exp_avg_sq), _p(grad), int(grad.dtype == f32),
                                _p(param_bf16), master.numel(), float(lr), float(beta1), float(beta2), float(eps),
                                float(wd), int(step), float(grad_scale), _p(grad_scale_dev), _p(dyn_lr_step),
                                _stream())
    _lib.check(rc, "ivb_adamw_step")


def pool_attn_fwd(q, k, v, B, n, H, d, scale):
    """q: [B, H*d]; k, v: [B*n, H*d] 2-D views. Returns (out bf16 [B, H*d], probs fp32 [B,H,n])."""
    _chk(q, bf16, "q"); _chk(k, bf16, "k"); _chk(v, bf16, "v")
    out = torch.empty((B, H * d), device=q.device, dtype=bf16)
    probs = torch.empty((B, H, n), device=q.device, dtype=f32)
    rc = _lib_().ivb_pool_attn_fwd(_p(q), _p(k), _rows2d(k, "k"), _p(v), _rows2d(v, "v"), B, n, H, d, float(scale),
                                   _p(out), _p(probs), _stream())
    _lib.check(rc, "ivb_pool_attn_fwd")
    return out, probs


def pool_attn_bwd(q, k, v, probs, dout, B, n, H, d, scale):
    _chk(dout, bf16, "dout"); _chk(probs, f32, "probs")
    dq = torch.empty((B, H * d), device=q.device, dtype=bf16)
    dk = torch.empty((B * n, H * d), device=q.device, dtype=bf16)
    dv = torch.empty((B * n, H * d), device=q.device, dtype=bf16)
    rc = _lib_().ivb_pool_attn_bwd(_p(q), _p(k), _rows2d(k, "k"), _p(v), _rows2d(v, "v"), _p(probs), _p(dout), B, n,
                                   H, d, float(scale), _p(dq), _p(dk), H * d, _p(dv), H * d, _stream())
    _lib.check(rc, "ivb_pool_attn_bwd")
    return dq, dk, dv


# ----------------------------------------------------------------------------------------- op profiler (dev tool)
_OPPROF = [None]


class OpProfiler:
    """CUDA-event timing of every lowlevel op, in situ (warm caches, real overlap)."""

    def __init__(self):
        self.records = []

    def enable(self):
        _OPPROF[0] = self

    def disable(self):
        _OPPROF[0] = None

    def summary(self):
        torch.cuda.synchronize()
        agg = {}
        for name, e0, e1 in self.records:
            c, t = agg.get(name, (0, 0.0))
            agg[name] = (c + 1, t + e0.elapsed_time(e1))
        return sorted(agg.items(), key=lambda kv: -kv[1][1])


def _timed(fn, namer=None):
    import functools

    @functools.wraps(fn)
    def w(*a, **k):
        prof = _OPPROF[0]
        if prof is None:
            return fn(*a, **k)
        e0 = torch.cuda.Event(enable_timing=True); e0.record()
        r = fn(*a, **k)
        e1 = torch.cuda.Event(enable_timing=True); e1.record()
        prof.records.append((namer(*a, **k) if namer else fn.__name__, e0, e1))
        return r
    return w


def _gemm_name(a, b, *, a_t=False, b_t=False, epi=EPI_BF16, **_):
    M = a.shape[1] if a_t else a.shape[0]
    K = a.shape[0] if a_t else a.shape[1]
    N = b.shape[1] if b_t else b.shape[0]
    return f"gemm[{'T' if a_t else 'N'}{'T' if b_t else 'N'} epi{epi}] {M}x{N}x{K}"


gemm = _timed(gemm, _gemm_name)
for _n in ("norm_fwd", "norm_bwd", "layerscale_bwd", "colsum", "attn_fwd", "attn_bwd", "visible_indices",
           "im2col_visible", "gather_add", "scatter_add", "ln_l2_fwd", "ln_l2_bwd", "vtc_loss_fwd", "vtc_loss_bwd",
           "l2norm_rows_fwd", "l2norm_rows_bwd", "pixel_targets", "mse_loss", "adamw_step"):
    globals()[_n] = _timed(globals()[_n])
