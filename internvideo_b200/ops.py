"""torch.autograd.Function wrappers over the C ABI (lowlevel.py): the differentiable op surface.

Everything here runs on the H100 through libivb200.so; there is no eager/PyTorch fallback for the
compute (tiny O(D) vector glue such as `gamma * colsum` uses torch elementwise ops on CUDA tensors).
Activations are bf16, the residual stream is fp32, parameters are bf16 (the reference's bf16
DeepSpeed mode converts the whole model: engines/engine_for_pretraining.py:128, SURVEY App.B-18).
"""
from __future__ import annotations

import torch

from . import lowlevel as ll

bf16, f32 = torch.bfloat16, torch.float32


def _need_cuda_bf16(t, name):
    if not t.is_cuda:
        raise ll._lib.IvbError(f"{name}: ivb200 ops need CUDA tensors (no CPU fallback)")
    if t.dtype != bf16:
        raise ll._lib.IvbError(f"{name}: expected bf16, got {t.dtype}")


def _pdt(g, p):
    """cast a gradient to its parameter's dtype (vector grads are accumulated in fp32)."""
    return None if g is None else g.to(p.dtype)


# ------------------------------------------------------------------------------------------ Linear
class LinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM (nn.Linear: internvideo2_pretrain.py:61-77,195,211,356)."""

    @staticmethod
    def forward(ctx, x, w, b, out_f32=False):
        _need_cuda_bf16(x, "x"); _need_cuda_bf16(w, "weight")
        x2 = x.reshape(-1, x.shape[-1])
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        y = ll.gemm(x2, w, bias=b, epi=ll.EPI_F32 if out_f32 else ll.EPI_BF16)
        ctx.save_for_backward(x2, w)
        ctx.has_bias = b is not None
        ctx.bias_dtype = b.dtype if b is not None else None
        ctx.in_shape = x.shape
        return y.reshape(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.dtype != bf16:
            dy2 = dy2.to(bf16)
        if dy2.stride(-1) != 1 or (dy2.stride(0) % 8) != 0:
            dy2 = dy2.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ll.gemm(dy2, w, b_t=True).reshape(ctx.in_shape)
        if ctx.needs_input_grad[1]:
            dw = ll.gemm(dy2, x2, a_t=True, b_t=True)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = ll.colsum(dy2).to(ctx.bias_dtype)
        return dx, dw, db, None


def linear(x, w, b=None, out_f32=False):
    return LinearFn.apply(x, w, b, out_f32)


class LinearGeluFn(torch.autograd.Function):
    """g = GELU(x W^T + b) with the activation fused in the GEMM epilogue (Mlp.fc1+act :239-240)."""

    @staticmethod
    def forward(ctx, x, w, b, gelu_tanh=False):
        _need_cuda_bf16(x, "x")
        x2 = x.reshape(-1, x.shape[-1])
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        h = torch.empty((x2.shape[0], w.shape[0]), device=x.device, dtype=bf16)
        flags = ll.FLAG_GELU_TANH if gelu_tanh else 0
        g = ll.gemm(x2, w, bias=b, epi=ll.EPI_BIAS_GELU, flags=flags, out1=h)
        ctx.save_for_backward(x2, w, h)
        ctx.flags = flags
        ctx.has_bias = b is not None
        ctx.bias_dtype = b.dtype if b is not None else None
        ctx.in_shape = x.shape
        return g.reshape(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dg):
        x2, w, h = ctx.saved_tensors
        dg2 = dg.reshape(-1, dg.shape[-1]).contiguous()
        # dh = dg * gelu'(h): run as an elementwise epilogue of an identity-free pass is not
        # available, so use the GEMM-fused variant only when dg itself comes from a GEMM; here:
        dh = _gelu_bwd(dg2, h, ctx.flags)
        dx = ll.gemm(dh, w, b_t=True).reshape(ctx.in_shape) if ctx.needs_input_grad[0] else None
        dw = ll.gemm(dh, x2, a_t=True, b_t=True) if ctx.needs_input_grad[1] else None
        db = ll.colsum(dh).to(ctx.bias_dtype) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return dx, dw, db, None


def _gelu_bwd(dg, h, flags):
    """dh = dg * gelu'(h) (small heads only; the block path fuses this into the fc2 dgrad GEMM)."""
    hf = h.float()
    if flags & ll.FLAG_GELU_TANH:
        u = 0.7978845608028654 * (hf + 0.044715 * hf ** 3)
        t = torch.tanh(u)
        d = 0.5 * (1 + t) + 0.5 * hf * (1 - t * t) * 0.7978845608028654 * (1 + 3 * 0.044715 * hf * hf)
    else:
        d = 0.5 * (1 + torch.erf(hf * 0.7071067811865476)) + hf * 0.3989422804014327 * torch.exp(-0.5 * hf * hf)
    return (dg.float() * d).to(bf16)


# ------------------------------------------------------------------------------------------ norms
class NormFn(torch.autograd.Function):
    """RMSNorm (:117-128) / LayerNorm (:525) rows; x fp32 or bf16 -> bf16."""

    @staticmethod
    def forward(ctx, x, w, b, eps, layernorm):
        if not x.is_cuda:
            raise ll._lib.IvbError("norm: ivb200 ops need CUDA tensors (no CPU fallback)")
        x2 = x.reshape(-1, x.shape[-1])
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        y, mean, rstd = ll.norm_fwd(x2, w, b, eps=eps, layernorm=layernorm)
        ctx.save_for_backward(x2, w, mean if mean is not None else rstd, rstd)
        ctx.layernorm = layernorm
        ctx.has_bias = b is not None
        ctx.in_shape = x.shape
        ctx.x_dtype = x.dtype
        return y.reshape(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, w, mean, rstd = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.dtype != bf16:
            dy2 = dy2.to(bf16)
        if dy2.stride(-1) != 1:
            dy2 = dy2.contiguous()
        D = x2.shape[1]
        dw = torch.zeros(D, device=x2.device, dtype=f32) if ctx.needs_input_grad[1] else None
        db = torch.zeros(D, device=x2.device, dtype=f32) if (ctx.layernorm and ctx.has_bias) else None
        dx = ll.norm_bwd(dy2, x2, w, mean if ctx.layernorm else None, rstd, layernorm=ctx.layernorm,
                         dx_dtype=ctx.x_dtype, dweight=dw, dbias=db)
        return (dx.reshape(ctx.in_shape), _pdt(dw, w), _pdt(db, w) if db is not None else None, None, None)


def rmsnorm(x, w, eps=1e-6):
    return NormFn.apply(x, w, None, eps, False)


def layernorm(x, w, b, eps=1e-5):
    return NormFn.apply(x, w, b, eps, True)


# ------------------------------------------------------------------------------------------ attention
class AttnFn(torch.autograd.Function):
    """softmax(scale q k^T) v over packed projection buffers (FlashAttention.forward, flash_attention_class.py:27-50)."""

    @staticmethod
    def forward(ctx, q, k, v, B, n, H, d, scale):
        out, lse = ll.attn_fwd(q, k, v, B, n, H, d, scale)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.dims = (B, n, H, d, scale)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        B, n, H, d, scale = ctx.dims
        D = H * d
        dqkv = torch.empty((B * n, 3 * D), device=q.device, dtype=bf16)
        dout = dout.contiguous()
        ll.attn_bwd(q, k, v, out, dout, lse, B, n, H, d, scale, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])
        return dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:], None, None, None, None, None


class PoolAttnFn(torch.autograd.Function):
    """One-query-per-clip cross attention of the AttentionPoolingBlock (internvideo2_pretrain.py:61-76)."""

    @staticmethod
    def forward(ctx, q, k, v, B, n, H, d, scale):
        q = q.contiguous()
        out, probs = ll.pool_attn_fwd(q, k, v, B, n, H, d, scale)
        ctx.save_for_backward(q, k, v, probs)
        ctx.dims = (B, n, H, d, scale)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, probs = ctx.saved_tensors
        B, n, H, d, scale = ctx.dims
        dq, dk, dv = ll.pool_attn_bwd(q, k, v, probs, dout.contiguous().to(bf16), B, n, H, d, scale)
        return dq, dk, dv, None, None, None, None, None


# ------------------------------------------------------------------------------------------ fused ViT block
def block_forward(x, dims, params, rs1=None, rs2=None, save=True):
    """One spatio-temporal ViT block over the fp32 residual stream [B*n, D] (Block.forward,
    internvideo2_pretrain.py:279-297):

      n1 = RMSNorm(x) ; qkv = n1 Wqkv^T ; (q,k) = RMSNorm_C(q), RMSNorm_C(k) ; a = attn(q,k,v)
      x1 = x + rs1 * g1 * (a Wp^T + bp)                [LayerScale + DropPath + residual fused in the GEMM epilogue]
      n2 = RMSNorm(x1) ; h = n2 W1^T + b1 ; g = GELU(h) [fused epilogue] ; x2 = x1 + rs2 * g2 * (g W2^T + b2)

    14 kernels.  save=True also writes what the backward needs (pre-LayerScale branch outputs, GELU') and returns
    it; save=False is the inference / recompute-later form (frozen towers, activation checkpointing): nothing
    extra is written.  Returns (x2, saved | None)."""
    B, n, H, gelu_tanh = dims[:4]
    n1w, qkvw, qkvb, qnw, knw, projw, projb, g1, n2w, fc1w, fc1b, fc2w, fc2b, g2 = params
    M, D = x.shape
    d = D // H
    if x.dtype != f32 or not x.is_cuda:
        raise ll._lib.IvbError("block_forward: residual stream must be a CUDA fp32 tensor [B*n, D]")
    n1, _, rstd1 = ll.norm_fwd(x, n1w, want_stats=save)
    qkv = ll.gemm(n1, qkvw, bias=qkvb)
    rq = rk = None
    if qnw is not None:
        qkn = torch.empty((M, 2 * D), device=x.device, dtype=bf16)
        if D <= 1536:      # q-norm and k-norm in ONE launch; rq holds rstd [M, 2] for both
            rq = ll.rmsnorm_pair_fwd(qkv, D, qnw, knw, qkn, want_stats=save)
        else:
            _, _, rq = ll.norm_fwd(qkv[:, :D], qnw, out=qkn[:, :D], want_stats=save)
            _, _, rk = ll.norm_fwd(qkv[:, D:2 * D], knw, out=qkn[:, D:], want_stats=save)
        q, k = qkn[:, :D], qkn[:, D:]
    else:
        qkn = None
        q, k = qkv[:, :D], qkv[:, D:2 * D]
    a, lse = ll.attn_fwd(q, k, qkv[:, 2 * D:], B, n, H, d, d ** -0.5, want_lse=save)
    y1 = torch.empty((M, D), device=x.device, dtype=bf16) if (g1 is not None and save) else None
    x1 = ll.gemm(a, projw, epi=ll.EPI_RESID, bias=projb, gamma=g1, aux=x, out1=y1, rowscale=rs1)
    n2, _, rstd2 = ll.norm_fwd(x1, n2w, want_stats=save)
    Hd = fc1w.shape[0]
    flags = ll.FLAG_GELU_TANH if gelu_tanh else 0
    h = None
    if save:
        # h holds gelu'(pre-activation): the only thing the backward needs of it (FLAG_GELU_SAVE_GRAD)
        h = torch.empty((M, Hd), device=x.device, dtype=bf16)
        flags |= ll.FLAG_GELU_SAVE_GRAD
    g = ll.gemm(n2, fc1w, epi=ll.EPI_BIAS_GELU, flags=flags, bias=fc1b, out1=h)
    y2 = torch.empty((M, D), device=x.device, dtype=bf16) if (g2 is not None and save) else None
    x2 = ll.gemm(g, fc2w, epi=ll.EPI_RESID, bias=fc2b, gamma=g2, aux=x1, out1=y2, rowscale=rs2)
    if not save:
        return x2, None
    return x2, (n1, qkv, qkn, a, lse, rstd1, rq, rk, x1, y1, n2, rstd2, h, g, y2, flags)


def block_forward_ln_infer(x, B, n, H, scale, params, head_axis_attention=False):
    """Inference-only LayerNorm pre-norm block of the VideoMAEv2 teacher (videomae.py:104-132; attention with q/v
    bias :62-101, erf GELU, optional gamma_1/gamma_2) over the fp32 residual stream [B*n, D]: 9 kernels,
    LayerScale + residual fused in the GEMM epilogues, nothing saved.  params = (n1w, n1b, eps1, qkvw, qkvb, projw,
    projb, g1, n2w, n2b, eps2, fc1w, fc1b, fc2w, fc2b, g2).  head_axis_attention=True reproduces the reference's
    flash_attn_func call on [B,H,N,d] tensors (softmax over the heads of each token); False is token-axis attention."""
    n1w, n1b, eps1, qkvw, qkvb, projw, projb, g1, n2w, n2b, eps2, fc1w, fc1b, fc2w, fc2b, g2 = params
    M, D = x.shape
    d = D // H
    if x.dtype != f32 or not x.is_cuda:
        raise ll._lib.IvbError("block_forward_ln_infer: residual stream must be a CUDA fp32 tensor [B*n, D]")
    with torch.no_grad():
        n1, _, _ = ll.norm_fwd(x, n1w, n1b, eps=eps1, layernorm=True, want_stats=False)
        qkv = ll.gemm(n1, qkvw, bias=qkvb)
        if head_axis_attention:
            # the reference's call (videomae.py:94-97) attends over the heads of each token and reinterprets the
            # [B, H, N, d] result as [B, N, H*d]: reproduced bit-for-layout
            a = ll.headaxis_attn_fwd(qkv, B, n, H, d, scale).reshape(M, D)
        else:
            a, _ = ll.attn_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B, n, H, d, scale, want_lse=False)
        x1 = ll.gemm(a, projw, epi=ll.EPI_RESID, bias=projb, gamma=g1, aux=x)
        n2, _, _ = ll.norm_fwd(x1, n2w, n2b, eps=eps2, layernorm=True, want_stats=False)
        g = ll.gemm(n2, fc1w, epi=ll.EPI_BIAS_GELU, bias=fc1b)
        return ll.gemm(g, fc2w, epi=ll.EPI_RESID, bias=fc2b, gamma=g2, aux=x1)


def block_backward(x, saved, dims, tensors, P, dx2, rs1, rs2):
    """Backward of block_forward: 26 kernels.  `tensors` are the parameter tensors as autograd handed them back,
    `P` the nn.Parameter objects (gradient sink).  Returns (dx0, per-parameter gradients | None when the sink took them)."""
    n1, qkv, qkn, a, lse, rstd1, rq, rk, x1, y1, n2, rstd2, h, g, y2, flags = saved
    n1w, qkvw, qkvb, qnw, knw, projw, projb, g1, n2w, fc1w, fc1b, fc2w, fc2b, g2 = tensors
    B, n, H = dims[:3]
    M, D = x.shape
    d = D // H
    Hd = fc1w.shape[0]
    dx2 = dx2.contiguous()
    if dx2.dtype != f32:
        dx2 = dx2.float()
    # Gradient sink (engine.PretrainEngine): when every parameter of the block lives in the engine's
    # flat gradient buffer, the wgrad GEMMs accumulate straight into it (FLAG_ACCUM epilogue) and the
    # O(D) gradients land with ONE fused add per block — no autograd AccumulateGrad kernels (16 per
    # block, each re-reading and re-writing the gradient).
    sink = _common_sink(P)
    small = (("g2", g2, D), ("fc2b", fc2b, D), ("n2w", n2w, D), ("g1", g1, D), ("projb", projb, D),
             ("qnw", qnw, D), ("knw", knw, D), ("n1w", n1w, D), ("fc1b", fc1b, Hd), ("qkvb", qkvb, 3 * D))
    seg, vec, span, base = _plan_small(small, P, sink, x.device)
    if sink is not None and span is None:
        sink = None           # small parameters not contiguous in the flat buffer: autograd path
    dg2, dcs2, dn2w, dg1, dcs1 = seg["g2"], seg["fc2b"], seg["n2w"], seg["g1"], seg["projb"]
    dqnw, dknw, dn1w, dfc1b, dqkvb = seg["qnw"], seg["knw"], seg["n1w"], seg["fc1b"], seg["qkvb"]
    pn1w, pqkvw, pqkvb, pqnw, pknw, pprojw, pprojb, pg1, pn2w, pfc1w, pfc1b, pfc2w, pfc2b, pg2 = P

    def wgrad(dy, act, param):
        if sink is None:
            return ll.gemm(dy, act, a_t=True, b_t=True)
        ll.gemm(dy, act, a_t=True, b_t=True, out0=param.grad, flags=ll.FLAG_ACCUM)
        sink.grad_written(param)
        return None
    # ---- MLP branch
    dy2 = ll.layerscale_bwd(dx2, y2, g2, dg2 if g2 is not None else None, dcs2, rowscale=rs2)
    dfc2w = wgrad(dy2, g, pfc2w)
    dh = ll.gemm(dy2, fc2w, b_t=True, epi=ll.EPI_GELU_BWD, flags=flags, aux=h)
    ll.colsum(dh, out=dfc1b)
    dfc1w = wgrad(dh, n2, pfc1w)
    dn2 = ll.gemm(dh, fc1w, b_t=True)
    # ---- attention branch
    if g1 is not None and D <= 1536 and M >= 1024:
        # norm2 backward fused with the attention branch's LayerScale backward: the gradient of the residual
        # stream is produced and consumed in one pass over the rows
        dx1, dy1 = ll.rmsnorm_bwd_layerscale(dn2, x1, n2w, rstd2, dx2, y1, g1, dn2w, dg1, dcs1, rowscale=rs1)
    else:
        dx1 = ll.norm_bwd(dn2, x1, n2w, None, rstd2, dx_in=dx2, dweight=dn2w)
        dy1 = ll.layerscale_bwd(dx1, y1, g1, dg1 if g1 is not None else None, dcs1, rowscale=rs1)
    dprojw = wgrad(dy1, a, pprojw)
    da = ll.gemm(dy1, projw, b_t=True)
    dqkv = torch.empty((M, 3 * D), device=x.device, dtype=bf16)
    if qkn is not None:
        q, k = qkn[:, :D], qkn[:, D:]
    else:
        q, k = qkv[:, :D], qkv[:, D:2 * D]
    ll.attn_bwd(q, k, qkv[:, 2 * D:], a, da, lse, B, n, H, d, d ** -0.5,
                dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])
    if qkn is not None and rk is None:
        ll.rmsnorm_pair_bwd(dqkv, qkv, D, qnw, knw, rq, dqnw, dknw)
    elif qkn is not None:
        ll.norm_bwd(dqkv[:, :D], qkv[:, :D], qnw, None, rq, dx_out=dqkv[:, :D], dweight=dqnw)
        ll.norm_bwd(dqkv[:, D:2 * D], qkv[:, D:2 * D], knw, None, rk, dx_out=dqkv[:, D:2 * D], dweight=dknw)
    dqkvw = wgrad(dqkv, n1, pqkvw)
    if qkvb is not None:
        ll.colsum(dqkv, out=dqkvb)
    dn1 = ll.gemm(dqkv, qkvw, b_t=True)
    dx0 = ll.norm_bwd(dn1, x, n1w, None, rstd1, dx_in=dx1, dweight=dn1w)
    # ---- O(D) glue: bias grads through LayerScale (layerscale_bwd already folds gamma into the
    # bias-gradient column sums), cast to the parameter dtype
    if sink is not None:
        sink.flat_grad[base:base + span].add_(vec[:span])
        for prm in (pn1w, pqkvb, pqnw, pknw, pprojb, pg1, pn2w, pfc1b, pfc2b, pg2):
            if prm is not None:
                sink.grad_written(prm)
        return dx0, None
    vb = vec.to(n1w.dtype)
    sl = lambda t: vb[t.storage_offset():t.storage_offset() + t.numel()]  # noqa: E731
    return dx0, (sl(dn1w), dqkvw, sl(dqkvb) if qkvb is not None else None,
                 sl(dqnw) if qnw is not None else None, sl(dknw) if knw is not None else None,
                 dprojw, sl(dcs1), sl(dg1) if g1 is not None else None, sl(dn2w),
                 dfc1w, sl(dfc1b), dfc2w, sl(dcs2), sl(dg2) if g2 is not None else None)


class BlockFn(torch.autograd.Function):
    """Differentiable block_forward.  dims = (B, n, H, gelu_tanh[, checkpoint]).

    checkpoint=True is the reference's `with_cp` / `use_checkpoint` (internvideo2_pretrain.py:294-295,
    torch.utils.checkpoint around the block): only the block INPUT (4 D bytes/token) is kept; backward first
    re-runs the 14 forward kernels to rebuild the 44 D bytes/token of saved activations, then the 26 backward
    kernels.  DropPath factors are inputs (rs1/rs2), so the recomputation sees the same draw."""

    @staticmethod
    def forward(ctx, x, dims, n1w, qkvw, qkvb, qnw, knw, projw, projb, g1, n2w, fc1w, fc1b, fc2w, fc2b, g2,
                rs1=None, rs2=None):
        # rs1/rs2: optional fp32 [B*n] per-row DropPath keep/scale factors of the two branches
        params = (n1w, qkvw, qkvb, qnw, knw, projw, projb, g1, n2w, fc1w, fc1b, fc2w, fc2b, g2)
        ckpt = len(dims) > 4 and bool(dims[4])
        x2, saved = block_forward(x, dims, params, rs1, rs2, save=not ckpt)
        ctx.dims, ctx.ckpt = tuple(dims[:4]), ckpt
        ctx.params = params
        if ckpt:
            ctx.nsaved = 0
            ctx.save_for_backward(x, rs1, rs2, *params)
        else:
            ctx.flags = saved[-1]
            ctx.save_for_backward(x, rs1, rs2, *params, *saved[:-1])
        return x2

    @staticmethod
    def backward(ctx, dx2):
        st = ctx.saved_tensors
        x, rs1, rs2 = st[:3]
        tensors = st[3:17]
        if ctx.ckpt:
            with torch.no_grad():
                _, saved = block_forward(x, ctx.dims, tensors, rs1, rs2, save=True)
        else:
            saved = tuple(st[17:]) + (ctx.flags,)
        dx0, grads = block_backward(x, saved, ctx.dims, tensors, ctx.params, dx2, rs1, rs2)
        if grads is None:
            return (dx0,) + (None,) * 17
        return (dx0, None) + tuple(grads) + (None, None)


def _common_sink(params):
    """The gradient sink shared by every parameter (None -> autograd accumulates as usual)."""
    sink = None
    for p in params:
        if p is None:
            continue
        s_ = getattr(p, "_ivb_sink", None)
        if s_ is None or p.grad is None or not p.requires_grad or (sink is not None and s_ is not sink):
            return None
        sink = s_
    return sink if (sink is not None and sink.direct_enabled()) else None


def _plan_small(small, params, sink, device):
    """fp32 scratch for the block's O(D) gradients.  With a sink the segments sit at the parameters'
    relative offsets inside the flat gradient buffer, so a single add_ lands them all.
    Returns (segments by name, scratch, span or None, base offset)."""
    seg = {}
    if sink is not None:
        present = [(nm, p, sz) for nm, p, sz in small if p is not None]
        base = min(p._ivb_off for _, p, _ in present)
        span = max(p._ivb_off + sz for _, p, sz in present) - base
        if span <= 2 * sum(sz for _, _, sz in present) + 4096:
            extra = sum(sz for _, p, sz in small if p is None)
            vec = torch.zeros(span + extra, device=device, dtype=f32)
            o = span
            for nm, p, sz in small:
                if p is not None:
                    seg[nm] = vec[p._ivb_off - base:p._ivb_off - base + sz]
                else:
                    seg[nm] = vec[o:o + sz]; o += sz
            return seg, vec, span, base
    vec = torch.zeros(sum(sz for _, _, sz in small), device=device, dtype=f32)
    o = 0
    for nm, _, sz in small:
        seg[nm] = vec[o:o + sz]; o += sz
    return seg, vec, None, 0


# ------------------------------------------------------------------------------------------ token front-end
class EmbedFn(torch.autograd.Function):
    """Visible-only tubelet embed + cls + pos-embed + compaction (internvideo2_pretrain.py:630-659).

    Embeds only the kept patches (the reference convolves all T*L patches and drops 80 %); token
    order is the bit-exact `x[~mask]` order given by `idx` (ivb_visible_indices).
    Returns the fp32 residual stream [B*n, D].
    """

    @staticmethod
    def forward(ctx, video, idx, w, b, cls, pos, tubelet, patch):
        _need_cuda_bf16(video, "video")
        B, C, T, H, W = video.shape
        n = idx.shape[1]
        D = w.shape[0]
        K = C * tubelet * patch * patch
        Kpad = (K + 7) // 8 * 8
        cols = ll.im2col_visible(video.contiguous(), idx, 1, n - 1, tubelet, patch, Kpad)
        wp = torch.zeros((D, Kpad), device=w.device, dtype=bf16)
        wp[:, :K] = w.reshape(D, K)
        emb = ll.gemm(cols, wp, bias=b, epi=ll.EPI_F32)                      # fp32 [B*(n-1), D]
        x0 = torch.empty((B, n, D), device=w.device, dtype=f32)
        pos2 = pos.reshape(-1, D)
        ll.gather_add(emb, (n - 1) * D, pos2, idx[:, 1:], n, 0, B, n - 1, D, x0[:, 1:], n * D)
        c0 = (cls.reshape(D).float() + pos2[0].float()).contiguous()
        ll.gather_add(c0, 0, None, None, 0, 0, B, 1, D, x0[:, 0], n * D)
        ctx.save_for_backward(cols, idx)
        ctx.meta = (B, n, D, K, Kpad, w.shape, pos.shape, cls.shape, w.dtype)
        return x0.reshape(B * n, D)

    @staticmethod
    def backward(ctx, dx0):
        cols, idx = ctx.saved_tensors
        B, n, D, K, Kpad, wshape, pshape, cshape, pdt = ctx.meta
        dx0 = dx0.contiguous().reshape(B, n, D)
        demb = torch.empty((B * (n - 1), D), device=dx0.device, dtype=bf16)
        ll.gather_add(dx0[:, 1:], n * D, None, None, 0, 0, B, n - 1, D, demb, (n - 1) * D)
        dw = ll.gemm(demb, cols, a_t=True, b_t=True)[:, :K].reshape(wshape)
        db = ll.colsum(demb).to(pdt)
        dpos = torch.zeros((pshape[-2], D), device=dx0.device, dtype=f32)
        ll.scatter_add(dx0, n * D, idx, n, 0, B, n, D, dpos)
        dcls = dx0[:, 0].sum(0)
        return (None, None, dw, db, dcls.reshape(cshape).to(pdt), dpos.reshape(pshape).to(pdt), None, None)


class GatherAddFn(torch.autograd.Function):
    """out(bf16)[b,j] = src(fp32)[b, j0+j] + table[idx[b, j0+j] + off]  — decoder pos-embed adds (:712-714, :735-737)."""

    @staticmethod
    def forward(ctx, src, table, idx, B, n, j0, off):
        D = src.shape[-1]
        rows = n - j0
        out = torch.empty((B * rows, D), device=src.device, dtype=bf16)
        s3 = src.reshape(B, n, D)
        ll.gather_add(s3[:, j0:], n * D, table.reshape(-1, D), idx[:, j0:], n, off, B, rows, D, out, rows * D)
        ctx.save_for_backward(idx)
        ctx.meta = (B, n, j0, off, D, table.shape, table.dtype)
        return out

    @staticmethod
    def backward(ctx, dout):
        (idx,) = ctx.saved_tensors
        B, n, j0, off, D, tshape, tdt = ctx.meta
        rows = n - j0
        dout = dout.contiguous()
        dsrc = torch.zeros((B, n, D), device=dout.device, dtype=f32) if j0 > 0 else torch.empty((B, n, D), device=dout.device, dtype=f32)
        dsrc[:, j0:] = dout.reshape(B, rows, D)
        dt = torch.zeros((tshape[-2], D), device=dout.device, dtype=f32)
        ll.scatter_add(dout, rows * D, idx[:, j0:], n, off, B, rows, D, dt)
        return dsrc.reshape(B * n, D), dt.reshape(tshape).to(tdt), None, None, None, None, None


# ------------------------------------------------------------------------------------------ decoder tails / losses
class LnL2Fn(torch.autograd.Function):
    """x / ||x|| after LayerNorm(1e-5): tail of Linear_Decoder / MLP_Decoder (:356-359, :394-397)."""

    @staticmethod
    def forward(ctx, z, w, b, eps):
        _need_cuda_bf16(z, "z")
        z2 = z.reshape(-1, z.shape[-1]).contiguous()
        out, stats = ll.ln_l2_fwd(z2, w, b, eps, want_out=True)
        ctx.save_for_backward(z2, w, b, stats)
        ctx.in_shape = z.shape
        return out.reshape(z.shape)

    @staticmethod
    def backward(ctx, dout):
        z2, w, b, stats = ctx.saved_tensors
        d2 = dout.reshape(-1, dout.shape[-1]).contiguous()
        if d2.dtype not in (bf16, f32):
            d2 = d2.float()
        C = z2.shape[1]
        dw = torch.zeros(C, device=z2.device, dtype=f32); db = torch.zeros(C, device=z2.device, dtype=f32)
        dz = ll.ln_l2_bwd(z2, w, b, stats, d2, 1.0, None, dw, db)
        return dz.reshape(ctx.in_shape), dw.to(w.dtype), db.to(b.dtype), None


class AlignLossFn(torch.autograd.Function):
    """mean_rows(2 - 2 <l2n(LN(z)), tgt>) without materialising the normalised features
    (decoder tail :356-359 + engines/engine_for_pretraining.py:131-136)."""

    @staticmethod
    def forward(ctx, z, w, b, tgt, eps):
        _need_cuda_bf16(z, "z")
        z2 = z.reshape(-1, z.shape[-1]).contiguous()
        t2 = tgt.reshape(-1, tgt.shape[-1])
        if t2.dtype not in (bf16, f32):
            t2 = t2.float()
        t2 = t2.contiguous()
        ls = torch.zeros(1, device=z.device, dtype=f32)
        _, stats = ll.ln_l2_fwd(z2, w, b, eps, want_out=False, target=t2, loss_sum=ls)
        ctx.save_for_backward(z2, w, b, stats, t2)
        ctx.in_shape = z.shape
        return (ls / z2.shape[0]).reshape(())

    @staticmethod
    def backward(ctx, g):
        z2, w, b, stats, t2 = ctx.saved_tensors
        C = z2.shape[1]
        dw = torch.zeros(C, device=z2.device, dtype=f32); db = torch.zeros(C, device=z2.device, dtype=f32)
        gd = g.reshape(1).to(f32).contiguous()
        dz = ll.ln_l2_bwd(z2, w, b, stats, t2, -2.0 / z2.shape[0], gd, dw, db)
        return dz.reshape(ctx.in_shape), dw.to(w.dtype), db.to(b.dtype), None, None


class VtcLossFn(torch.autograd.Function):
    """Video-text contrastive loss over the gathered batch; gradients flow to the LOCAL rows only
    (get_sim + vtc_loss + AllGather.backward: criterions.py:15-55,65-103; models/utils.py:205-209)."""

    @staticmethod
    def forward(ctx, v_all, t_all, idx_all, temp, rank, b_local):
        vn, vinv = ll.l2norm_rows_fwd(v_all.contiguous())
        tn, tinv = ll.l2norm_rows_fwd(t_all.contiguous())
        G = vn.shape[0]
        Gp = (G + 7) // 8 * 8
        if Gp != G:     # tiny gathered batches (tests): the GEMM wants 16-byte row pitches -> zero-pad to 8 rows
            pad = lambda x: torch.cat([x, x.new_zeros((Gp - G, x.shape[1]))], 0)  # noqa: E731
            vn, tn = pad(vn), pad(tn)
            cosm = ll.gemm(vn, tn, epi=ll.EPI_F32)[:G, :G].contiguous()
        else:
            cosm = ll.gemm(vn, tn, epi=ll.EPI_F32)
        # a tensor temperature (the learnable `temp`, internvideo2_clip_small.py:45) never leaves the device
        if torch.is_tensor(temp):
            tdev = temp.detach().to(device=cosm.device, dtype=f32).reshape(1).contiguous()
            tval = 1.0
        else:
            tdev, tval = None, float(temp)
        loss, lr_, lc_ = ll.vtc_loss_fwd(cosm, idx_all.contiguous(), tval, temp_dev=tdev)
        ctx.save_for_backward(vn, tn, vinv, tinv, cosm, lr_, lc_, idx_all, tdev)
        ctx.meta = (tval, rank, b_local, v_all.dtype, t_all.dtype, temp.dtype if torch.is_tensor(temp) else None)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g):
        vn, tn, vinv, tinv, cosm, lr_, lc_, idx_all, tdev = ctx.saved_tensors
        tval, rank, bl, vdt, tdt, temp_dt = ctx.meta
        Gp, C = vn.shape
        G = cosm.shape[0]
        gd = g.reshape(1).to(f32).contiguous()
        dcos, dtemp = ll.vtc_loss_bwd(cosm, idx_all, tval, lr_, lc_, 1.0, gd, temp_dev=tdev)
        if Gp != G:
            dp = dcos.new_zeros((Gp, Gp)); dp[:G, :G] = dcos; dcos = dp
        lo, hi = rank * bl, (rank + 1) * bl
        # d vn[local] = dcos[local, :] @ tn ; d tn[local] = dcos[:, local]^T @ vn
        if Gp != G:     # padded: whole-matrix products (row/column slices of a padded buffer may break the 16 B pitch)
            dvn = ll.gemm(dcos, tn, b_t=True, epi=ll.EPI_F32)[lo:hi].contiguous()
            dtn = ll.gemm(dcos, vn, a_t=True, b_t=True, epi=ll.EPI_F32)[lo:hi].contiguous()
        else:
            dvn = ll.gemm(dcos[lo:hi], tn, b_t=True, epi=ll.EPI_F32)
            dtn = ll.gemm(dcos[:, lo:hi], vn, a_t=True, b_t=True, epi=ll.EPI_F32)
        dv = torch.zeros((G, C), device=vn.device, dtype=f32)
        dt = torch.zeros((G, C), device=vn.device, dtype=f32)
        dv[lo:hi] = ll.l2norm_rows_bwd(dvn, vn[lo:hi].contiguous(), vinv[lo:hi])
        dt[lo:hi] = ll.l2norm_rows_bwd(dtn, tn[lo:hi].contiguous(), tinv[lo:hi])
        return dv.to(vdt), dt.to(tdt), None, (dtemp.reshape(()).to(temp_dt) if temp_dt is not None else None), None, None
