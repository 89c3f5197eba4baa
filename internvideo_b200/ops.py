"""torch.autograd.Function wrappers over the C ABI (lowlevel.py): the differentiable op surface.

Everything here runs on the H100 through libivb200.so; there is no eager/PyTorch fallback for the
compute (tiny O(D) vector glue such as `gamma * colsum` uses torch elementwise ops on CUDA tensors).
Activations are bf16, the residual stream is fp32, parameters are bf16 (the reference's bf16
DeepSpeed mode converts the whole model: engines/engine_for_pretraining.py:128, SURVEY App.B-18).
"""
from __future__ import annotations

from collections import namedtuple
from typing import NamedTuple

import torch

from . import lowlevel as ll

bf16, f32 = torch.bfloat16, torch.float32


def _pdt(g, p):
    """cast a gradient to its parameter's dtype (vector grads are accumulated in fp32)."""
    return None if g is None else g.to(p.dtype)


# ------------------------------------------------------------------------------------------ Linear
class LinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM (nn.Linear: internvideo2_pretrain.py:61-77,195,211,356).  w_t: W is stored
    transposed, [in, out], and y = x W + b reads it as the GEMM's MN-major operand (the text tower's projection_layer,
    text_encoder.py:219)."""

    @staticmethod
    def forward(ctx, x, w, b, out_f32=False, w_t=False):
        x2 = x.reshape(-1, x.shape[-1])
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        y = ll.gemm(x2, w, b_t=w_t, bias=b, epi=ll.EPI_F32 if out_f32 else ll.EPI_BF16)
        ctx.save_for_backward(x2, w)
        ctx.w_t = w_t
        ctx.has_bias = b is not None
        ctx.bias_dtype = b.dtype if b is not None else None
        ctx.in_shape = x.shape
        return y.reshape(*x.shape[:-1], w.shape[1] if w_t else w.shape[0])

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
            dx = ll.gemm(dy2, w, b_t=not ctx.w_t).reshape(ctx.in_shape)
        if ctx.needs_input_grad[1]:
            dw = ll.gemm(x2, dy2, a_t=True, b_t=True) if ctx.w_t else ll.gemm(dy2, x2, a_t=True, b_t=True)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = ll.colsum(dy2).to(ctx.bias_dtype)
        return dx, dw, db, None, None


def linear(x, w, b=None, out_f32=False, w_t=False):
    return LinearFn.apply(x, w, b, out_f32, w_t)


class LinearGeluFn(torch.autograd.Function):
    """g = GELU(x W^T + b) with the activation fused in the GEMM epilogue (Mlp.fc1+act :239-240)."""

    @staticmethod
    def forward(ctx, x, w, b, gelu_tanh=False):
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
# A block's precision (BlockSpec.precision): BF16; FP8_TENSOR, FP8 with per-tensor scales and the weights cast in the
# call (modules.set_fp8); FP8_TOKEN, FP8 with per-token scales and the weights cast per channel in the call
# (modules.set_fp8 with scaling="token"); FP8_TOKEN_WGRAD, FP8_TOKEN whose weight gradients also run in FP8, from
# operands cast with one scale per channel per 128-token block (modules.set_fp8 with scaling="token", wgrad=True); or
# per-token FP8 inference (modules.set_fp8_inference, no-grad calls only), given as the four weights' per-channel E4M3
# copies themselves: ((q, scale_inv) for qkv, proj, fc1, fc2).
BF16, FP8_TENSOR, FP8_TOKEN, FP8_TOKEN_WGRAD = "bf16", "fp8", "fp8_token", "fp8_token_wgrad"
_PER_TOKEN = (FP8_TOKEN, FP8_TOKEN_WGRAD)      # the precisions whose forward and input gradients are FP8_TOKEN's


class BlockSpec(NamedTuple):
    """Everything a fused block call needs besides its tensors.  layernorm: the VideoMAE LayerNorm block (InternVideo1,
    VideoMAEv2 teacher) instead of the RMSNorm block; eps1 / eps2 are the eps of its two norms.  scale: the attention
    scale (None: d ** -0.5).  head_axis: the VideoMAEv2 teacher's attention over the heads of each token (inference
    only).  checkpoint: BlockFn keeps only the block input and recomputes the forward in the backward.  attn_fp8: the
    token-axis attention runs on the FP8 tensor cores (lowlevel._attn_fp8_pack + _attn_fwd_fp8; inference only:
    block_forward refuses it with save=True or head_axis).  causal: token-axis attention masks every key after its
    query (the MobileCLIP text tower; block_forward refuses it with head_axis, attn_fp8 or a DropPath plan).
    gelu_quick: the MLP's activation is QuickGELU, x * sigmoid(1.702 x) (OpenAI-CLIP blocks: ViCLIP), instead of the
    erf GELU; it excludes gelu_tanh."""
    B: int
    n: int
    H: int
    gelu_tanh: bool = False
    layernorm: bool = False
    eps1: float = 1e-6
    eps2: float = 1e-6
    scale: float | None = None
    head_axis: bool = False
    checkpoint: bool = False
    precision: object = BF16
    attn_fp8: bool = False
    causal: bool = False
    gelu_quick: bool = False

    def attn_scale(self, d):
        return d ** -0.5 if self.scale is None else self.scale

    def gelu_flags(self, save):
        """fc1's epilogue flags; with save, h holds gelu'(pre-activation), the only thing the backward needs of it."""
        if self.gelu_tanh and self.gelu_quick:
            raise ll._lib.IvbError("BlockSpec: gelu_tanh and gelu_quick exclude each other")
        return ((ll.FLAG_GELU_TANH if self.gelu_tanh else 0) | (ll.FLAG_GELU_QUICK if self.gelu_quick else 0)
                | (ll.FLAG_GELU_SAVE_GRAD if save else 0))


# A block's tensors.  qkvb, qnw / knw (q/k norms) and g1 / g2 (LayerScale) may be None; n1b / n2b are the LayerNorm
# biases, None on RMSNorm blocks.
BlockParams = namedtuple("BlockParams", "n1w qkvw qkvb qnw knw projw projb g1 n2w fc1w fc1b fc2w fc2b g2 n1b n2b",
                         defaults=(None, None))

# What block_forward(save=True) keeps for block_backward: activations and norm statistics (mean1 / mean2 None on RMSNorm
# blocks), and in FP8 the E4M3 copies of the four weights' transposes with their scales (the input-gradient GEMMs'
# operands; per-tensor scalars in FP8_TENSOR, one scale per input channel in FP8_TOKEN and FP8_TOKEN_WGRAD; None in
# bf16).
BlockSaved = namedtuple("BlockSaved", "n1 qkv qkn a lse mean1 rstd1 rq rk x1 y1 n2 mean2 rstd2 h g y2 "
                                      "qkvw_t qkvw_s projw_t projw_s fc1w_t fc1w_s fc2w_t fc2w_s")


def droppath_plan(rowscale):
    """DropPath plans of the rows of rowscale fp32 [R, M], one block branch's per-row factors each (ivb_droppath_plan,
    one launch): int32 [R, ivb_droppath_plan_ints(M)], row r the plan of branch r, for block_forward / block_backward."""
    ll._chk(("rowscale", rowscale, f32))
    R, M = rowscale.shape
    plan = torch.empty((R, int(ll._lib.load().ivb_droppath_plan_ints(M))), device=rowscale.device, dtype=torch.int32)
    ll._call("droppath_plan", rowscale, ll._rows2d(rowscale, "rowscale"), R, M, plan, plan.stride(0))
    return plan


def _branch_plans(plan, M, prec):
    """(M plan, K plan) of a branch's DropPath plan row for the block's GEMMs over its M rows: the M plan for a GEMM
    whose M rows are the block's rows (bf16, or FP8 with per-token scales), the K plan for a weight gradient whose K runs
    over them (bf16: the plan's 64-row k-blocks; FP8_TOKEN_WGRAD: the M plan itself, whose live 128-row tiles are the
    FP8 weight gradient's 128-token k-blocks).  (None, None) without a plan or in FP8_TENSOR: there a dropped clip's
    rows still count in each activation's and gradient's per-tensor amax, and skipping them would zero those rows and
    change the scales, so every row runs.  In FP8_TOKEN each scale belongs to one row: a dropped row's zeros change
    only its own (finite) scale, and it feeds only dead tiles or rows the epilogue multiplies by 0.  The FP8 weight
    gradient's block scales span 128 rows: its casts zero the dropped rows of both operands (block_backward), so they
    do not depend on the plan either."""
    if plan is None or prec not in (BF16, *_PER_TOKEN):
        return None, None
    nm = (M + 127) // 128
    return plan[:nm + 1], plan[:nm + 1] if prec == FP8_TOKEN_WGRAD else plan[nm + 1:]


def block_forward(x, spec, p, rs1=None, rs2=None, save=True, plan1=None, plan2=None):
    """One pre-norm ViT block over the fp32 residual stream [B*n, D]: spec a BlockSpec, p the BlockParams.  The
    InternVideo2 block (Block.forward, internvideo2_pretrain.py:279-297), or with spec.layernorm the VideoMAE block
    (videomae.py:104-132, IV1 modeling_finetune.py:132-181: LayerNorm with bias, q/v bias on qkv, no q/k norm, erf GELU):

      n1 = Norm(x) ; qkv = n1 Wqkv^T + bqkv ; (q,k) = RMSNorm_C(q), RMSNorm_C(k) ; a = attn(q,k,v)
      x1 = x + rs1 * g1 * (a Wp^T + bp)                [LayerScale + DropPath + residual fused in the GEMM epilogue]
      n2 = Norm(x1) ; h = n2 W1^T + b1 ; g = GELU(h) [fused epilogue] ; x2 = x1 + rs2 * g2 * (g W2^T + b2)

    In bf16, 7 library calls, and 1 more for the q/k norms (2 when D > 1536).  save=True also writes what the backward
    needs (pre-LayerScale branch outputs, GELU') and returns it; save=False is the inference / recompute-later form
    (frozen towers, teachers, activation checkpointing): nothing extra is written.  Returns (x2, BlockSaved | None).

    FP8_TENSOR (8 more calls): the four weights are cast to E4M3 (with save, also transposed, for the backward's dgrad)
    and n1, a, n2 and g before their GEMM, each with its own per-tensor scale; the GEMMs keep their fused epilogues.
    Per-token FP8 (FP8_TOKEN, or the inference weight copies; 2 more calls): n1 and n2 come out of the norm kernel as
    E4M3 rows with per-row scales, a and g are cast row by row, and the four GEMMs apply row and column scales before
    their fused epilogues.  FP8_TOKEN also casts the four weights per output channel (4 calls) and, with save, per input
    channel into their transposed copies (4 more), and its norm kernel then also writes the bf16 row and statistics
    the backward needs (without save: the same E4M3 bits from the inference norm kernel).  Attention, the q/k norms and
    the residual stream stay as above.  FP8_TOKEN_WGRAD runs the forward exactly as FP8_TOKEN and saves the same state.

    spec.attn_fp8 (save=False and token-axis attention only; anything else raises IvbError): attention casts q, k and v
    to E4M3 (one more call) and runs on the FP8 tensor cores instead of ivb_attn_fwd.

    plan1 / plan2: optional DropPath plans of the two branches (rows of droppath_plan of rs1 / rs2): in bf16 and
    FP8_TOKEN the GEMMs of a branch then skip the row tiles whose rows rs zeroes, writing what the epilogue table of
    ivb_gemm_bf16_plan gives them (x1 = x, zeros elsewhere), and attention skips the clips rs1 drops (a = 0 there);
    the rows they do compute and x2 are as without a plan."""
    B, n, H = spec.B, spec.n, spec.H
    M, D = x.shape
    d = D // H
    if spec.attn_fp8 and (save or spec.head_axis):
        raise ll._lib.IvbError("block_forward: FP8 attention (spec.attn_fp8) is inference-only and token-axis: it needs "
                               "save=False and head_axis=False")
    if spec.causal and (spec.attn_fp8 or spec.head_axis or plan1 is not None or plan2 is not None):
        raise ll._lib.IvbError("block_forward: causal attention runs in bf16 over the tokens, without DropPath plans: "
                               "it excludes attn_fp8, head_axis and plan1 / plan2")
    if x.dtype != f32 or not x.is_cuda:
        raise ll._lib.IvbError("block_forward: residual stream must be a CUDA fp32 tensor [B*n, D]")
    prec = spec.precision
    per_token = prec in _PER_TOKEN or not isinstance(prec, str)
    weights = (p.qkvw, p.projw, p.fc1w, p.fc2w)
    # (q, scale_inv, q_t, scale_inv of q_t) per weight; q_t only when the backward will need it
    if prec == FP8_TENSOR:
        w8 = [(q, s, q_t, s) for q, q_t, s, _ in (ll.fp8_quantize(w, ll.FP8_E4M3, transpose=save) for w in weights)]
    elif prec in _PER_TOKEN:
        w8 = [(*ll.fp8_quantize_rows(w), *(ll.fp8_quantize_rows(w, transposed=True) if save else (None, None))) for w in weights]
    elif per_token:
        w8 = [(q, s, None, None) for q, s in prec]

    def norm(t, w, b, eps):   # (n1 or n2 as its GEMM reads it, the bf16 row the backward reads, mean, rstd)
        if not per_token:
            y, mean, rstd = ll.norm_fwd(t, w, b, eps=eps, layernorm=spec.layernorm, want_stats=save)
            return y, y, mean, rstd
        if not save:
            return ll.norm_fwd_fp8(t, w, b, eps=eps, layernorm=spec.layernorm), None, None, None
        q, s, y, mean, rstd = ll.norm_fwd_fp8(t, w, b, eps=eps, layernorm=spec.layernorm, save=True)
        return (q, s), y, mean, rstd

    mp = (_branch_plans(plan1, M, prec)[0], _branch_plans(plan2, M, prec)[0])

    def linear(act, i, w, **epilogue):
        if prec == BF16:
            return ll.gemm(act, w, m_plan=mp[i // 2], **epilogue)
        if per_token:     # act: bf16, or the (E4M3 rows, scale_inv) pair the norm wrote
            q, s = ll.fp8_quantize_rows(act) if torch.is_tensor(act) else act
        else:
            q, _, s, _ = ll.fp8_quantize(act, ll.FP8_E4M3)
        return ll._gemm_fp8_plan(q, s, w8[i][0], w8[i][1], mp[i // 2], **epilogue)
    n1_in, n1, mean1, rstd1 = norm(x, p.n1w, p.n1b, spec.eps1)
    qkv = linear(n1_in, 0, p.qkvw, bias=p.qkvb)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    qkn = rq = rk = lse = None
    if p.qnw is not None:
        qkn = torch.empty((M, 2 * D), device=x.device, dtype=bf16)
        if D <= 1536:      # q-norm and k-norm in ONE launch; rq holds rstd [M, 2] for both
            rq = ll.rmsnorm_pair_fwd(qkv, D, p.qnw, p.knw, qkn, want_stats=save)
        else:
            _, _, rq = ll.norm_fwd(q, p.qnw, out=qkn[:, :D], want_stats=save)
            _, _, rk = ll.norm_fwd(k, p.knw, out=qkn[:, D:], want_stats=save)
        q, k = qkn[:, :D], qkn[:, D:]
    if spec.head_axis:
        # the reference's call (videomae.py:94-97) attends over the heads of each token and reinterprets the
        # [B, H, N, d] result as [B, N, H*d]: reproduced bit-for-layout
        a = ll.headaxis_attn_fwd(qkv, B, n, H, d, spec.attn_scale(d)).reshape(M, D)
    elif spec.attn_fp8:
        a = ll._attn_fwd_fp8(*ll._attn_fp8_pack(q, k, v, B, n, H, d), B, n, H, d, spec.attn_scale(d))
    else:
        a, lse = ll.attn_fwd(q, k, v, B, n, H, d, spec.attn_scale(d), want_lse=save,
                             rowscale=rs1 if mp[0] is not None else None, causal=spec.causal)
    y1 = torch.empty((M, D), device=x.device, dtype=bf16) if (p.g1 is not None and save) else None
    x1 = linear(a, 1, p.projw, epi=ll.EPI_RESID, bias=p.projb, gamma=p.g1, aux=x, out1=y1, rowscale=rs1)
    n2_in, n2, mean2, rstd2 = norm(x1, p.n2w, p.n2b, spec.eps2)
    h = torch.empty((M, p.fc1w.shape[0]), device=x.device, dtype=bf16) if save else None
    g = linear(n2_in, 2, p.fc1w, epi=ll.EPI_BIAS_GELU, flags=spec.gelu_flags(save), bias=p.fc1b, out1=h)
    y2 = torch.empty((M, D), device=x.device, dtype=bf16) if (p.g2 is not None and save) else None
    x2 = linear(g, 3, p.fc2w, epi=ll.EPI_RESID, bias=p.fc2b, gamma=p.g2, aux=x1, out1=y2, rowscale=rs2)
    if not save:
        return x2, None
    wt8 = [t for _, _, q_t, s_t in w8 for t in (q_t, s_t)] if prec != BF16 else [None] * 8
    return x2, BlockSaved(n1, qkv, qkn, a, lse, mean1, rstd1, rq, rk, x1, y1, n2, mean2, rstd2, h, g, y2, *wt8)


def block_backward(x, s, spec, t, P, dx2, rs1, rs2, plan1=None, plan2=None):
    """Backward of block_forward(save=True), from its BlockSaved s: 13 to 17 library calls in bf16 (with or without the
    q/k norms and the qkv bias, the fused RMSNorm norm2 + LayerScale backward), and in FP8 one more per input-gradient
    GEMM (the cast of its gradient: E5M2 with a per-tensor scale in FP8_TENSOR, E4M3 rows with per-row scales in
    FP8_TOKEN).  FP8_TOKEN_WGRAD also runs the four weight gradients in FP8, with two more calls each: the transposing
    casts of dy and of the saved bf16 activation, one scale per channel per 128-token block (lowlevel._fp8_quantize_blocks_t;
    the activation's rows whose DropPath factor is 0 are cast as zeros, as their gradient rows are), then
    lowlevel._gemm_fp8_wgrad, with or without the gradient sink.  The LayerNorm block (spec.layernorm) also returns its norms'
    bias gradients and always runs the attention branch's LayerScale backward as its own call.  `t` are the block's
    tensors as autograd handed them back, `P` the nn.Parameter objects (gradient sink), both BlockParams.  Returns
    (dx0, BlockParams of gradients | None when the sink took them).  plan1 / plan2: the DropPath plans block_forward
    ran with; the input-gradient GEMMs of a branch skip its dead row tiles (zeros), its weight gradients the
    64-row (FP8 weight gradients: 128-row) k-blocks of dropped rows, whose gradient rows layerscale_bwd made zero, and
    attention the dropped clips."""
    B, n, H = spec.B, spec.n, spec.H
    M, D = x.shape
    d = D // H
    Hd = t.fc1w.shape[0]
    dx2 = dx2.contiguous()
    if dx2.dtype != f32:
        dx2 = dx2.float()
    # Gradient sink (engine.PretrainEngine): when every parameter of the block lives in the engine's
    # flat gradient buffer, the wgrad GEMMs accumulate straight into it (FLAG_ACCUM epilogue) and the
    # O(D) gradients land with ONE fused add per block — no autograd AccumulateGrad kernels (16 per
    # block, each re-reading and re-writing the gradient).
    sink = _common_sink(P)
    small = [(nm, getattr(t, nm), D) for nm in ("g2", "fc2b", "n2w", "g1", "projb", "qnw", "knw", "n1w")]
    small += [("fc1b", t.fc1b, Hd), ("qkvb", t.qkvb, 3 * D)]
    if spec.layernorm:
        small += [("n2b", t.n2b, D), ("n1b", t.n1b, D)]
    seg, vec, span, base = _plan_small(small, sink, x.device)
    if sink is not None and span is None:
        sink = None           # small parameters not contiguous in the flat buffer: autograd path
    dg2, dcs2, dn2w, dg1, dcs1 = seg["g2"], seg["fc2b"], seg["n2w"], seg["g1"], seg["projb"]

    (m1, k1), (m2, k2) = _branch_plans(plan1, M, spec.precision), _branch_plans(plan2, M, spec.precision)

    def dgrad(dy, w, w_t, w_s, m_plan, **epilogue):   # dx = dy W; in FP8 on the cast gradient and the E4M3 copy of W^T
        if spec.precision in _PER_TOKEN:
            q, sc = ll.fp8_quantize_rows(dy)
        elif spec.precision == FP8_TENSOR:
            q, _, sc, _ = ll.fp8_quantize(dy, ll.FP8_E5M2)
        else:
            return ll.gemm(dy, w, b_t=True, m_plan=m_plan, **epilogue)
        return ll._gemm_fp8_plan(q, sc, w_t, w_s, m_plan, **epilogue)

    def wgrad(dy, act, param, k_plan, rs):   # dW = dy^T act; with the sink accumulated into the flat gradient
        out0, flags = (None, 0) if sink is None else (param.grad, ll.FLAG_ACCUM)
        if spec.precision == FP8_TOKEN_WGRAD:
            (qd, sd), (qa, sa) = ll._fp8_quantize_blocks_t(dy), ll._fp8_quantize_blocks_t(act, rowscale=rs)
            dw = ll._gemm_fp8_wgrad(qd, sd, qa, sa, out0=out0, flags=flags, k_plan=k_plan)
        else:
            dw = ll.gemm(dy, act, a_t=True, b_t=True, out0=out0, flags=flags, k_plan=k_plan)
        if sink is None:
            return dw
        sink.grad_written(param)
        return None
    # ---- MLP branch
    dy2 = ll.layerscale_bwd(dx2, s.y2, t.g2, dg2 if t.g2 is not None else None, dcs2, rowscale=rs2)
    dfc2w = wgrad(dy2, s.g, P.fc2w, k2, rs2)
    dh = dgrad(dy2, t.fc2w, s.fc2w_t, s.fc2w_s, m2, epi=ll.EPI_GELU_BWD, flags=spec.gelu_flags(True), aux=s.h)
    ll.colsum(dh, out=seg["fc1b"])
    dfc1w = wgrad(dh, s.n2, P.fc1w, k2, rs2)
    dn2 = dgrad(dh, t.fc1w, s.fc1w_t, s.fc1w_s, m2)
    # ---- attention branch
    if not spec.layernorm and t.g1 is not None and D <= 1536 and M >= 1024:
        # norm2 backward fused with the attention branch's LayerScale backward: the gradient of the residual
        # stream is produced and consumed in one pass over the rows
        dx1, dy1 = ll.rmsnorm_bwd_layerscale(dn2, s.x1, t.n2w, s.rstd2, dx2, s.y1, t.g1, dn2w, dg1, dcs1, rowscale=rs1)
    else:
        dx1 = ll.norm_bwd(dn2, s.x1, t.n2w, s.mean2, s.rstd2, layernorm=spec.layernorm, dx_in=dx2, dweight=dn2w,
                          dbias=seg.get("n2b"))
        dy1 = ll.layerscale_bwd(dx1, s.y1, t.g1, dg1 if t.g1 is not None else None, dcs1, rowscale=rs1)
    dprojw = wgrad(dy1, s.a, P.projw, k1, rs1)
    da = dgrad(dy1, t.projw, s.projw_t, s.projw_s, m1)
    dqkv = torch.empty((M, 3 * D), device=x.device, dtype=bf16)
    qk = s.qkn if s.qkn is not None else s.qkv
    ll.attn_bwd(qk[:, :D], qk[:, D:2 * D], s.qkv[:, 2 * D:], s.a, da, s.lse, B, n, H, d, spec.attn_scale(d),
                dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:], rowscale=rs1 if m1 is not None else None,
                causal=spec.causal)
    if s.qkn is not None and s.rk is None:
        ll.rmsnorm_pair_bwd(dqkv, s.qkv, D, t.qnw, t.knw, s.rq, seg["qnw"], seg["knw"])
    elif s.qkn is not None:
        ll.norm_bwd(dqkv[:, :D], s.qkv[:, :D], t.qnw, None, s.rq, dx_out=dqkv[:, :D], dweight=seg["qnw"])
        ll.norm_bwd(dqkv[:, D:2 * D], s.qkv[:, D:2 * D], t.knw, None, s.rk, dx_out=dqkv[:, D:2 * D], dweight=seg["knw"])
    dqkvw = wgrad(dqkv, s.n1, P.qkvw, k1, rs1)
    if t.qkvb is not None:
        ll.colsum(dqkv, out=seg["qkvb"])
    dn1 = dgrad(dqkv, t.qkvw, s.qkvw_t, s.qkvw_s, m1)
    dx0 = ll.norm_bwd(dn1, x, t.n1w, s.mean1, s.rstd1, layernorm=spec.layernorm, dx_in=dx1, dweight=seg["n1w"],
                      dbias=seg.get("n1b"))
    # ---- O(D) glue: bias grads through LayerScale (layerscale_bwd already folds gamma into the
    # bias-gradient column sums), cast to the parameter dtype
    if sink is not None:
        sink.flat_grad[base:base + span].add_(vec[:span])
        for nm in BlockParams._fields:
            if nm in seg and getattr(P, nm) is not None:
                sink.grad_written(getattr(P, nm))
        return dx0, None
    vb = vec.to(t.n1w.dtype)
    small_grads = {nm: None if prm is None else vb[seg[nm].storage_offset():seg[nm].storage_offset() + seg[nm].numel()]
                   for nm, prm, _ in small}
    return dx0, BlockParams(qkvw=dqkvw, projw=dprojw, fc1w=dfc1w, fc2w=dfc2w, **small_grads)


class BlockFn(torch.autograd.Function):
    """Differentiable block_forward: apply(x, spec, rs1, rs2, *params[, plan1, plan2]) with spec a BlockSpec
    (spec.head_axis refused), params the BlockParams, rs1 / rs2 optional fp32 [B*n] per-row DropPath keep/scale factors
    of the two branches and plan1 / plan2 their optional DropPath plans (block_forward).

    spec.checkpoint is the reference's `with_cp` / `use_checkpoint` (internvideo2_pretrain.py:294-295,
    torch.utils.checkpoint around the block): only the block INPUT (4 D bytes/token) is kept; backward first
    re-runs the forward to rebuild the 44 D bytes/token of saved activations, then the backward.  DropPath factors
    and plans are inputs, so the recomputation sees the same draw."""

    @staticmethod
    def forward(ctx, x, spec, rs1, rs2, *args):
        if spec.head_axis:
            raise ll._lib.IvbError("BlockFn: head-axis attention (the VideoMAEv2 teacher's) has no backward")
        nparams = len(BlockParams._fields)
        params = BlockParams(*args[:nparams])
        plans = tuple(args[nparams:]) or (None, None)
        x2, saved = block_forward(x, spec, params, rs1, rs2, save=not spec.checkpoint, plan1=plans[0], plan2=plans[1])
        ctx.spec, ctx.params, ctx.nplans = spec, params, len(args) - nparams
        ctx.save_for_backward(x, rs1, rs2, *plans, *params, *(saved or ()))
        return x2

    @staticmethod
    def backward(ctx, dx2):
        x, rs1, rs2, plan1, plan2, *rest = ctx.saved_tensors
        nparams = len(BlockParams._fields)
        tensors = BlockParams._make(rest[:nparams])
        if ctx.spec.checkpoint:
            with torch.no_grad():
                _, saved = block_forward(x, ctx.spec._replace(checkpoint=False), tensors, rs1, rs2, save=True,
                                         plan1=plan1, plan2=plan2)
        else:
            saved = BlockSaved._make(rest[nparams:])
        dx0, grads = block_backward(x, saved, ctx.spec, tensors, ctx.params, dx2, rs1, rs2, plan1, plan2)
        return (dx0, None, None, None) + (grads or (None,) * nparams) + (None,) * ctx.nplans


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


def _plan_small(small, sink, device):
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

    idx: int32 [B, 1 + m], column 0 the cls slot, then the m patch tokens.  ncls: the number k of cls rows in front of
    the patch rows (InternVideo-Next has 4): row i < k is cls[i] + pos[i], and a patch token t >= 1 takes position row
    t + k - 1, so n = k + m.  norm_w / norm_before_w: the RMSNorm weights of InternVideo-Next's dual-norm patch embed
    (InternVideo_next.py:302-342), eps their eps: the patch's pixels go through norm_before inside the im2col
    (ivb_im2col_prenorm), the bf16 conv output through norm (ivb_norm_fwd).  With k = 1 and no norms the calls are the
    single-cls ones of every other tower.
    """

    @staticmethod
    def forward(ctx, video, idx, w, b, cls, pos, tubelet, patch, ncls=1, norm_w=None, norm_before_w=None, eps=1e-6):
        B, C, T, H, W = video.shape
        ni = idx.shape[1]
        m, k = ni - 1, ncls
        n = k + m
        D = w.shape[0]
        K = C * tubelet * patch * patch
        Kpad = (K + 7) // 8 * 8
        video = video.contiguous()
        if norm_before_w is not None:
            cols, rstd_pix = ll._im2col_prenorm(video, idx, 1, m, tubelet, patch, Kpad, norm_before_w, eps)
        else:
            cols, rstd_pix = ll.im2col_visible(video, idx, 1, m, tubelet, patch, Kpad), None
        wp = torch.zeros((D, Kpad), device=w.device, dtype=bf16)
        wp[:, :K] = w.reshape(D, K)
        if norm_w is None:
            conv = rstd_emb = None
            emb = ll.gemm(cols, wp, bias=b, epi=ll.EPI_F32)                  # fp32 [B*m, D]
        else:     # the reference normalises the bf16 conv output; the bf16 norm output is widened for the stream
            conv = ll.gemm(cols, wp, bias=b, epi=ll.EPI_BF16)
            y, _, rstd_emb = ll.norm_fwd(conv, norm_w, eps=eps)
            emb = y.float()
        x0 = torch.empty((B, n, D), device=w.device, dtype=f32)
        pos2 = pos.reshape(-1, D)
        ll.gather_add(emb, m * D, pos2, idx[:, 1:], ni, k - 1, B, m, D, x0[:, k:], n * D)
        c0 = (cls.reshape(k, D).float() + pos2[:k].float()).contiguous()
        ll.gather_add(c0, 0, None, None, 0, 0, B, k, D, x0[:, :k], n * D)
        ctx.save_for_backward(cols, idx, wp if norm_before_w is not None else None,
                              video if norm_before_w is not None else None, rstd_pix, conv, norm_w, rstd_emb)
        ctx.meta = (B, n, k, D, K, Kpad, tubelet, patch, w.shape, pos.shape, cls.shape, w.dtype)
        return x0.reshape(B * n, D)

    @staticmethod
    def backward(ctx, dx0):
        cols, idx, wp, video, rstd_pix, conv, norm_w, rstd_emb = ctx.saved_tensors
        B, n, k, D, K, Kpad, tubelet, patch, wshape, pshape, cshape, pdt = ctx.meta
        m = n - k
        dx0 = dx0.contiguous().reshape(B, n, D)
        demb = torch.empty((B * m, D), device=dx0.device, dtype=bf16)
        ll.gather_add(dx0[:, k:], n * D, None, None, 0, 0, B, m, D, demb, m * D)
        dnw = dnbw = None
        if conv is not None:
            dnw = torch.zeros(D, device=dx0.device, dtype=f32)
            demb = ll.norm_bwd(demb, conv, norm_w, None, rstd_emb, dx_dtype=bf16, dweight=dnw)
            dnw = dnw.to(pdt)
        dw = ll.gemm(demb, cols, a_t=True, b_t=True)[:, :K].reshape(wshape)
        db = ll.colsum(demb).to(pdt)
        if video is not None:
            dcols = ll.gemm(demb, wp, b_t=True)                               # bf16 [B*m, Kpad]
            dnbw = ll._prenorm_wgrad(video, idx, 1, m, tubelet, patch, Kpad, rstd_pix, dcols).to(pdt)
        dpos = torch.zeros((pshape[-2], D), device=dx0.device, dtype=f32)
        # the last cls row and the patch rows: idx's cls slot (0) lands on table row k - 1
        ll.scatter_add(dx0[:, k - 1:], n * D, idx, m + 1, k - 1, B, m + 1, D, dpos)
        dcls = dx0[:, :k].sum(0)
        if k > 1:
            dpos[:k - 1] += dcls[:k - 1]
        return (None, None, dw, db, dcls.reshape(cshape).to(pdt), dpos.reshape(pshape).to(pdt), None, None, None,
                dnw, dnbw, None)


class TokenEmbedFn(torch.autograd.Function):
    """The text tower's token embedding (TextTransformer.forward_embedding, text_encoder.py:131-147): the fp32
    residual stream [B*L, D] = table[ids] + pos[:L] (ll._token_embed_fwd), and the fixed-order table and position
    gradients (ll._token_embed_bwd).  Returns (stream, int32[1] bad-id flag)."""

    @staticmethod
    def forward(ctx, ids, table, pos):
        ids = ids.contiguous()
        out, err = ll._token_embed_fwd(ids, table, pos.reshape(ids.shape[1], table.shape[1]))
        ctx.save_for_backward(ids)
        ctx.meta = (table.shape[0], table.dtype, pos.shape, pos.dtype)
        ctx.mark_non_differentiable(err)
        return out, err

    @staticmethod
    def backward(ctx, dout, _derr):
        (ids,) = ctx.saved_tensors
        V, tdt, pshape, pdt = ctx.meta
        dtable, dpos = ll._token_embed_bwd(ids, dout.contiguous().float(), V)
        return None, dtable.to(tdt), dpos.reshape(pshape).to(pdt)


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
