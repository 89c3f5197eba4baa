"""nn.Module mirror of the reference's module surface for the hot path (drop-in boundary, SURVEY §8b).

Constructor signatures, attribute names and state_dict keys follow
InternVideo2/single_modality/models/internvideo2_pretrain.py (classes at :18-403, model at :406-744),
so a reference checkpoint loads with `load_state_dict` and the model drops into
run_pretraining.get_model / engines.engine_for_pretraining.train_one_epoch.  All compute goes through
libivb200.so (ops.py); constructing the modules needs no GPU, calling them does (there is no CPU
fallback — a CPU tensor raises).
"""
from __future__ import annotations

import math
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops

bf16, f32 = torch.bfloat16, torch.float32


def to_2tuple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x)


def trunc_normal_(t, mean=0.0, std=1.0, a=-2.0, b=2.0):
    return nn.init.trunc_normal_(t, mean, std, a, b)


# ------------------------------------------------------------------------------- pos-embed tables (init only)
def _sincos_1d(dim, pos):
    omega = np.arange(dim // 2, dtype=np.float32) / (dim / 2.0)
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def get_3d_sincos_pos_embed(embed_dim, grid_size, t_size, cls_token=False):
    """Same table as models/pos_embed.py:9-54 (3/4 of the channels spatial, 1/4 temporal)."""
    assert embed_dim % 4 == 0
    ds, dt = embed_dim // 4 * 3, embed_dim // 4
    gh = np.arange(grid_size, dtype=np.float32)
    gw = np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(gw, gh), axis=0).reshape([2, 1, grid_size, grid_size])
    emb_h = _sincos_1d(ds // 2, grid[0])
    emb_w = _sincos_1d(ds // 2, grid[1])
    pos_s = np.concatenate([emb_h, emb_w], axis=1)
    pos_t = _sincos_1d(dt, np.arange(t_size, dtype=np.float32))
    pos_t = np.repeat(pos_t[:, np.newaxis, :], grid_size ** 2, axis=1)
    pos_s = np.repeat(pos_s[np.newaxis, :, :], t_size, axis=0)
    pe = np.concatenate([pos_t, pos_s], axis=-1).reshape([-1, embed_dim])
    if cls_token:
        pe = np.concatenate([np.zeros([1, embed_dim]), pe], axis=0)
    return pe


def get_2d_sincos_pos_embed(embed_dim, grid_size):
    """models/pos_embed.py:61-79 (half the channels encode h, half w; meshgrid with w first)."""
    gh = np.arange(grid_size, dtype=np.float32)
    gw = np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(gw, gh), axis=0).reshape([2, 1, grid_size, grid_size])
    return np.concatenate([_sincos_1d(embed_dim // 2, grid[0]), _sincos_1d(embed_dim // 2, grid[1])], axis=1)


def get_1d_sincos_pos_embed(embed_dim, t_size):
    """models/pos_embed.py:82-95."""
    return _sincos_1d(embed_dim, np.arange(t_size, dtype=np.float32))


class DropPath(nn.Module):
    """Per-sample stochastic depth.  In the fused Block the keep/scale factor is applied as the
    GEMM epilogue's `rowscale` (timm DropPath semantics: Bernoulli(keep)/keep, training only)."""

    def __init__(self, drop_prob=0.0):
        super().__init__()
        self.drop_prob = float(drop_prob)

    def sample(self, B, device):
        if self.drop_prob == 0.0 or not self.training:
            return None
        keep = 1.0 - self.drop_prob
        return torch.empty(B, device=device, dtype=f32).bernoulli_(keep) / keep

    def forward(self, x):
        s = self.sample(x.shape[0], x.device)
        return x if s is None else x * s.view(-1, *([1] * (x.ndim - 1))).to(x.dtype)


class RMSNorm(nn.Module):
    """internvideo2_pretrain.py:117-128.  Also accepts the fused call form `(x, residual)` of FA2's
    DropoutAddRMSNorm(prenorm=True) and then returns `(y, x + residual)`."""

    def __init__(self, hidden_size, eps=1e-6, prenorm=False, **_):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, hidden_states, residual=None):
        if residual is not None:
            res = hidden_states.float() + residual.float()
            return ops.rmsnorm(res, self.weight, self.variance_epsilon), res
        return ops.rmsnorm(hidden_states, self.weight, self.variance_epsilon)


class LayerNormB(nn.LayerNorm):
    """nn.LayerNorm parameters, ivb200 kernel."""

    def forward(self, x):
        return ops.layernorm(x, self.weight, self.bias, self.eps)


class LayerScale(nn.Module):
    """internvideo2_pretrain.py:131-146 (parameter container; the multiply is fused in GEMM epilogues)."""

    def __init__(self, dim, init_values=1e-5, inplace=False, force_fp32=False):
        super().__init__()
        self.inplace = inplace
        self.gamma = nn.Parameter(init_values * torch.ones(dim))
        self.force_fp32 = force_fp32

    def forward(self, x):
        return (x.float() * self.gamma.float()).to(x.dtype)


class Attention(nn.Module):
    """internvideo2_pretrain.py:149-217.  `use_flash_attn` is accepted for signature parity; there is
    one implementation (wgmma flash-style attention)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, attn_drop=0.0, proj_drop=0.0, use_flash_attn=False,
                 causal=False, norm_layer=nn.LayerNorm, qk_normalization=False, use_fused_rmsnorm=False):
        super().__init__()
        assert dim % num_heads == 0, "dim should be divisible by num_heads"
        if attn_drop or proj_drop or causal:
            raise NotImplementedError("ivb200 Attention: dropout / causal are not on the pre-training path")
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.qk_normalization = qk_normalization
        self.q_norm = RMSNorm(dim) if qk_normalization else nn.Identity()
        self.k_norm = RMSNorm(dim) if qk_normalization else nn.Identity()

    def forward(self, x):
        B, n, C = x.shape
        H = self.num_heads
        qkv = ops.linear(x.reshape(B * n, C), self.qkv.weight, self.qkv.bias)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        if self.qk_normalization:
            q = ops.rmsnorm(q, self.q_norm.weight, self.q_norm.variance_epsilon)
            k = ops.rmsnorm(k, self.k_norm.weight, self.k_norm.variance_epsilon)
        o = ops.AttnFn.apply(q, k, v, B, n, H, C // H, self.scale)
        return ops.linear(o, self.proj.weight, self.proj.bias).reshape(B, n, C)


class Mlp(nn.Module):
    """internvideo2_pretrain.py:220-244; `gelu_tanh=True` gives FA2 FusedMLP's activation (:269)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, bias=True,
                 drop=0.0, gelu_tanh=False, heuristic=None):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        bias = to_2tuple(bias)
        self.fc1 = nn.Linear(in_features, hidden_features, bias=bias[0])
        self.fc2 = nn.Linear(hidden_features, out_features, bias=bias[1])
        self.gelu_tanh = gelu_tanh

    def forward(self, x):
        g = ops.LinearGeluFn.apply(x, self.fc1.weight, self.fc1.bias, self.gelu_tanh)
        return ops.linear(g, self.fc2.weight, self.fc2.bias)


FusedMLP = partial(Mlp, gelu_tanh=True)


class Block(nn.Module):
    """internvideo2_pretrain.py:247-297.  Both call forms are supported: `blk(x)` (naive, returns x) and
    `blk(x, residual)` (fused pre-norm form, returns `(branch, residual)` such that x_out = branch + residual)."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, drop=0.0, attn_drop=0.0, init_values=None,
                 drop_path=0.0, act_layer=nn.GELU, norm_layer=nn.LayerNorm, use_flash_attn=False,
                 use_fused_mlp=False, fused_mlp_heuristic=1, with_cp=False, qk_normalization=False,
                 layerscale_no_force_fp32=False, use_fused_rmsnorm=False):
        super().__init__()
        self.norm1 = RMSNorm(dim, eps=1e-6)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, attn_drop=attn_drop, proj_drop=drop,
                              use_flash_attn=use_flash_attn, qk_normalization=qk_normalization)
        self.ls1 = LayerScale(dim, init_values=init_values,
                              force_fp32=(not layerscale_no_force_fp32)) if init_values else nn.Identity()
        self.drop_path1 = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm2 = RMSNorm(dim, eps=1e-6)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop,
                       gelu_tanh=bool(use_fused_mlp))
        self.ls2 = LayerScale(dim, init_values=init_values,
                              force_fp32=(not layerscale_no_force_fp32)) if init_values else nn.Identity()
        self.drop_path2 = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        # activation checkpointing (reference :294-295): only the block input is kept, backward recomputes the
        # forward (ops.BlockFn).  Unnecessary for the 1B recipe on an 80 GB H100, needed for 6B / large unmasked batches
        self.with_cp = bool(with_cp)
        self.use_fused_rmsnorm = use_fused_rmsnorm
        self.num_heads = num_heads

    def forward_stream(self, x2d, B, n, rowscale=None):
        """fp32 residual stream [B*n, D] -> [B*n, D] (the hot path used by the model).
        rowscale: optional (rs1, rs2) fp32 [B*n] DropPath factors sampled by the caller for all blocks at once."""
        a = self.attn
        g1 = self.ls1.gamma if isinstance(self.ls1, LayerScale) else None
        g2 = self.ls2.gamma if isinstance(self.ls2, LayerScale) else None
        rs1 = rs2 = None
        if rowscale is not None:
            rs1, rs2 = rowscale
        elif isinstance(self.drop_path1, DropPath):   # per-sample stochastic depth -> per-row epilogue scale
            s1 = self.drop_path1.sample(B, x2d.device)
            s2 = self.drop_path2.sample(B, x2d.device)
            rs1 = s1.repeat_interleave(n) if s1 is not None else None
            rs2 = s2.repeat_interleave(n) if s2 is not None else None
        if not torch.is_grad_enabled():
            return self.forward_infer(x2d, B, n, (rs1, rs2))
        return ops.BlockFn.apply(
            x2d, (B, n, self.num_heads, self.mlp.gelu_tanh, self.with_cp), self.norm1.weight, a.qkv.weight, a.qkv.bias,
            a.q_norm.weight if a.qk_normalization else None, a.k_norm.weight if a.qk_normalization else None,
            a.proj.weight, a.proj.bias, g1, self.norm2.weight, self.mlp.fc1.weight, self.mlp.fc1.bias,
            self.mlp.fc2.weight, self.mlp.fc2.bias, g2, rs1, rs2)

    def _param_tuple(self):
        a = self.attn
        g1 = self.ls1.gamma if isinstance(self.ls1, LayerScale) else None
        g2 = self.ls2.gamma if isinstance(self.ls2, LayerScale) else None
        return (self.norm1.weight, a.qkv.weight, a.qkv.bias,
                a.q_norm.weight if a.qk_normalization else None, a.k_norm.weight if a.qk_normalization else None,
                a.proj.weight, a.proj.bias, g1, self.norm2.weight, self.mlp.fc1.weight, self.mlp.fc1.bias,
                self.mlp.fc2.weight, self.mlp.fc2.bias, g2)

    def forward_infer(self, x2d, B, n, rowscale=(None, None)):
        """No-grad form (frozen towers / teachers): 14 kernels, nothing saved, no GELU' / pre-LayerScale copies."""
        with torch.no_grad():
            out, _ = ops.block_forward(x2d, (B, n, self.num_heads, self.mlp.gelu_tanh), self._param_tuple(),
                                       rowscale[0], rowscale[1], save=False)
        return out

    def forward(self, x, residual=None):
        B, n, D = x.shape
        if residual is not None:
            xin = (x.float() + residual.float()).reshape(B * n, D)
            out = self.forward_stream(xin, B, n).reshape(B, n, D)
            return torch.zeros_like(x), out.to(residual.dtype)
        out = self.forward_stream(x.float().reshape(B * n, D).contiguous(), B, n)
        return out.reshape(B, n, D).to(x.dtype)


class PatchEmbed(nn.Module):
    """internvideo2_pretrain.py:300-331 — Conv3d(k=s=(tubelet,p,p)) as an im2col GEMM on wgmma."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, num_frames=8, tubelet_size=1,
                 norm_layer=None):
        super().__init__()
        img_size = to_2tuple(img_size)
        patch_size = to_2tuple(patch_size)
        self.img_size, self.patch_size, self.tubelet_size = img_size, patch_size, tubelet_size
        self.grid_size = (num_frames // tubelet_size, img_size[0] // patch_size[0], img_size[1] // patch_size[1])
        self.num_patches = self.grid_size[0] * self.grid_size[1] * self.grid_size[2]
        self.proj = nn.Conv3d(in_chans, embed_dim, kernel_size=(tubelet_size, patch_size[0], patch_size[1]),
                              stride=(tubelet_size, patch_size[0], patch_size[1]))
        if norm_layer:
            raise NotImplementedError("PatchEmbed norm_layer is not used on this path")
        self.norm = nn.Identity()

    def forward(self, x):
        """All-token embed [B,C,T,H,W] -> [B, T', L, D] (bf16), same layout as the reference."""
        B, C, T, H, W = x.shape
        D = self.proj.weight.shape[0]
        N = self.num_patches
        idx = torch.arange(0, N + 1, device=x.device, dtype=torch.int32).repeat(B, 1).contiguous()
        zeros_tab = torch.zeros((N + 1, D), device=x.device, dtype=bf16)
        zcls = torch.zeros((1, 1, D), device=x.device, dtype=bf16)
        out = ops.EmbedFn.apply(x.to(bf16), idx, self.proj.weight, self.proj.bias, zcls, zeros_tab,
                                self.tubelet_size, self.patch_size[0])
        out = out.reshape(B, N + 1, D)[:, 1:]
        return out.reshape(B, self.grid_size[0], self.grid_size[1] * self.grid_size[2], D).to(bf16)


class CrossAttention(nn.Module):
    """internvideo2_pretrain.py:18-80 (parameter layout); used by the attention-pooling head."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0.0, proj_drop=0.0,
                 attn_head_dim=None, out_dim=None):
        super().__init__()
        out_dim = out_dim or dim
        self.num_heads = num_heads
        head_dim = attn_head_dim if attn_head_dim is not None else dim // num_heads
        all_head_dim = head_dim * num_heads
        self.scale = qk_scale or head_dim ** -0.5
        assert all_head_dim == dim
        self.q = nn.Linear(dim, all_head_dim, bias=False)
        self.k = nn.Linear(dim, all_head_dim, bias=False)
        self.v = nn.Linear(dim, all_head_dim, bias=False)
        if qkv_bias:
            self.q_bias = nn.Parameter(torch.zeros(all_head_dim))
            self.k_bias = nn.Parameter(torch.zeros(all_head_dim))
            self.v_bias = nn.Parameter(torch.zeros(all_head_dim))
        else:
            self.q_bias = self.k_bias = self.v_bias = None
        self.proj = nn.Linear(all_head_dim, out_dim)

    def forward(self, x, k=None, v=None, return_attn=False):
        """return_attn (teacher form, internvl_clip_vision.py:55-88): also returns the head-averaged attention
        [B, Nk] of the single query (inference only)."""
        B, Nq, C = x.shape
        Nk = k.shape[1]
        H = self.num_heads
        q = ops.linear(x, self.q.weight, self.q_bias)
        kk = ops.linear(k, self.k.weight, self.k_bias)
        vv = ops.linear(v, self.v.weight, self.v_bias)
        if Nq != 1:
            raise NotImplementedError("ivb200 CrossAttention: only the 1-query pooling form is on the path")
        d = C // H
        if return_attn:
            o, probs = ll.pool_attn_fwd(q.reshape(B, C).contiguous(), kk.reshape(B * Nk, C), vv.reshape(B * Nk, C),
                                        B, Nk, H, d, self.scale)
            return ops.linear(o.reshape(B, 1, C), self.proj.weight, self.proj.bias), probs.mean(1)
        o = ops.PoolAttnFn.apply(q.reshape(B, C), kk.reshape(B * Nk, C), vv.reshape(B * Nk, C), B, Nk, H, d,
                                 self.scale).reshape(B, 1, C)
        return ops.linear(o, self.proj.weight, self.proj.bias)


class AttentiveBlock(nn.Module):
    """internvideo2_pretrain.py:83-104."""

    def __init__(self, dim, num_heads, qkv_bias=False, qk_scale=None, drop=0.0, attn_drop=0.0, drop_path=0.0,
                 norm_layer=nn.LayerNorm, attn_head_dim=None, out_dim=None):
        super().__init__()
        eps = getattr(norm_layer(8), "eps", 1e-5) if norm_layer is not None else 1e-5
        self.norm1_q = LayerNormB(dim, eps=eps)
        self.norm1_k = LayerNormB(dim, eps=eps)
        self.norm1_v = LayerNormB(dim, eps=eps)
        self.cross_attn = CrossAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale,
                                         attn_drop=attn_drop, proj_drop=drop, attn_head_dim=attn_head_dim,
                                         out_dim=out_dim)

    def forward(self, x_q, x_kv, pos_q, pos_k, bool_masked_pos, rel_pos_bias=None, return_attn=False):
        x_q = self.norm1_q(x_q + pos_q)
        x_k = self.norm1_k(x_kv + pos_k)
        x_v = self.norm1_v(x_kv)
        return self.cross_attn(x_q, k=x_k, v=x_v, return_attn=return_attn)


class AttentionPoolingBlock(AttentiveBlock):
    """internvideo2_pretrain.py:107-114."""

    def forward(self, x, return_attn=False):
        x_q = x.mean(1, keepdim=True)
        if return_attn:
            o, attn = super().forward(x_q, x, 0, 0, bool_masked_pos=None, rel_pos_bias=None, return_attn=True)
            return o.squeeze(1), attn
        return super().forward(x_q, x, 0, 0, bool_masked_pos=None, rel_pos_bias=None).squeeze(1)


class Linear_Decoder(nn.Module):
    """internvideo2_pretrain.py:334-365."""

    def __init__(self, in_channels=1408, out_channels=3200, norm_layer=nn.LayerNorm, norm_type="l2"):
        super().__init__()
        self.norm_type = norm_type
        self.head = nn.Linear(in_channels, out_channels)
        self.norm = LayerNormB(out_channels, eps=getattr(norm_layer(8), "eps", 1e-5))
        nn.init.xavier_uniform_(self.head.weight)
        nn.init.constant_(self.head.bias, 0)

    def pre_norm(self, x):
        return ops.linear(x, self.head.weight, self.head.bias)

    def forward(self, x):
        z = self.pre_norm(x)
        if self.norm_type == "l2":
            return ops.LnL2Fn.apply(z, self.norm.weight, self.norm.bias, self.norm.eps)
        if self.norm_type == "none":
            return self.norm(z)
        raise NotImplementedError

    def align_loss(self, x, target):
        """(2 - 2 <forward(x), target>).mean() with the normalised features never materialised."""
        assert self.norm_type == "l2"
        return ops.AlignLossFn.apply(self.pre_norm(x), self.norm.weight, self.norm.bias, target, self.norm.eps)


class MLP_Decoder(Linear_Decoder):
    """internvideo2_pretrain.py:368-403."""

    def __init__(self, in_channels=768, out_channels=768, norm_layer=nn.LayerNorm, norm_type="l2"):
        nn.Module.__init__(self)
        self.norm_type = norm_type
        self.head = nn.Sequential(nn.Linear(in_channels, in_channels), nn.GELU(), nn.Linear(in_channels, out_channels))
        self.norm = LayerNormB(out_channels, eps=getattr(norm_layer(8), "eps", 1e-5))
        for m in (self.head[0], self.head[2]):
            nn.init.xavier_uniform_(m.weight)
            nn.init.constant_(m.bias, 0)

    def pre_norm(self, x):
        g = ops.LinearGeluFn.apply(x, self.head[0].weight, self.head[0].bias, False)
        return ops.linear(g, self.head[2].weight, self.head[2].bias)


class PretrainInternVideo2(nn.Module):
    """internvideo2_pretrain.py:406-744 — same ctor kwargs, same state_dict keys, same forward contract:
    forward(x[B,3,T,H,W], mask[B,1+T*L] bool) -> (x_clip_align[K,B,n,Ct], x_align[B,Cf], x_mae_align[K',B,n-1,Cm]).
    """

    def __init__(self, in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.25,
                 embed_dim=1408, num_heads=16, mlp_ratio=4.3637, init_values=1e-5, qk_normalization=True,
                 depth=40, use_flash_attn=True, use_fused_rmsnorm=True, use_fused_mlp=True, fused_mlp_heuristic=1,
                 attn_pool_num_heads=16, clip_embed_dim=768, layerscale_no_force_fp32=False, num_frames=8,
                 tubelet_size=1, sep_pos_embed=False, use_checkpoint=False, checkpoint_num=0,
                 clip_teacher_embed_dim=3200, clip_teacher_final_dim=768, clip_norm_type="l2", clip_return_layer=1,
                 clip_student_return_interval=1, mae_teacher_embed_dim=1408, mae_norm_type="l2", mae_return_layer=1,
                 mae_student_return_interval=1):
        super().__init__()
        assert use_flash_attn == use_fused_rmsnorm == use_fused_mlp, \
            "use_flash_attn, use_fused_rmsnorm and use_fused_mlp should be consistent"
        self.use_flash_attn = use_flash_attn
        self.embed_dim = embed_dim
        self.depth = depth
        self.clip_norm_type, self.mae_norm_type = clip_norm_type, mae_norm_type
        self.clip_return_index = [depth - int(i * clip_student_return_interval) - 1 for i in range(clip_return_layer)]
        self.mae_return_index = [depth - int(i * mae_student_return_interval) - 1 for i in range(mae_return_layer)]
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim, num_frames=num_frames,
                                      tubelet_size=tubelet_size)
        num_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.sep_pos_embed = bool(sep_pos_embed)
        if self.sep_pos_embed:      # :481-493 — separable spatial / temporal / cls tables, one set per consumer
            gs = self.grid_size = self.patch_embed.grid_size
            Z = lambda *shape: nn.Parameter(torch.zeros(*shape))  # noqa: E731
            self.pos_embed_spatial, self.pos_embed_temporal = Z(1, gs[1] * gs[2], embed_dim), Z(1, gs[0], embed_dim)
            self.pos_embed_cls = Z(1, 1, embed_dim)
            self.clip_pos_embed_spatial, self.clip_pos_embed_temporal = Z(1, gs[1] * gs[2], embed_dim), Z(1, gs[0], embed_dim)
            self.clip_pos_embed_cls = Z(1, 1, embed_dim)
            self.mae_pos_embed_spatial, self.mae_pos_embed_temporal = Z(1, gs[1] * gs[2], embed_dim), Z(1, gs[0], embed_dim)
        else:
            self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim))
            self.clip_pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim))
            self.mae_pos_embed = nn.Parameter(torch.zeros(1, num_patches, embed_dim))
        dpr = [drop_path_rate * i / (depth - 1) if depth > 1 else 0.0 for i in range(depth)]  # == linspace(0, r, depth)
        with_cp = [bool(use_checkpoint) and i < checkpoint_num for i in range(depth)]           # :503-507
        self.blocks = nn.ModuleList([
            Block(embed_dim, num_heads, mlp_ratio, qkv_bias=qkv_bias, norm_layer=RMSNorm, drop_path=dpr[i],
                  init_values=init_values, attn_drop=0.0, use_flash_attn=use_flash_attn, use_fused_mlp=use_fused_mlp,
                  fused_mlp_heuristic=fused_mlp_heuristic, with_cp=with_cp[i], qk_normalization=qk_normalization,
                  layerscale_no_force_fp32=layerscale_no_force_fp32, use_fused_rmsnorm=use_fused_rmsnorm)
            for i in range(depth)])
        self.clip_projector = AttentionPoolingBlock(dim=embed_dim, num_heads=attn_pool_num_heads, qkv_bias=True,
                                                    qk_scale=None, drop=0.0, attn_drop=0.0,
                                                    norm_layer=partial(nn.LayerNorm, eps=1e-5), out_dim=clip_embed_dim)
        ln = partial(nn.LayerNorm, eps=1e-5)
        self.clip_decoder = nn.ModuleList([
            Linear_Decoder(embed_dim, clip_teacher_embed_dim, norm_layer=ln, norm_type=clip_norm_type)
            for _ in range(clip_return_layer)])
        self.final_clip_decoder = nn.Identity()
        if clip_teacher_final_dim > 0:
            self.final_clip_decoder = Linear_Decoder(clip_embed_dim, clip_teacher_final_dim, norm_layer=ln,
                                                     norm_type=clip_norm_type)
        self.mae_decoder = nn.ModuleList([
            MLP_Decoder(embed_dim, mae_teacher_embed_dim, norm_layer=ln, norm_type=mae_norm_type)
            for _ in range(mae_return_layer)])
        self.init_pos_embed()
        trunc_normal_(self.cls_token, std=0.02)
        self.apply(self._init_weights)
        self.fix_init_weight()

    # ---- init (internvideo2_pretrain.py:560-603)
    def init_pos_embed(self):
        gs = self.patch_embed.grid_size
        if self.sep_pos_embed:
            D = self.pos_embed_spatial.shape[-1]
            sp = torch.from_numpy(get_2d_sincos_pos_embed(D, gs[1])).float().unsqueeze(0)
            tp = torch.from_numpy(get_1d_sincos_pos_embed(D, gs[0])).float().unsqueeze(0)
            for pre in ("", "clip_", "mae_"):
                getattr(self, pre + "pos_embed_spatial").data.copy_(sp)
                getattr(self, pre + "pos_embed_temporal").data.copy_(tp)
            return
        pe = get_3d_sincos_pos_embed(self.pos_embed.shape[-1], gs[1], gs[0], cls_token=True)
        t = torch.from_numpy(pe).float().unsqueeze(0)
        self.pos_embed.data.copy_(t)
        self.clip_pos_embed.data.copy_(t)
        self.mae_pos_embed.data.copy_(t[:, 1:])

    def _pos_table(self, which):
        """The [1, 1+T*L, D] ('' / 'clip_') or [1, T*L, D] ('mae_') position table: the joint parameter, or the
        separable tables composed exactly like :640-656 / :700-711 / :727-734 (torch glue, O(N*D), differentiable)."""
        if not self.sep_pos_embed:
            return getattr(self, which + "pos_embed")
        gs = self.grid_size
        sp, tp = getattr(self, which + "pos_embed_spatial"), getattr(self, which + "pos_embed_temporal")
        pe = sp.repeat(1, gs[0], 1) + torch.repeat_interleave(tp, gs[1] * gs[2], dim=1)
        if which == "mae_":
            return pe
        return torch.cat([getattr(self, which + "pos_embed_cls").expand(pe.shape[0], -1, -1), pe], 1)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def fix_init_weight(self):
        for layer_id, layer in enumerate(self.blocks):
            layer.attn.proj.weight.data.div_(math.sqrt(2.0 * (layer_id + 1)))
            layer.mlp.fc2.weight.data.div_(math.sqrt(2.0 * (layer_id + 1)))

    @property
    def dtype(self):
        return self.patch_embed.proj.weight.dtype

    def get_num_layers(self):
        return len(self.blocks)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_embed", "pos_embed_spatial", "pos_embed_temporal", "pos_embed_cls", "cls_token",
                "clip_pos_embed", "clip_pos_embed_spatial", "clip_pos_embed_temporal", "clip_pos_embed_cls",
                "mae_pos_embed", "mae_pos_embed_spatial", "mae_pos_embed_temporal"}

    # ---- the hot path
    def _check(self):
        if self.dtype != bf16:
            raise ll._lib.IvbError("ivb200 PretrainInternVideo2 computes in bf16: call model.bfloat16() first "
                                   "(engine_for_pretraining.py:128 does the same in the reference's bf16 mode)")

    def visible_index(self, mask, n_visible=None):
        """int32 [B, n] positions of the kept tokens in `x[~mask]` order (bit-exact)."""
        if n_visible is None:
            n_visible = int(mask.shape[1] - int(mask[0].sum()))   # one tiny D2H when the mask lives on the GPU
        idx, err = ll.visible_indices(mask.to(self.cls_token.device, non_blocking=True), n_visible)
        return idx, err, n_visible

    def forward_features(self, x, mask, n_visible=None, drop_path_factors=None):
        """-> (taps: dict block_idx -> fp32 [B*n, D], final fp32 [B*n, D], idx int32 [B,n], B, n).
        drop_path_factors: optional fp32 [2*depth, B] per-sample stochastic-depth factors (Bernoulli(keep)/keep;
        rows 2i, 2i+1 = the two branches of block i) used instead of a fresh draw — parity tests inject the
        draw the reference made (SURVEY App.B-16: RNG-dependent pieces are injected, not compared)."""
        self._check()
        if not x.is_cuda:
            raise ll._lib.IvbError("ivb200 PretrainInternVideo2: input must be a CUDA tensor (no CPU fallback)")
        B = x.shape[0]
        idx, err, n = self.visible_index(mask, n_visible)
        self.index_error = err       # int32[1] on the device: 0, or 1 + (a clip whose visible-token count != n)
        pe = self.patch_embed
        h = ops.EmbedFn.apply(x.to(bf16), idx, pe.proj.weight, pe.proj.bias, self.cls_token, self._pos_table(""),
                              pe.tubelet_size, pe.patch_size[0])
        taps = {}
        if drop_path_factors is not None:
            rs_all = drop_path_factors.to(device=h.device, dtype=f32).repeat_interleave(n, dim=1).contiguous()
        else:
            rs_all = self._sample_drop_path(B, n, h.device)
        for i, blk in enumerate(self.blocks):
            h = blk.forward_stream(h, B, n, None if rs_all is None else (rs_all[2 * i], rs_all[2 * i + 1]))
            if i in self.clip_return_index or i in self.mae_return_index:
                taps[i] = h
        return taps, h, idx, B, n

    def _sample_drop_path(self, B, n, device):
        """Per-sample stochastic-depth factors of ALL blocks in one shot: fp32 [2*depth, B*n] (timm DropPath:
        Bernoulli(keep)/keep per sample, independently for the attention and the MLP branch), or None in eval /
        when every rate is 0.  The factors are consumed as the `rowscale` of the residual GEMM epilogues."""
        if not self.training:
            return None
        cache = getattr(self, "_dp_keep", None)
        if cache is None or cache[0] != device:
            rates = []
            for blk in self.blocks:
                for dp in (blk.drop_path1, blk.drop_path2):
                    rates.append(dp.drop_prob if isinstance(dp, DropPath) else 0.0)
            keep_t = None if max(rates) == 0.0 else 1.0 - torch.tensor(rates, device=device, dtype=f32)[:, None]
            cache = self._dp_keep = (device, keep_t)      # built once (eagerly), reused inside CUDA-graph capture
        keep = cache[1]
        if keep is None:
            return None
        m = (torch.rand((keep.shape[0], B), device=device, dtype=f32) < keep).to(f32) / keep
        return m.repeat_interleave(n, dim=1).contiguous()

    def _decoder_inputs(self, taps, idx, B, n):
        cpe, mpe = self._pos_table("clip_"), self._pos_table("mae_")
        clip_in = [ops.GatherAddFn.apply(taps[i], cpe, idx, B, n, 0, 0) for i in sorted(self.clip_return_index)]
        mae_in = [ops.GatherAddFn.apply(taps[i], mpe, idx, B, n, 1, -1) for i in sorted(self.mae_return_index)]
        return clip_in, mae_in

    def forward(self, x, mask, n_visible=None, drop_path_factors=None):
        taps, h, idx, B, n = self.forward_features(x, mask, n_visible, drop_path_factors)
        D = self.embed_dim
        pooled = self.clip_projector(h.reshape(B, n, D))                       # bf16 [B, clip_embed_dim]
        clip_in, mae_in = self._decoder_inputs(taps, idx, B, n)
        x_clip_align = torch.stack([dec(xi).reshape(B, n, -1) for dec, xi in zip(self.clip_decoder, clip_in)])
        x_align = self.final_clip_decoder(pooled)
        x_align = x_align + self._index_poison().to(x_align.dtype)      # ragged mask -> NaN, no sync (see forward_loss)
        x_mae_align = torch.stack([dec(xi).reshape(B, n - 1, -1) for dec, xi in zip(self.mae_decoder, mae_in)])
        return x_clip_align, x_align, x_mae_align

    def forward_loss(self, x, mask, tgt_clip, tgt_final, tgt_mae, n_visible=None, drop_path_factors=None):
        """Student forward + the three alignment losses of engine_for_pretraining.py:131-148 with the
        LayerNorm -> L2 -> (2-2cos) tail fused (the [K,B,n,3200] normalised features are never written).
        Returns (loss_clip, loss_final, loss_mae)."""
        taps, h, idx, B, n = self.forward_features(x, mask, n_visible, drop_path_factors)
        D = self.embed_dim
        pooled = self.clip_projector(h.reshape(B, n, D))
        clip_in, mae_in = self._decoder_inputs(taps, idx, B, n)
        K = len(clip_in)
        loss_clip = sum(dec.align_loss(xi, tgt_clip[k]) for k, (dec, xi) in enumerate(zip(self.clip_decoder, clip_in))) / K
        if isinstance(self.final_clip_decoder, Linear_Decoder):
            loss_final = self.final_clip_decoder.align_loss(pooled, tgt_final)
        else:
            loss_final = (2 - 2 * (pooled.float() * tgt_final.float()).sum(-1)).mean()
        Km = len(mae_in)
        loss_mae = sum(dec.align_loss(xi, tgt_mae[k]) for k, (dec, xi) in enumerate(zip(self.mae_decoder, mae_in))) / Km
        # a mask whose rows keep different numbers of tokens cannot be reshaped to [B, n, C] (the reference raises at
        # :659); here the flag lives on the device, so it is surfaced without a sync: the loss becomes NaN
        # (and engine.step(check_finite=True) skips the update)
        loss_final = loss_final + self._index_poison()
        return loss_clip, loss_final, loss_mae

    def _index_poison(self):
        z = torch.zeros((), device=self.index_error.device, dtype=f32)
        return torch.where(self.index_error[0] != 0, torch.full_like(z, float("nan")), z)


def pretrain_internvideo2_1B_patch14_224(pretrained=False, **kwargs):
    """internvideo2_pretrain.py:747-755."""
    return PretrainInternVideo2(img_size=224, patch_size=14, embed_dim=1408, depth=40, num_heads=16,
                                mlp_ratio=48 / 11, attn_pool_num_heads=16, clip_embed_dim=768, **kwargs)


def pretrain_internvideo2_6B_patch14_224(pretrained=False, **kwargs):
    """internvideo2_pretrain.py:758-766."""
    return PretrainInternVideo2(img_size=224, patch_size=14, embed_dim=3200, depth=48, num_heads=25,
                                mlp_ratio=4, attn_pool_num_heads=16, clip_embed_dim=768, **kwargs)
