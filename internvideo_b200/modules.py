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


def get_3d_sincos_pos_embed(embed_dim, grid_size, t_size, cls_token=False, cls_token_num=1):
    """Same table as models/pos_embed.py:9-54 (3/4 of the channels spatial, 1/4 temporal), behind cls_token_num zero
    rows with cls_token (InternVideo-Next/models/pos_embed.py:9-54)."""
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
        pe = np.concatenate([np.zeros([cls_token_num, embed_dim]), pe], axis=0)
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


def get_sinusoid_encoding_table(n_position, d_hid):
    """The VideoMAE towers' fixed table (IV1 modeling_finetune.py:224-242; videomae.py:152-205 for the recipe case
    n_position == pre_n_position, no interpolation): [1, n_position, d_hid] fp32, sin on even / cos on odd channels."""
    pos = np.arange(n_position, dtype=np.float64)[:, None]
    j = np.arange(d_hid)[None, :]
    table = pos / np.power(10000, 2 * (j // 2) / d_hid)
    table[:, 0::2] = np.sin(table[:, 0::2])
    table[:, 1::2] = np.cos(table[:, 1::2])
    return torch.tensor(table, dtype=torch.float).unsqueeze(0)


def _pos_tensor(a):
    """numpy table -> a new fp32 [1, rows, D] tensor."""
    return torch.tensor(a, dtype=torch.float).unsqueeze(0)


# ------------------------------------------------------------------------------- pieces every tower shares
def init_weights(m):
    """The towers' Linear / LayerNorm init (internvideo2_pretrain.py:589-597, videomae.py:238-245)."""
    if isinstance(m, nn.Linear):
        trunc_normal_(m.weight, std=0.02)
        if m.bias is not None:
            nn.init.constant_(m.bias, 0)
    elif isinstance(m, nn.LayerNorm):
        nn.init.constant_(m.bias, 0)
        nn.init.constant_(m.weight, 1.0)


def check_input(tower, x, dtype):
    """The refusal at the top of every tower forward: the parameters must be bf16 and the input a CUDA tensor."""
    if dtype != bf16:
        raise ll._lib.IvbError(f"ivb200 {type(tower).__name__} computes in bf16: call model.bfloat16() first")
    if not x.is_cuda:
        raise ll._lib.IvbError(f"ivb200 {type(tower).__name__}: input must be a CUDA tensor (no CPU fallback)")


def index_poison(err):
    """0, or NaN when the int32[1] device flag of a visible-token index build is set (the clips of a ragged mask keep
    different numbers of tokens): added to an output, it surfaces the error without a host sync."""
    z = torch.zeros((), device=err.device, dtype=f32)
    return torch.where(err[0] != 0, torch.full_like(z, float("nan")), z)


def embed_tokens(patch_embed, x, idx, cls_token, table):
    """The token front-end of every tower (ops.EmbedFn): the patch embed's Conv3d on the tokens idx[:, 1:] names, as an
    im2col + wgmma GEMM, plus their rows of the position table, behind `cls_token + table[0]`.  x: video [B,C,T,H,W];
    idx: int32 [B, n], column 0 the cls slot.  Returns the fp32 residual stream [B*n, D].
    cls_token None (towers without one): `table` holds the patch rows only; EmbedFn gets a zero cls token and a zero
    table row, and the cls row is dropped again, giving [B*(n-1), D].  A cls_token [1, k, D] puts k cls rows in front
    (the stream is then [B*(k+n-1), D]), and a patch embed with `norm_before` (InternVideo-Next's dual-RMSNorm
    PatchEmbed) runs its two norms inside EmbedFn."""
    tubelet, patch, _ = patch_embed.proj.kernel_size
    w, b = patch_embed.proj.weight, patch_embed.proj.bias
    nb = getattr(patch_embed, "norm_before", None)
    norms = () if nb is None else (patch_embed.norm.weight, nb.weight, nb.variance_epsilon)
    if cls_token is not None:
        return ops.EmbedFn.apply(x.to(bf16), idx, w, b, cls_token, table, tubelet, patch, cls_token.shape[1], *norms)
    B, n = idx.shape
    D = w.shape[0]
    table = torch.cat([table.new_zeros(1, 1, D), table], 1).to(bf16)
    zcls = torch.zeros((1, 1, D), device=x.device, dtype=bf16)
    h = ops.EmbedFn.apply(x.to(bf16), idx, w, b, zcls, table, tubelet, patch, 1, *norms)
    return h.reshape(B, n, D)[:, 1:].reshape(B * (n - 1), D)


def run_blocks(blocks, h, call, taps=(), last=None):
    """Runs blocks 0..last (all when `last` is no block index) over the stream h, block i as `call(i, block, h)`.
    Returns the final stream and {i: output of block i} for each i in `taps`, in block order."""
    out = {}
    for i, blk in enumerate(blocks):
        h = call(i, blk, h)
        if i in taps:
            out[i] = h
        if i == last:
            break
    return h, out


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


class Fp8InferenceSwitch:
    """The switch set_fp8_inference sets on a module, read when it runs: fp8_inference holds the Fp8InferenceWeights of
    its _fp8_linears() while the mode is on (None when off), fp8_attention whether set_fp8_inference(attention=True)
    asked for attention on the FP8 tensor cores too."""
    fp8_inference = None
    fp8_attention = False

    def _fp8_linears(self):
        raise NotImplementedError


class Fp8Block(Fp8InferenceSwitch):
    """The fused blocks both FP8 switches set (Block, VideoMAEBlock, text_modules.TransformerEncoder): set_fp8's
    training mode, its scaling, "tensor" or "token", and with "token" whether the weight gradients run in FP8 too, read
    at call time through block_precision; and set_fp8_inference's switch."""
    fp8 = False
    fp8_scaling = "tensor"
    fp8_wgrad = False

    def _fp8_linears(self):
        """The block's four GEMM weights' Linears: qkv, proj, fc1, fc2."""
        a, mlp = self.attn, self.mlp
        return (a.qkv, a.proj, mlp.fc1, mlp.fc2)


class Block(Fp8Block, nn.Module):
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

    def forward_stream(self, x2d, B, n, rowscale=None, plans=None):
        """fp32 residual stream [B*n, D] -> [B*n, D] (the hot path used by the model).
        rowscale: optional (rs1, rs2) fp32 [B*n] DropPath factors sampled by the caller for all blocks at once.
        plans: optional (plan1, plan2) DropPath plans of those factors (ops.droppath_plan rows, None for a branch
        without one): the training GEMMs then skip the rows the draw dropped."""
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
        return ops.BlockFn.apply(x2d, self._spec(B, n, training=True), rs1, rs2, *self._param_tuple(),
                                 *(plans or ()))

    def _spec(self, B, n, training):
        return ops.BlockSpec(B, n, self.num_heads, self.mlp.gelu_tanh, eps1=self.norm1.variance_epsilon,
                             eps2=self.norm2.variance_epsilon, checkpoint=self.with_cp,
                             precision=block_precision(self, training), attn_fp8=block_attn_fp8(self))

    def _param_tuple(self):
        a = self.attn
        return ops.BlockParams(
            n1w=self.norm1.weight, qkvw=a.qkv.weight, qkvb=a.qkv.bias,
            qnw=a.q_norm.weight if a.qk_normalization else None, knw=a.k_norm.weight if a.qk_normalization else None,
            projw=a.proj.weight, projb=a.proj.bias, g1=self.ls1.gamma if isinstance(self.ls1, LayerScale) else None,
            n2w=self.norm2.weight, fc1w=self.mlp.fc1.weight, fc1b=self.mlp.fc1.bias, fc2w=self.mlp.fc2.weight,
            fc2b=self.mlp.fc2.bias, g2=self.ls2.gamma if isinstance(self.ls2, LayerScale) else None)

    def forward_infer(self, x2d, B, n, rowscale=(None, None)):
        """No-grad form (frozen towers / teachers): ops.block_forward with nothing saved, no GELU' / pre-LayerScale
        copies."""
        with torch.no_grad():
            out, _ = ops.block_forward(x2d, self._spec(B, n, training=False), self._param_tuple(), rowscale[0],
                                       rowscale[1], save=False)
        return out

    def forward(self, x, residual=None):
        B, n, D = x.shape
        if residual is not None:
            xin = (x.float() + residual.float()).reshape(B * n, D)
            out = self.forward_stream(xin, B, n).reshape(B, n, D)
            return torch.zeros_like(x), out.to(residual.dtype)
        out = self.forward_stream(x.float().reshape(B * n, D).contiguous(), B, n)
        return out.reshape(B, n, D).to(x.dtype)


class VideoMAEAttention(nn.Module):
    """Parameters of the VideoMAE attention (videomae.py:62-101, IV1 modeling_finetune.py:77-129): qkv without bias plus
    separate q_bias / v_bias.  Both fused block paths need heads * head_dim == dim."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_head_dim=None):
        super().__init__()
        head_dim = attn_head_dim if attn_head_dim is not None else dim // num_heads
        if head_dim * num_heads != dim:
            raise NotImplementedError(f"ivb200 VideoMAEAttention: heads * head_dim ({num_heads} * {head_dim}) must be "
                                      f"dim ({dim})")
        self.num_heads = num_heads
        self.scale = qk_scale or head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=False)
        if qkv_bias:
            self.q_bias = nn.Parameter(torch.zeros(dim))
            self.v_bias = nn.Parameter(torch.zeros(dim))
        else:
            self.q_bias = self.v_bias = None
        self.proj = nn.Linear(dim, dim)

    def qkv_bias_vector(self):
        """q_bias | 0 | v_bias (k has no bias), or None."""
        if self.q_bias is None:
            return None
        return torch.cat((self.q_bias, torch.zeros_like(self.v_bias), self.v_bias))


class VideoMAEBlock(Fp8Block, nn.Module):
    """The VideoMAE LayerNorm block (videomae.py:104-132 for the VideoMAEv2 teacher, IV1 modeling_finetune.py:132-181):
    LayerNorm pre-norm, q/v-bias attention, erf GELU MLP, optional gamma_1 / gamma_2, through ops.block_forward with
    spec.layernorm and, when trained, ops.BlockFn.  with_cp: keep only the block input and recompute its forward in
    backward (IV1's with_cp)."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop=0.0, attn_drop=0.0,
                 drop_path=0.0, init_values=None, act_layer=nn.GELU, norm_layer=nn.LayerNorm, attn_head_dim=None,
                 with_cp=False):
        super().__init__()
        if drop or attn_drop:
            raise NotImplementedError("ivb200 VideoMAEBlock: dropout is 0 in every recipe")
        self.norm1 = norm_layer(dim)
        self.attn = VideoMAEAttention(dim, num_heads, qkv_bias, qk_scale, attn_head_dim)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        if init_values and init_values > 0:
            self.gamma_1 = nn.Parameter(init_values * torch.ones(dim))
            self.gamma_2 = nn.Parameter(init_values * torch.ones(dim))
        else:
            self.gamma_1 = self.gamma_2 = None
        self.drop_prob = float(drop_path)
        self.with_cp = bool(with_cp)

    def _drop_path_rows(self, B, n, device):
        """IV1's DropPath draw (timm drop_path: Bernoulli(keep) / keep per sample, `rand < keep`), once per branch in
        branch order, as per-row epilogue factors: (rs1, rs2) fp32 [B*n], or (None, None) in eval or at rate 0."""
        if self.drop_prob == 0.0 or not self.training:
            return None, None
        keep = 1.0 - self.drop_prob
        return tuple(((torch.rand(B, device=device) < keep).to(f32) / keep).repeat_interleave(n) for _ in range(2))

    def _spec(self, B, n, training=False, head_axis=False):
        a = self.attn
        return ops.BlockSpec(B, n, a.num_heads, layernorm=True, eps1=self.norm1.eps, eps2=self.norm2.eps, scale=a.scale,
                             head_axis=head_axis, checkpoint=self.with_cp, precision=block_precision(self, training),
                             attn_fp8=block_attn_fp8(self, head_axis))

    def _param_tuple(self):
        a = self.attn
        return ops.BlockParams(
            n1w=self.norm1.weight, n1b=self.norm1.bias, qkvw=a.qkv.weight, qkvb=a.qkv_bias_vector(), qnw=None, knw=None,
            projw=a.proj.weight, projb=a.proj.bias, g1=self.gamma_1, n2w=self.norm2.weight, n2b=self.norm2.bias,
            fc1w=self.mlp.fc1.weight, fc1b=self.mlp.fc1.bias, fc2w=self.mlp.fc2.weight, fc2b=self.mlp.fc2.bias,
            g2=self.gamma_2)

    def forward_stream(self, x2d, B, n):
        """fp32 residual stream [B*n, D] -> same, through ops.BlockFn when a gradient is needed."""
        rs = self._drop_path_rows(B, n, x2d.device)
        if not torch.is_grad_enabled():
            return self.forward_infer(x2d, B, n, rs)
        return ops.BlockFn.apply(x2d, self._spec(B, n, training=True), *rs, *self._param_tuple())

    def forward_infer(self, x2d, B, n, rowscale=(None, None), head_axis=False):
        """No-grad form: ops.block_forward with nothing saved.  head_axis: the VideoMAEv2 teacher's attention over the
        heads of each token, as the reference executes it (BlockSpec.head_axis)."""
        with torch.no_grad():
            out, _ = ops.block_forward(x2d, self._spec(B, n, head_axis=head_axis), self._param_tuple(), rowscale[0],
                                       rowscale[1], save=False)
        return out

    def forward(self, x):
        B, n, D = x.shape
        return self.forward_stream(x.reshape(B * n, D).float().contiguous(), B, n).reshape(B, n, D)


FP8_SCALINGS = {"tensor": ops.FP8_TENSOR, "token": ops.FP8_TOKEN}


def set_droppath_skip(model: nn.Module, enabled: bool = True) -> int:
    """Switch, in every PretrainInternVideo2 tower of `model`, whether a training step skips the GEMM and attention work
    of the clips its DropPath draw drops (on by default; ops.droppath_plan, ivb_gemm_bf16_plan, ivb_gemm_fp8_plan,
    ivb_attn_fwd_plan / ivb_attn_bwd_plan), in bf16 and in per-token FP8 (set_fp8 with scaling="token"; per-tensor FP8
    runs every row).  Off runs every row, with the same parameters and gradients; the switch is there to measure the two
    in one process.  Returns how many towers were switched."""
    towers = [m for m in model.modules() if isinstance(m, PretrainInternVideo2)]
    for m in towers:
        m.droppath_skip = bool(enabled)
    return len(towers)


def set_fp8(model: nn.Module, enabled: bool = True, scaling: str = "tensor", wgrad: bool = False) -> int:
    """Switch the FP8 mode of every fused block in `model` on or off; returns how many blocks were switched.  The
    blocks: the RMSNorm Blocks (stage-1 student, CLIP tower, stage-2 tower, InternVL teacher), the LayerNorm
    VideoMAEBlocks (InternVideo1's VideoMAE encoder and decoder, the VideoMAEv2 teacher) and the MobileCLIP text
    tower's text_modules.TransformerEncoder blocks.  The LayerNorm blocks take every scaling the RMSNorm block takes;
    their norms write the same E4M3 rows (with the LayerNorm bias), their GEMMs the same epilogues (the VideoMAE q/v
    bias and gamma, the text tower's full qkv bias), and the text tower's causal attention stays bf16.

    In FP8 mode a block runs its forward GEMMs (qkv, proj, fc1, fc2) and its input-gradient GEMMs on the FP8 tensor
    cores, every scale a power of two from the amax of what it scales (no state, nothing in the state_dict).
    scaling="tensor": activations and weights in E4M3, gradients in E5M2, one scale per tensor.  scaling="token":
    activations and gradients in E4M3 with one scale per row (token), cast in one pass over each row (n1 and n2 inside
    the norm kernel), and the weights in E4M3 with one scale per output channel for the forward and per input channel
    for the input-gradient GEMMs.  Weight gradients, attention, norms and everything outside the blocks stay bf16.
    wgrad=True (scaling="token" only; any other scaling raises ValueError) also runs the four weight gradients on the
    FP8 tensor cores: dy and the saved bf16 activation are cast transposed to E4M3 with one scale per channel per
    128-token block, applied as the GEMM promotes each 128-token k-block to fp32 (ops.FP8_TOKEN_WGRAD); every GEMM of
    the block then runs in FP8.  The mode is read when a block runs: switch it before capturing a CUDA graph of the
    step."""
    if scaling not in FP8_SCALINGS:
        raise ValueError(f"set_fp8: scaling must be one of {sorted(FP8_SCALINGS)}, got {scaling!r}")
    if wgrad and scaling != "token":
        raise ValueError(f"set_fp8: wgrad=True needs scaling='token', got {scaling!r}")
    n = 0
    for mod in model.modules():
        if isinstance(mod, Fp8Block):
            mod.fp8 = bool(enabled)
            mod.fp8_scaling = scaling
            mod.fp8_wgrad = bool(wgrad)
            n += 1
    return n


class Fp8InferenceWeights:
    """The E4M3 copies of a block's four GEMM weights (qkv, proj, fc1, fc2) with one power-of-two scale per output
    channel (lowlevel.fp8_quantize_rows), for FP8 inference.  get() re-quantises a weight whose storage or version
    counter changed since its copy was made (a .to(), an in-place update, load_state_dict): a host-side check that
    needs no device sync.  Not module state: nothing here is in the state_dict."""

    def __init__(self, linears):
        self.linears = linears
        self.keys = [None] * len(linears)
        self.copies = [None] * len(linears)

    def get(self):
        for i, lin in enumerate(self.linears):
            w = lin.weight
            key = (w.data_ptr(), w._version)
            if key != self.keys[i]:
                with torch.no_grad():
                    self.copies[i] = ll.fp8_quantize_rows(w.detach())
                self.keys[i] = key
        return tuple(self.copies)


def block_precision(block, training=False):
    """The ops.BlockSpec precision a forward of `block` (an Fp8Block, or a BertLayer for its fp8_inference) runs at,
    from its switches: set_fp8 (fp8) and set_fp8_inference (fp8_inference).  training: the forward needs a gradient."""
    fp8 = getattr(block, "fp8", False)
    if block.fp8_inference is None:
        if not fp8:
            return ops.BF16
        return ops.FP8_TOKEN_WGRAD if getattr(block, "fp8_wgrad", False) else FP8_SCALINGS[block.fp8_scaling]
    if training:
        raise ll._lib.IvbError("Block: FP8 inference mode (set_fp8_inference) has no gradient; switch it off to train")
    if fp8:
        raise ll._lib.IvbError("FP8 inference (set_fp8_inference) and FP8 training (set_fp8) are both on for a block")
    return block.fp8_inference.get()


def block_attn_fp8(block, head_axis=False):
    """The ops.BlockSpec attn_fp8 of a forward of `block`: set_fp8_inference(attention=True) is on for it and the call's
    attention runs over the tokens (head-axis attention keeps its kernel)."""
    return block.fp8_inference is not None and block.fp8_attention and not head_axis


def set_fp8_inference(model: nn.Module, enabled: bool = True, attention: bool = False) -> int:
    """Switch FP8 inference on or off for every fused block (Block, VideoMAEBlock, text_modules.TransformerEncoder)
    and every text layer of bert_modules.BertModel in `model` (frozen towers: the InternVL and VideoMAE teachers, the
    frozen CLIP and stage-2 towers, the MobileCLIP text tower, the stage-2 BERT text encoder); returns how many blocks
    and layers were switched (a BERT layer from fusion_layer on runs nothing in text mode and is not switched).

    In this mode a block's no-grad forward runs its four GEMMs (qkv, proj, fc1, fc2) on the FP8 tensor cores with
    per-token activation scales, computed where each activation is produced (n1 and n2 inside the norm kernel, a and
    g by a row-wise cast), and per-output-channel weight scales.  Switching on quantises each block's weights once;
    they are re-quantised only when a weight changes.  The q/k norms and the fp32 residual stream stay bf16 / fp32.
    attention=False (the default) keeps attention bf16; attention=True also runs the token-axis attention on the FP8
    tensor cores: q and k cast to E4M3 with one scale per (token, head), v per (clip, head, channel), P in E4M3
    (lowlevel._attn_fp8_pack, _attn_fwd_fp8).  The VideoMAEv2 teacher's head-axis attention (head_axis_attention=True)
    keeps its own kernel either way, and so do the text tower's causal attention and BERT's key-length attention, which
    stay bf16.  A BERT layer runs its qkv, attention-output, intermediate and output GEMMs on the FP8 tensor cores;
    each post-LN LayerNorm writes its row once as the bf16 residual and as the E4M3 rows of the next GEMM
    (lowlevel.norm_fwd_fp8 with save=True).  Switching off restores the bf16 path bit for bit.  A switched block
    refuses a forward that needs a gradient, and the mode excludes set_fp8 on the same block."""
    blocks = [m for m in model.modules() if isinstance(m, Fp8InferenceSwitch) and m._fp8_linears()]
    if enabled and any(getattr(m, "fp8", False) for m in blocks):
        raise ll._lib.IvbError("set_fp8_inference: a block is in FP8 training mode (set_fp8); switch that off first")
    for m in blocks:
        m.fp8_attention = bool(enabled and attention)
        if not enabled:
            m.fp8_inference = None
        elif m.fp8_inference is None:
            m.fp8_inference = Fp8InferenceWeights(m._fp8_linears())
            m.fp8_inference.get()
    return len(blocks)


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
        B, N, D = x.shape[0], self.num_patches, self.proj.weight.shape[0]
        idx = torch.arange(0, N + 1, device=x.device, dtype=torch.int32).repeat(B, 1).contiguous()
        out = embed_tokens(self, x, idx, None, torch.zeros((1, N, D), device=x.device, dtype=bf16))
        return out.reshape(B, self.grid_size[0], self.grid_size[1] * self.grid_size[2], D).to(bf16)


class TubeletPatchEmbed(PatchEmbed):
    """The VideoMAE towers' patch embed (videomae.py:135-149, IV1 modeling_finetune.py:184-219): PatchEmbed with their
    defaults, 16 frames in tubelets of 2."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, num_frames=16, tubelet_size=2):
        super().__init__(img_size, patch_size, in_chans, embed_dim, num_frames, int(tubelet_size))


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


def vit_stack(embed_dim, depth, num_heads, mlp_ratio, drop_path_rate, attn_pool_num_heads, clip_embed_dim,
              checkpoint_num=0, **block_kw):
    """`blocks` and `clip_projector` of the InternVideo2 towers and the InternVL teacher (internvideo2_pretrain.py:
    495-518): `depth` RMSNorm Blocks whose DropPath rate rises linearly from 0 to drop_path_rate, the first
    checkpoint_num of them recomputing their forward in backward, then the attention-pooling projector.
    block_kw: the Block switches (qkv_bias, init_values, qk_normalization, layerscale_no_force_fp32, use_*)."""
    dpr = [drop_path_rate * i / (depth - 1) if depth > 1 else 0.0 for i in range(depth)]  # == linspace(0, r, depth)
    blocks = nn.ModuleList([Block(embed_dim, num_heads, mlp_ratio, norm_layer=RMSNorm, drop_path=dpr[i], attn_drop=0.0,
                                  with_cp=i < checkpoint_num, **block_kw) for i in range(depth)])
    return blocks, AttentionPoolingBlock(dim=embed_dim, num_heads=attn_pool_num_heads, qkv_bias=True, qk_scale=None,
                                         drop=0.0, attn_drop=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-5),
                                         out_dim=clip_embed_dim)


class InternVideo2Tower(nn.Module):
    """What the InternVideo2 towers share (the student, the stage-2 tower and the CLIP tower): `patch_embed`,
    `cls_token`, the position tables of `pos_prefixes` ('' for the blocks, 'clip_' / 'mae_' for the decoders; joint,
    or spatial / temporal / cls with sep_pos_embed), `blocks` and `clip_projector`, registered in this order.
    A subclass registers its heads and then calls init_tower(), so the init draws follow every constructor draw.
    cls_token_num: the number of cls tokens (InternVideo-Next: 4), each with its own zero row in front of the joint
    tables; patch_embed_layer: the patch embed's class."""

    pos_prefixes = ("",)
    patch_embed_layer = PatchEmbed
    sep_image_video_pos_embed = False

    def __init__(self, in_chans, patch_size, img_size, qkv_bias, drop_path_rate, embed_dim, num_heads, mlp_ratio,
                 init_values, qk_normalization, depth, use_flash_attn, use_fused_rmsnorm, use_fused_mlp,
                 fused_mlp_heuristic, attn_pool_num_heads, clip_embed_dim, layerscale_no_force_fp32, num_frames,
                 tubelet_size, sep_pos_embed, use_checkpoint, checkpoint_num, cls_token_num=1):
        super().__init__()
        assert use_flash_attn == use_fused_rmsnorm == use_fused_mlp, \
            "use_flash_attn, use_fused_rmsnorm and use_fused_mlp should be consistent"
        self.use_flash_attn = use_flash_attn
        self.embed_dim = embed_dim
        self.depth = depth
        self.patch_embed = self.patch_embed_layer(img_size, patch_size, in_chans, embed_dim, num_frames=num_frames,
                                                  tubelet_size=tubelet_size)
        self.cls_token_num = cls_token_num
        self.cls_token = nn.Parameter(torch.zeros(1, cls_token_num, embed_dim))
        self.sep_pos_embed = bool(sep_pos_embed)
        gs = self.grid_size = self.patch_embed.grid_size
        self.image_pos_groups = gs[0]        # an image's joint table: the mean over these groups of the video table
        Z = lambda *shape: nn.Parameter(torch.zeros(*shape))  # noqa: E731
        for pre in self.pos_prefixes:        # :481-493 — a table (set) per consumer; the MAE decoder's has no cls row
            if not self.sep_pos_embed:
                setattr(self, pre + "pos_embed", Z(1, self.patch_embed.num_patches + (pre != "mae_") * cls_token_num,
                                                   embed_dim))
                continue
            setattr(self, pre + "pos_embed_spatial", Z(1, gs[1] * gs[2], embed_dim))
            setattr(self, pre + "pos_embed_temporal", Z(1, gs[0], embed_dim))
            if pre != "mae_":
                setattr(self, pre + "pos_embed_cls", Z(1, 1, embed_dim))
        self.blocks, self.clip_projector = vit_stack(
            embed_dim, depth, num_heads, mlp_ratio, drop_path_rate, attn_pool_num_heads, clip_embed_dim,
            checkpoint_num if use_checkpoint else 0, qkv_bias=qkv_bias, init_values=init_values,
            use_flash_attn=use_flash_attn, use_fused_mlp=use_fused_mlp, fused_mlp_heuristic=fused_mlp_heuristic,
            qk_normalization=qk_normalization, layerscale_no_force_fp32=layerscale_no_force_fp32,
            use_fused_rmsnorm=use_fused_rmsnorm)

    # ---- init (internvideo2_pretrain.py:547-603)
    def init_tower(self):
        self.init_pos_embed()
        trunc_normal_(self.cls_token, std=0.02)
        self.apply(init_weights)
        self.fix_init_weight()

    def init_pos_embed(self):
        gs, D = self.grid_size, self.embed_dim
        if self.sep_pos_embed:
            sp, tp = _pos_tensor(get_2d_sincos_pos_embed(D, gs[1])), _pos_tensor(get_1d_sincos_pos_embed(D, gs[0]))
            for pre in self.pos_prefixes:
                getattr(self, pre + "pos_embed_spatial").data.copy_(sp)
                getattr(self, pre + "pos_embed_temporal").data.copy_(tp)
            return
        t = _pos_tensor(get_3d_sincos_pos_embed(D, gs[1], gs[0], cls_token=True, cls_token_num=self.cls_token_num))
        for pre in self.pos_prefixes:
            pe = getattr(self, pre + "pos_embed")
            pe.data.copy_(t[:, -pe.shape[1]:])

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
        names = {"cls_token"}
        for pre in self.pos_prefixes:
            names |= {pre + "pos_embed", pre + "pos_embed_spatial", pre + "pos_embed_temporal"}
            if pre != "mae_":
                names.add(pre + "pos_embed_cls")
        return names

    def _pos_table(self, prefix, use_image=False):
        """The position table a forward adds for the blocks ('') or a decoder ('clip_', 'mae_'): [1, 1+tokens, D]
        ([1, tokens, D] for 'mae_'), torch glue, O(N*D), differentiable.  Separable: the spatial table, for a video plus
        the temporal one (:640-656 / :700-711 / :727-734), behind the cls table.  Joint: the parameter for a video; for
        an image stage 2's image parameter (sep_image_video_pos_embed), else the mean of the video table over
        `image_pos_groups` groups (internvideo2_clip_vision.py:524-527, internvideo2.py:598-606)."""
        gs = self.grid_size
        if self.sep_pos_embed:
            pe = getattr(self, prefix + "pos_embed_spatial")
            if not use_image:
                pe = pe.repeat(1, gs[0], 1) + torch.repeat_interleave(getattr(self, prefix + "pos_embed_temporal"),
                                                                       gs[1] * gs[2], dim=1)
            if prefix == "mae_":
                return pe
            return torch.cat([getattr(self, prefix + "pos_embed_cls").expand(pe.shape[0], -1, -1), pe], 1)
        pe = getattr(self, prefix + "pos_embed")
        if not use_image:
            return pe
        if self.sep_image_video_pos_embed:
            return getattr(self, prefix + "img_pos_embed")
        img = pe[:, 1:, :].view(1, self.image_pos_groups, -1, pe.shape[-1]).mean(dim=1)
        return torch.cat([pe[:, :1, :], img], dim=1)


class PretrainInternVideo2(InternVideo2Tower):
    """internvideo2_pretrain.py:406-744 — same ctor kwargs, same state_dict keys, same forward contract:
    forward(x[B,3,T,H,W], mask[B,1+T*L] bool) -> (x_clip_align[K,B,n,Ct], x_align[B,Cf], x_mae_align[K',B,n-1,Cm]).
    """

    pos_prefixes = ("", "clip_", "mae_")
    droppath_skip = True      # set_droppath_skip

    def __init__(self, in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.25,
                 embed_dim=1408, num_heads=16, mlp_ratio=4.3637, init_values=1e-5, qk_normalization=True,
                 depth=40, use_flash_attn=True, use_fused_rmsnorm=True, use_fused_mlp=True, fused_mlp_heuristic=1,
                 attn_pool_num_heads=16, clip_embed_dim=768, layerscale_no_force_fp32=False, num_frames=8,
                 tubelet_size=1, sep_pos_embed=False, use_checkpoint=False, checkpoint_num=0,
                 clip_teacher_embed_dim=3200, clip_teacher_final_dim=768, clip_norm_type="l2", clip_return_layer=1,
                 clip_student_return_interval=1, mae_teacher_embed_dim=1408, mae_norm_type="l2", mae_return_layer=1,
                 mae_student_return_interval=1):
        super().__init__(in_chans, patch_size, img_size, qkv_bias, drop_path_rate, embed_dim, num_heads, mlp_ratio,
                         init_values, qk_normalization, depth, use_flash_attn, use_fused_rmsnorm, use_fused_mlp,
                         fused_mlp_heuristic, attn_pool_num_heads, clip_embed_dim, layerscale_no_force_fp32, num_frames,
                         tubelet_size, sep_pos_embed, use_checkpoint, checkpoint_num)
        self.clip_norm_type, self.mae_norm_type = clip_norm_type, mae_norm_type
        self.clip_return_index = [depth - int(i * clip_student_return_interval) - 1 for i in range(clip_return_layer)]
        self.mae_return_index = [depth - int(i * mae_student_return_interval) - 1 for i in range(mae_return_layer)]
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
        self.init_tower()

    # ---- the hot path
    def visible_index(self, mask, n_visible=None):
        """int32 [B, n] positions of the kept tokens in `x[~mask]` order (bit-exact)."""
        if n_visible is None:
            n_visible = int(mask.shape[1] - int(mask[0].sum()))   # one tiny D2H when the mask lives on the GPU
        idx, err = ll.visible_indices(mask.to(self.cls_token.device, non_blocking=True), n_visible)
        return idx, err, n_visible

    def forward_features(self, x, mask, n_visible=None, drop_path_factors=None, use_image=False, last=None):
        """-> (taps: dict block_idx -> fp32 [B*n, D], final fp32 [B*n, D], idx int32 [B,n], B, n).
        drop_path_factors: optional fp32 [2*depth, B] per-sample stochastic-depth factors (Bernoulli(keep)/keep;
        rows 2i, 2i+1 = the two branches of block i) used instead of a fresh draw — parity tests inject the
        draw the reference made (SURVEY App.B-16: RNG-dependent pieces are injected, not compared).
        use_image / last: stage 2's image position table and early exit after block `last`."""
        check_input(self, x, self.dtype)
        B = x.shape[0]
        idx, err, n = self.visible_index(mask, n_visible)
        self.index_error = err       # int32[1] on the device: 0, or 1 + (a clip whose visible-token count != n)
        h = embed_tokens(self.patch_embed, x, idx, self.cls_token, self._pos_table("", use_image))
        if drop_path_factors is not None:
            rs = drop_path_factors.to(device=h.device, dtype=f32).repeat_interleave(n, dim=1).contiguous()
        else:
            rs = self._sample_drop_path(B, n, h.device)
        plans = self._droppath_plans(rs)

        def block(i, blk, h):
            return blk.forward_stream(h, B, n, None if rs is None else (rs[2 * i], rs[2 * i + 1]),
                                      None if plans is None else plans[2 * i:2 * i + 2])
        h, taps = run_blocks(self.blocks, h, block, self.clip_return_index + self.mae_return_index, last)
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

    def _droppath_plans(self, rs):
        """The DropPath plans of the step's factors rs [2*depth, B*n] (one launch, ops.droppath_plan): per branch its
        plan row, or None for a branch of rate 0 (block 0), which runs every row.  None when there is nothing to skip:
        no factors, no gradient (the no-grad block path takes no plan) or set_droppath_skip(model, False)."""
        if rs is None or not self.droppath_skip or not torch.is_grad_enabled():
            return None
        plan = ops.droppath_plan(rs)
        return [plan[2 * i + j] if isinstance(dp, DropPath) else None
                for i, blk in enumerate(self.blocks) for j, dp in enumerate((blk.drop_path1, blk.drop_path2))]

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
        x_align = x_align + index_poison(self.index_error).to(x_align.dtype)   # ragged mask -> NaN (see forward_loss)
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
        loss_final = loss_final + index_poison(self.index_error)
        return loss_clip, loss_final, loss_mae


def pretrain_internvideo2_1B_patch14_224(pretrained=False, **kwargs):
    """internvideo2_pretrain.py:747-755."""
    return PretrainInternVideo2(img_size=224, patch_size=14, embed_dim=1408, depth=40, num_heads=16,
                                mlp_ratio=48 / 11, attn_pool_num_heads=16, clip_embed_dim=768, **kwargs)


def pretrain_internvideo2_6B_patch14_224(pretrained=False, **kwargs):
    """internvideo2_pretrain.py:758-766."""
    return PretrainInternVideo2(img_size=224, patch_size=14, embed_dim=3200, depth=48, num_heads=25,
                                mlp_ratio=4, attn_pool_num_heads=16, clip_embed_dim=768, **kwargs)
