"""InternVideo1 VideoMAE pre-training model on the libivb200 kernels (SURVEY §8 a15 + f-4: the literal pixel-reconstruction
form of the hot path — tubelet embed of the visible tokens, LayerNorm/q-v-bias encoder blocks, a light decoder over
visible + mask tokens, pixel head on the masked tokens, MSE against per-patch normalised pixels).

Mirrors InternVideo1/Pretrain/VideoMAE:
  Attention, Block                      modeling_finetune.py:77-181   (qkv without bias + q_bias / v_bias, optional gamma_1/2)
  PatchEmbed                            modeling_finetune.py:184-219  (Conv3d k = s = (tubelet, p, p))
  get_sinusoid_encoding_table           modeling_finetune.py:224-242
  PretrainVisionTransformerEncoder      modeling_pretrain.py:34-171
  PretrainVisionTransformerDecoder      modeling_pretrain.py:174-266
  PretrainVisionTransformer             modeling_pretrain.py:269-387  (+ the named factories :390-548)
  pixel_labels / pretrain_loss          engine_for_pretraining.py:66-106 (target build + nn.MSELoss)
Same constructor arguments, same state_dict keys, same forward contract
`model(x[B,3,T,H,W], mask[B,N] bool) -> [B, N_mask, 3*tubelet*p*p]`.

Built from the differentiable primitives of ops.py (LayerNorm rows, wgmma GEMM with bias / GELU epilogues, wgmma flash
attention, visible-only im2col embed); the residual stream is fp32, everything else bf16.  No CPU path.
"""
from __future__ import annotations

from functools import partial

import numpy as np
import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops

bf16, f32 = torch.bfloat16, torch.float32
IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)


def to_2tuple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x)


def get_sinusoid_encoding_table(n_position, d_hid):
    """modeling_finetune.py:224-242 — [1, n_position, d_hid] fp32, sin on even / cos on odd channels."""
    pos = np.arange(n_position, dtype=np.float64)[:, None]
    j = np.arange(d_hid)[None, :]
    table = pos / np.power(10000, 2 * (j // 2) / d_hid)
    table[:, 0::2] = np.sin(table[:, 0::2])
    table[:, 1::2] = np.cos(table[:, 1::2])
    return torch.tensor(table, dtype=torch.float, requires_grad=False).unsqueeze(0)


def _drop_path_rows(a, B, n, p, training):
    """timm drop_path on a [B*n, D] stream: one Bernoulli(keep)/keep factor per sample."""
    if p == 0.0 or not training:
        return a
    keep = 1.0 - p
    m = (torch.rand(B, device=a.device) < keep).to(a.dtype) / keep
    return a * m.repeat_interleave(n)[:, None]


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)
        if drop:
            raise NotImplementedError("ivb200 VideoMAE: dropout is 0 in every pre-training recipe")


class Attention(nn.Module):
    """modeling_finetune.py:77-129."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0.0, proj_drop=0.0, attn_head_dim=None):
        super().__init__()
        self.num_heads = num_heads
        head_dim = attn_head_dim if attn_head_dim is not None else dim // num_heads
        self.head_dim = head_dim
        all_head_dim = head_dim * num_heads
        self.scale = qk_scale or head_dim ** -0.5
        self.qkv = nn.Linear(dim, all_head_dim * 3, bias=False)
        if qkv_bias:
            self.q_bias = nn.Parameter(torch.zeros(all_head_dim))
            self.v_bias = nn.Parameter(torch.zeros(all_head_dim))
        else:
            self.q_bias = self.v_bias = None
        self.proj = nn.Linear(all_head_dim, dim)
        if attn_drop or proj_drop:
            raise NotImplementedError("ivb200 VideoMAE: attention / projection dropout are 0 in every pre-training recipe")

    def forward_rows(self, h, B, n):
        """h: bf16 [B*n, dim] -> fp32 [B*n, dim]."""
        bias = None
        if self.q_bias is not None:       # :111-115 — k has no bias
            bias = torch.cat((self.q_bias, torch.zeros_like(self.v_bias, requires_grad=False), self.v_bias))
        qkv = ops.linear(h, self.qkv.weight, bias)
        A = self.num_heads * self.head_dim
        o = ops.AttnFn.apply(qkv[:, :A], qkv[:, A:2 * A], qkv[:, 2 * A:], B, n, self.num_heads, self.head_dim, self.scale)
        return ops.linear(o, self.proj.weight, self.proj.bias, True)


class Block(nn.Module):
    """modeling_finetune.py:132-181."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop=0.0, attn_drop=0.0,
                 drop_path=0.0, init_values=None, act_layer=nn.GELU, norm_layer=nn.LayerNorm, attn_head_dim=None):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                              proj_drop=drop, attn_head_dim=attn_head_dim)
        self.drop_prob = float(drop_path)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)
        if init_values is not None and init_values > 0:
            self.gamma_1 = nn.Parameter(init_values * torch.ones(dim), requires_grad=True)
            self.gamma_2 = nn.Parameter(init_values * torch.ones(dim), requires_grad=True)
        else:
            self.gamma_1 = self.gamma_2 = None

    def forward_rows(self, x, B, n):
        """x: fp32 residual stream [B*n, dim] -> same."""
        a = self.attn.forward_rows(ops.layernorm(x, self.norm1.weight, self.norm1.bias, self.norm1.eps), B, n)
        if self.gamma_1 is not None:
            a = a * self.gamma_1.float()
        x = x + _drop_path_rows(a, B, n, self.drop_prob, self.training)
        h = ops.layernorm(x, self.norm2.weight, self.norm2.bias, self.norm2.eps)
        g = ops.LinearGeluFn.apply(h, self.mlp.fc1.weight, self.mlp.fc1.bias, False)
        m = ops.linear(g, self.mlp.fc2.weight, self.mlp.fc2.bias, True)
        if self.gamma_2 is not None:
            m = m * self.gamma_2.float()
        return x + _drop_path_rows(m, B, n, self.drop_prob, self.training)

    def forward(self, x):
        B, n, D = x.shape
        return self.forward_rows(x.reshape(B * n, D).float(), B, n).reshape(B, n, D)


class PatchEmbed(nn.Module):
    """modeling_finetune.py:184-219 (parameters only; the convolution runs as im2col of the visible patches + GEMM)."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, num_frames=16, tubelet_size=2):
        super().__init__()
        img_size, patch_size = to_2tuple(img_size), to_2tuple(patch_size)
        self.tubelet_size = int(tubelet_size)
        self.num_patches = (img_size[1] // patch_size[1]) * (img_size[0] // patch_size[0]) * (num_frames // self.tubelet_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.proj = nn.Conv3d(in_channels=in_chans, out_channels=embed_dim,
                              kernel_size=(self.tubelet_size, patch_size[0], patch_size[1]),
                              stride=(self.tubelet_size, patch_size[0], patch_size[1]))


def _xavier_init(m):
    if isinstance(m, nn.Linear):
        nn.init.xavier_uniform_(m.weight)
        if m.bias is not None:
            nn.init.constant_(m.bias, 0)
    elif isinstance(m, nn.LayerNorm):
        nn.init.constant_(m.bias, 0)
        nn.init.constant_(m.weight, 1.0)


def kept_indices(mask, keep_masked=False, count=None):
    """int32 [B, 1+k] (slot 0 = the unused cls position, then 1 + patch index in x[~mask] order, bit-exact) of the visible
    patches, or of the masked ones.  count: k when the caller knows it (fixed mask ratio) — saves the host read."""
    m = ~mask if keep_masked else mask
    B, N = m.shape
    with_cls = torch.cat([torch.zeros((B, 1), dtype=torch.bool, device=m.device), m], dim=1)
    k = int(count) if count is not None else N - int(m[0].sum())     # one tiny D2H when the mask lives on the GPU
    idx, err = ll.visible_indices(with_cls.contiguous(), k + 1)
    return idx, err, k


class PretrainVisionTransformerEncoder(nn.Module):
    """modeling_pretrain.py:34-171."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=0, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.0,
                 norm_layer=nn.LayerNorm, init_values=None, tubelet_size=2, use_learnable_pos_emb=False, with_cp=False):
        super().__init__()
        self.num_classes = num_classes
        self.num_features = self.embed_dim = embed_dim
        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, in_chans=in_chans, embed_dim=embed_dim,
                                      tubelet_size=tubelet_size)
        num_patches = self.patch_embed.num_patches
        self.with_cp = with_cp
        if use_learnable_pos_emb:
            self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim))
        else:
            self.pos_embed = get_sinusoid_encoding_table(num_patches, embed_dim)     # plain tensor, like the reference
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.blocks = nn.ModuleList([
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale,
                  drop=drop_rate, attn_drop=attn_drop_rate, drop_path=dpr[i], norm_layer=norm_layer,
                  init_values=init_values) for i in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()
        if use_learnable_pos_emb:
            nn.init.trunc_normal_(self.pos_embed, std=0.02, a=-0.02, b=0.02)
        self.apply(_xavier_init)

    def get_num_layers(self):
        return len(self.blocks)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_embed", "cls_token"}

    def forward_rows(self, x, idx, B, nv):
        """x bf16 video, idx int32 [B, 1+nv] (cls slot + visible patches) -> bf16 [B*nv, C_e] after the final LayerNorm."""
        pe = self.patch_embed
        D = self.embed_dim
        pos = self.pos_embed[:, -pe.num_patches:].to(device=x.device)          # learnable table has an unused first row
        # EmbedFn embeds tokens idx[:, 1:] and puts `cls + pos[0]` in front: give it a zero cls row and drop it again
        table = torch.cat([torch.zeros(1, 1, D, device=x.device, dtype=pos.dtype), pos], 1).to(bf16)
        zcls = torch.zeros(1, 1, D, device=x.device, dtype=bf16)
        h = ops.EmbedFn.apply(x, idx, pe.proj.weight, pe.proj.bias, zcls, table, pe.tubelet_size, pe.patch_size[0])
        h = h.reshape(B, nv + 1, D)[:, 1:].reshape(B * nv, D)
        for blk in self.blocks:
            if self.with_cp and torch.is_grad_enabled():
                h = torch.utils.checkpoint.checkpoint(blk.forward_rows, h, B, nv, use_reentrant=False)
            else:
                h = blk.forward_rows(h, B, nv)
        h = ops.layernorm(h, self.norm.weight, self.norm.bias, self.norm.eps)
        if isinstance(self.head, nn.Linear):
            h = ops.linear(h, self.head.weight, self.head.bias)
        return h

    def forward(self, x, mask):
        _check_input(self.patch_embed.proj.weight, x)
        idx, err, nv = kept_indices(mask.to(x.device))
        B = x.shape[0]
        return self.forward_rows(x.to(bf16), idx, B, nv).reshape(B, nv, -1)


class PretrainVisionTransformerDecoder(nn.Module):
    """modeling_pretrain.py:174-266."""

    def __init__(self, patch_size=16, num_classes=768, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0,
                 qkv_bias=False, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.0,
                 norm_layer=nn.LayerNorm, init_values=None, num_patches=196, tubelet_size=2, with_cp=False, with_fp16=True):
        super().__init__()
        self.num_classes = num_classes
        assert num_classes == 3 * tubelet_size * patch_size ** 2
        self.num_features = self.embed_dim = embed_dim
        self.patch_size = patch_size
        self.with_cp, self.with_fp16 = with_cp, with_fp16
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.blocks = nn.ModuleList([
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale,
                  drop=drop_rate, attn_drop=attn_drop_rate, drop_path=dpr[i], norm_layer=norm_layer,
                  init_values=init_values) for i in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()
        self.apply(_xavier_init)

    def get_num_layers(self):
        return len(self.blocks)

    def forward_rows(self, h, B, N, return_token_num):
        """h fp32 [B*N, C_d] -> bf16 [B, return_token_num (or N), num_classes]."""
        for blk in self.blocks:
            if self.with_cp and torch.is_grad_enabled():
                h = torch.utils.checkpoint.checkpoint(blk.forward_rows, h, B, N, use_reentrant=False)
            else:
                h = blk.forward_rows(h, B, N)
        C = h.shape[-1]
        h = h.reshape(B, N, C)
        if return_token_num > 0:
            h = h[:, -return_token_num:]                   # only the mask tokens predict pixels (:260-262)
        k = h.shape[1]
        y = ops.layernorm(h.reshape(B * k, C), self.norm.weight, self.norm.bias, self.norm.eps)
        if isinstance(self.head, nn.Linear):
            y = ops.linear(y, self.head.weight, self.head.bias)
        return y.reshape(B, k, -1)

    def forward(self, x, return_token_num):
        B, N, C = x.shape
        return self.forward_rows(x.reshape(B * N, C).float(), B, N, return_token_num)


def _check_input(w, x):
    if w.dtype != bf16:
        raise ll._lib.IvbError("ivb200 VideoMAE computes in bf16: call model.bfloat16() first")
    if not x.is_cuda:
        raise ll._lib.IvbError("ivb200 VideoMAE: input must be a CUDA tensor (no CPU fallback)")


class PretrainVisionTransformer(nn.Module):
    """modeling_pretrain.py:269-387."""

    def __init__(self, img_size=224, patch_size=16, encoder_in_chans=3, encoder_num_classes=0, encoder_embed_dim=768,
                 encoder_depth=12, encoder_num_heads=12, decoder_num_classes=1536, decoder_embed_dim=512, decoder_depth=8,
                 decoder_num_heads=8, mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0,
                 drop_path_rate=0.0, norm_layer=nn.LayerNorm, init_values=0.0, use_learnable_pos_emb=False, tubelet_size=2,
                 num_classes=0, in_chans=0, with_cp=False):
        super().__init__()
        self.encoder = PretrainVisionTransformerEncoder(
            img_size=img_size, patch_size=patch_size, in_chans=encoder_in_chans, num_classes=encoder_num_classes,
            embed_dim=encoder_embed_dim, depth=encoder_depth, num_heads=encoder_num_heads, mlp_ratio=mlp_ratio,
            qkv_bias=qkv_bias, qk_scale=qk_scale, drop_rate=drop_rate, attn_drop_rate=attn_drop_rate,
            drop_path_rate=drop_path_rate, norm_layer=norm_layer, init_values=init_values, tubelet_size=tubelet_size,
            use_learnable_pos_emb=use_learnable_pos_emb, with_cp=with_cp)
        self.decoder = PretrainVisionTransformerDecoder(
            patch_size=patch_size, num_patches=self.encoder.patch_embed.num_patches, num_classes=decoder_num_classes,
            embed_dim=decoder_embed_dim, depth=decoder_depth, num_heads=decoder_num_heads, mlp_ratio=mlp_ratio,
            qkv_bias=qkv_bias, qk_scale=qk_scale, drop_rate=drop_rate, attn_drop_rate=attn_drop_rate,
            drop_path_rate=drop_path_rate, norm_layer=norm_layer, init_values=init_values, tubelet_size=tubelet_size,
            with_cp=with_cp, with_fp16=True)
        self.encoder_to_decoder = nn.Linear(encoder_embed_dim, decoder_embed_dim, bias=False)
        self.mask_token = nn.Parameter(torch.zeros(1, 1, decoder_embed_dim))
        self.pos_embed = get_sinusoid_encoding_table(self.encoder.patch_embed.num_patches, decoder_embed_dim)
        nn.init.trunc_normal_(self.mask_token, std=0.02, a=-0.02, b=0.02)
        self.patch_size, self.tubelet_size = patch_size, tubelet_size

    def get_num_layers(self):
        return len(self.encoder.blocks)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_embed", "cls_token", "mask_token"}

    def forward(self, x, mask, return_indices=False, n_masked=None):
        """n_masked: masked tubelets per clip when known (the recipes use a fixed ratio): no host read of the mask."""
        _check_input(self.encoder.patch_embed.proj.weight, x)
        B = x.shape[0]
        mask = mask.to(x.device)
        N = mask.shape[1]
        vis, err_v, nv = kept_indices(mask, count=None if n_masked is None else N - n_masked)
        msk, err_m, nm = kept_indices(mask, keep_masked=True, count=n_masked)
        self.index_error = err_v + err_m                         # non-zero: clips keep different numbers of tokens
        h = self.encoder.forward_rows(x.to(bf16), vis, B, nv)                                 # bf16 [B*nv, C_e]
        h = ops.linear(h, self.encoder_to_decoder.weight, None, True).reshape(B, nv, -1)      # fp32 [B, nv, C_d]
        pos = self.pos_embed[0].to(device=x.device, dtype=f32)                                # [N, C_d], no gradient
        pos_vis = pos[(vis[:, 1:] - 1).long()]                   # the visible tokens keep their order, the table follows it
        pos_msk = pos[(msk[:, 1:] - 1).long()]
        x_full = torch.cat([h + pos_vis, self.mask_token.float() + pos_msk], dim=1)           # :380-383
        out = self.decoder.forward_rows(x_full.reshape(B * N, -1), B, N, nm)
        out = out + _poison(self.index_error).to(out.dtype)
        return (out, msk[:, 1:] - 1) if return_indices else out


def _poison(err):
    z = torch.zeros((), device=err.device, dtype=f32)
    return torch.where(err[0] != 0, torch.full_like(z, float("nan")), z)


def pixel_labels(images, masked_idx, patch_size, tubelet_size=2, normalize_target=True):
    """engine_for_pretraining.py:66-96 — targets of the masked tubelets: un-normalise the frames, cut (tubelet, p, p)
    tubelets, optionally normalise each tubelet per channel (unbiased variance, +1e-6).  fp32 [B, N_mask, tubelet*p*p*3]."""
    B, n_mask = masked_idx.shape
    dev = images.device
    mean3 = torch.tensor(IMAGENET_DEFAULT_MEAN, device=dev, dtype=f32)
    std3 = torch.tensor(IMAGENET_DEFAULT_STD, device=dev, dtype=f32)
    lab = ll.pixel_targets(images.to(bf16), masked_idx.to(torch.int32).contiguous().flatten(), n_mask, tubelet_size,
                           patch_size, bool(normalize_target), mean3, std3)
    return lab.reshape(B, n_mask, -1)


class _MseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, label):
        pred2 = pred.reshape(-1, pred.shape[-1]).contiguous()
        ls = torch.zeros(1, device=pred.device, dtype=f32)
        dp = torch.empty_like(pred2)
        ll.mse_loss(pred2, label.reshape(pred2.shape).contiguous(), ls, gscale_host=1.0 / pred2.numel(), dpred=dp)
        ctx.save_for_backward(dp)
        ctx.shape = pred.shape
        return (ls / pred2.numel()).reshape(())

    @staticmethod
    def backward(ctx, g):
        (dp,) = ctx.saved_tensors
        return (dp.float() * g).to(dp.dtype).reshape(ctx.shape), None


def pretrain_loss(model, images, bool_masked_pos, normalize_target=True, n_masked=None):
    """The body of InternVideo1's train_one_epoch (engine_for_pretraining.py:60-101): labels from the frames, forward on the
    masked clip, nn.MSELoss.  images: ImageNet-normalised frames [B,3,T,H,W]; bool_masked_pos [B, N] (True = masked)."""
    mask = bool_masked_pos.to(images.device).flatten(1).to(torch.bool)
    out, midx = model(images, mask, return_indices=True, n_masked=n_masked)
    with torch.no_grad():
        labels = pixel_labels(images, midx, model.patch_size, model.tubelet_size, normalize_target)
    return _MseFn.apply(out, labels)


# ---- factories (modeling_pretrain.py:390-548)
def _make(mlp_ratio=4, **kw):
    return PretrainVisionTransformer(img_size=224, encoder_num_classes=0, mlp_ratio=mlp_ratio, qkv_bias=True,
                                     norm_layer=partial(nn.LayerNorm, eps=1e-6), **kw)


def pretrain_mae_small_patch16_224(pretrained=False, **kwargs):
    return _make(patch_size=16, encoder_embed_dim=384, encoder_depth=12, encoder_num_heads=6, decoder_num_classes=1536,
                 decoder_embed_dim=192, decoder_num_heads=3, **kwargs)


def pretrain_mae_base_patch16_224(pretrained=False, **kwargs):
    return _make(patch_size=16, encoder_embed_dim=768, encoder_depth=12, encoder_num_heads=12, decoder_num_classes=1536,
                 decoder_embed_dim=384, decoder_num_heads=6, **kwargs)


def pretrain_mae_large_patch16_224(pretrained=False, **kwargs):
    return _make(patch_size=16, encoder_embed_dim=1024, encoder_depth=24, encoder_num_heads=16, decoder_num_classes=1536,
                 decoder_embed_dim=512, decoder_num_heads=8, **kwargs)


def pretrain_mae_huge_patch16_224(pretrained=False, **kwargs):
    return _make(patch_size=16, encoder_embed_dim=1280, encoder_depth=32, encoder_num_heads=16, decoder_num_classes=1536,
                 decoder_embed_dim=512, decoder_num_heads=8, **kwargs)


def pretrain_mae_giant_patch16_224(pretrained=False, **kwargs):
    return _make(mlp_ratio=48 / 11, patch_size=16, encoder_embed_dim=1408, encoder_depth=40, encoder_num_heads=16,
                 decoder_num_classes=1536, decoder_embed_dim=512, decoder_num_heads=8, **kwargs)


def pretrain_mae_giant_patch14_224(pretrained=False, **kwargs):
    return _make(mlp_ratio=48 / 11, patch_size=14, encoder_embed_dim=1408, encoder_depth=40, encoder_num_heads=16,
                 decoder_num_classes=1176, decoder_embed_dim=512, decoder_num_heads=8, **kwargs)


def pretrain_mae_gigantic_patch14_224(pretrained=False, **kwargs):
    return _make(mlp_ratio=64 / 13, patch_size=14, encoder_embed_dim=1664, encoder_depth=48, encoder_num_heads=16,
                 decoder_num_classes=1176, decoder_embed_dim=512, decoder_num_heads=8, **kwargs)
