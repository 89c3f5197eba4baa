"""InternVideo1 VideoMAE pre-training model on the libivb200 kernels (SURVEY §8 a15 + f-4: the literal pixel-reconstruction
form of the hot path — tubelet embed of the visible tokens, LayerNorm/q-v-bias encoder blocks, a light decoder over
visible + mask tokens, pixel head on the masked tokens, MSE against per-patch normalised pixels).

Mirrors InternVideo1/Pretrain/VideoMAE:
  Attention, Block                      modeling_finetune.py:77-181   (modules.VideoMAEBlock, shared with the VideoMAEv2 teacher)
  PatchEmbed                            modeling_finetune.py:184-219  (Conv3d k = s = (tubelet, p, p))
  get_sinusoid_encoding_table           modeling_finetune.py:224-242
  PretrainVisionTransformerEncoder      modeling_pretrain.py:34-171
  PretrainVisionTransformerDecoder      modeling_pretrain.py:174-266
  PretrainVisionTransformer             modeling_pretrain.py:269-387  (+ the named factories :390-548)
  pixel_labels / pretrain_loss          engine_for_pretraining.py:66-106 (target build + nn.MSELoss)
Same constructor arguments, same state_dict keys, same forward contract
`model(x[B,3,T,H,W], mask[B,N] bool) -> [B, N_mask, 3*tubelet*p*p]`.

The blocks run through the fused block of ops.py (ops.BlockFn with spec.layernorm: LayerScale, DropPath and the residual
add in the GEMM epilogues); the embed, final norms and heads through its primitives.  The residual stream is fp32,
everything else bf16.  No CPU path.
"""
from __future__ import annotations

from functools import partial

import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .modules import TubeletPatchEmbed as PatchEmbed  # modeling_finetune.py:184-219 (parameters; im2col + GEMM)
from .modules import (VideoMAEBlock, bf16, check_input, embed_tokens, f32, get_sinusoid_encoding_table, index_poison,
                      run_blocks)
from .modules import to_2tuple  # noqa: F401  (a name of the reference module)

IMAGENET_DEFAULT_MEAN = (0.485, 0.456, 0.406)
IMAGENET_DEFAULT_STD = (0.229, 0.224, 0.225)


def _blocks(dim, depth, num_heads, mlp_ratio, qkv_bias, qk_scale, drop, attn_drop, drop_path_rate, norm_layer,
            init_values, with_cp):
    """The encoder's or the decoder's blocks (modeling_pretrain.py:78-92, :208-222), DropPath rising linearly to
    drop_path_rate; with_cp: each block keeps only its input and recomputes its forward in backward."""
    dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
    return nn.ModuleList([
        VideoMAEBlock(dim, num_heads, mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale, drop=drop, attn_drop=attn_drop,
                      drop_path=dpr[i], init_values=init_values, norm_layer=norm_layer, with_cp=with_cp)
        for i in range(depth)])


def _run_blocks(blocks, h, B, n):
    """The encoder's and the decoder's block loop over the fp32 stream [B*n, D]."""
    return run_blocks(blocks, h, lambda i, blk, h: blk.forward_stream(h, B, n))[0]


def _device_table(module, device):
    """module.pos_embed on `device`.  The fixed sinusoid table is a plain host tensor, not module state (as in the
    reference): it is copied to the device once and the copy kept, so a forward makes no host-to-device copy and the
    training step can be captured in a CUDA graph.  A learnable table (nn.Parameter) is returned as it is."""
    pe = module.pos_embed
    if isinstance(pe, nn.Parameter) or pe.device == device:
        return pe
    dev = getattr(module, "_pos_embed_on_device", None)
    if dev is None or dev.device != device:
        dev = module._pos_embed_on_device = pe.to(device)
    return dev


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
        if use_learnable_pos_emb:
            self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim))
        else:
            self.pos_embed = get_sinusoid_encoding_table(num_patches, embed_dim)     # plain tensor, like the reference
        self.blocks = _blocks(embed_dim, depth, num_heads, mlp_ratio, qkv_bias, qk_scale, drop_rate, attn_drop_rate,
                              drop_path_rate, norm_layer, init_values, with_cp)
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
        pos = _device_table(self, x.device)[:, -pe.num_patches:]              # learnable table has an unused first row
        h = _run_blocks(self.blocks, embed_tokens(pe, x, idx, None, pos), B, nv)
        h = ops.layernorm(h, self.norm.weight, self.norm.bias, self.norm.eps)
        if isinstance(self.head, nn.Linear):
            h = ops.linear(h, self.head.weight, self.head.bias)
        return h

    def forward(self, x, mask):
        check_input(self, x, self.patch_embed.proj.weight.dtype)
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
        self.with_fp16 = with_fp16
        self.blocks = _blocks(embed_dim, depth, num_heads, mlp_ratio, qkv_bias, qk_scale, drop_rate, attn_drop_rate,
                              drop_path_rate, norm_layer, init_values, with_cp)
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()
        self.apply(_xavier_init)

    def get_num_layers(self):
        return len(self.blocks)

    def forward_rows(self, h, B, N, return_token_num):
        """h fp32 [B*N, C_d] -> bf16 [B, return_token_num (or N), num_classes]."""
        h = _run_blocks(self.blocks, h, B, N)
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
        check_input(self, x, self.encoder.patch_embed.proj.weight.dtype)
        B = x.shape[0]
        mask = mask.to(x.device)
        N = mask.shape[1]
        vis, err_v, nv = kept_indices(mask, count=None if n_masked is None else N - n_masked)
        msk, err_m, nm = kept_indices(mask, keep_masked=True, count=n_masked)
        self.index_error = err_v + err_m                         # non-zero: clips keep different numbers of tokens
        h = self.encoder.forward_rows(x.to(bf16), vis, B, nv)                                 # bf16 [B*nv, C_e]
        h = ops.linear(h, self.encoder_to_decoder.weight, None, True).reshape(B, nv, -1)      # fp32 [B, nv, C_d]
        pos = _device_table(self, x.device)[0].to(dtype=f32)                                 # [N, C_d], no gradient
        pos_vis = pos[(vis[:, 1:] - 1).long()]                   # the visible tokens keep their order, the table follows it
        pos_msk = pos[(msk[:, 1:] - 1).long()]
        x_full = torch.cat([h + pos_vis, self.mask_token.float() + pos_msk], dim=1)           # :380-383
        out = self.decoder.forward_rows(x_full.reshape(B * N, -1), B, N, nm)
        out = out + index_poison(self.index_error).to(out.dtype)
        return (out, msk[:, 1:] - 1) if return_indices else out


_MEAN_STD = {}


def _imagenet_mean_std(device):
    """fp32 [3] ImageNet mean and std on `device`, made once per device (no host-to-device copy in a captured step)."""
    if device not in _MEAN_STD:
        _MEAN_STD[device] = tuple(torch.tensor(v, device=device, dtype=f32)
                                  for v in (IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD))
    return _MEAN_STD[device]


def pixel_labels(images, masked_idx, patch_size, tubelet_size=2, normalize_target=True):
    """engine_for_pretraining.py:66-96 — targets of the masked tubelets: un-normalise the frames, cut (tubelet, p, p)
    tubelets, optionally normalise each tubelet per channel (unbiased variance, +1e-6).  fp32 [B, N_mask, tubelet*p*p*3]."""
    B, n_mask = masked_idx.shape
    mean3, std3 = _imagenet_mean_std(images.device)
    lab =ll.pixel_targets(images.to(bf16), masked_idx.to(torch.int32).contiguous().flatten(), n_mask, tubelet_size,
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
