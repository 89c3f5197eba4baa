"""InternVideo-Next's video encoder on the libivb200 kernels.

Mirrors InternVideo-Next/models/InternVideo_next.py (constructor kwargs, attribute names, state_dict keys and order,
init draws, forward contract): `PatchEmbed` (:302-342), `InternVideo2` (:345-538) and the two factories (:541-559), so
a released checkpoint loads with strict=True.

The encoder is the InternVideo2 tower with three differences, each handled by the shared front end:
  - the patch embed normalises each patch's raw pixels with an RMSNorm (`norm_before`) before the Conv3d and the conv
    output with a second one (`norm`): ops.EmbedFn runs the first inside the im2col (ivb_im2col_prenorm) and the
    second with ivb_norm_fwd, and its backward returns both weights' gradients (ivb_prenorm_wgrad for norm_before);
  - four cls tokens, each with a zero row of the position table (cls_token_num, pos_embed.py:9-54);
  - the blocks see every one of the 4 + T*L tokens (4 100 at 16 x 224^2); the blocks and the attention-pooling
    projector are modules.Block / AttentionPoolingBlock, so set_fp8_inference reaches them as in every tower.
"""
from __future__ import annotations

import math

import torch

from . import lowlevel as ll
from .modules import InternVideo2Tower, PatchEmbed as _PlainPatchEmbed, RMSNorm, check_input, embed_tokens, run_blocks

bf16 = torch.bfloat16


class PatchEmbed(_PlainPatchEmbed):
    """InternVideo_next.py:302-342: the Conv3d patch embed between two RMSNorms (eps 1e-6), `norm_before` over a
    patch's tubelet_size * p * p * in_chans pixels in (t hp wp c) order and `norm` over the D conv outputs.
    forward(x [B,C,T,H,W]) -> bf16 [B, T', L, D], the reference's layout."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, num_frames=8, tubelet_size=1,
                 norm_layer=None):
        super().__init__(img_size, patch_size, in_chans, embed_dim, num_frames, tubelet_size)
        norm_layer = norm_layer or (lambda d: RMSNorm(d, eps=1e-6))
        self.norm = norm_layer(embed_dim)
        self.norm_before = norm_layer(tubelet_size * math.prod(self.patch_size) * in_chans)
        if self.norm.variance_epsilon != self.norm_before.variance_epsilon:
            raise NotImplementedError("ivb200 PatchEmbed: the two norms must share one eps")


class InternVideo2(InternVideo2Tower):
    """InternVideo_next.py:345-538 — forward(x [B,3,T,H,W], projected=False): the patch tokens [B, T*L, D] (bf16, the
    cls tokens dropped), or with projected=True the attention-pooling projector over all cls_token_num + T*L tokens,
    [B, clip_embed_dim].  Both are differentiable through every parameter.

    Refused: sep_pos_embed=True (the reference then builds a one-row cls table, :402 and :514-520, that cannot be added
    to four cls tokens, so that configuration fails there too), inputs whose frame count or resolution differs from
    the position table (the reference adds pos_embed unresized), non-bf16 parameters and CPU inputs."""

    patch_embed_layer = PatchEmbed

    def __init__(self, in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.25,
                 embed_dim=1408, head_drop_path_rate=0.0, num_heads=16, mlp_ratio=4.3637, init_values=1e-5,
                 qk_normalization=True, depth=40, use_flash_attn=True, use_fused_rmsnorm=True, use_fused_mlp=True,
                 fused_mlp_heuristic=1, attn_pool_num_heads=16, clip_embed_dim=768, layerscale_no_force_fp32=False,
                 num_frames=16, tubelet_size=1, sep_pos_embed=False, use_checkpoint=False, checkpoint_num=0,
                 cls_token_num=4):
        if sep_pos_embed:
            raise NotImplementedError("ivb200 InternVideo-Next: sep_pos_embed=True builds a one-row cls table that "
                                      "cannot be added to the cls tokens (InternVideo_next.py:402,514-520)")
        # head_drop_path_rate is accepted and has no effect: the reference constructs the projector's DropPath
        # (:97-99) but AttentiveBlock.forward never applies it (:101-107)
        super().__init__(in_chans, patch_size, img_size, qkv_bias, drop_path_rate, embed_dim, num_heads, mlp_ratio,
                         init_values, qk_normalization, depth, use_flash_attn, use_fused_rmsnorm, use_fused_mlp,
                         fused_mlp_heuristic, attn_pool_num_heads, clip_embed_dim, layerscale_no_force_fp32, num_frames,
                         tubelet_size, sep_pos_embed, use_checkpoint, checkpoint_num, cls_token_num=cls_token_num)
        self.init_tower()

    def forward_tokens(self, x):
        """-> fp32 residual stream [B*n, D] after the last block, B, n (n = cls_token_num + T*L)."""
        pe = self.patch_embed
        want = (pe.grid_size[0] * pe.tubelet_size, *pe.img_size)
        if x.dim() != 5 or tuple(x.shape[2:]) != want:
            raise ll._lib.IvbError(f"ivb200 InternVideo-Next: input [B, C, T, H, W] must have (T, H, W) = {want}, the "
                                   f"position table's geometry; got {tuple(x.shape)}")
        check_input(self, x, self.dtype)
        B, N = x.shape[0], pe.num_patches
        idx = torch.arange(0, N + 1, device=x.device, dtype=torch.int32).repeat(B, 1).contiguous()
        h = embed_tokens(pe, x, idx, self.cls_token, self.pos_embed)
        n = self.cls_token_num + N
        h, _ = run_blocks(self.blocks, h, lambda i, blk, h: blk.forward_stream(h, B, n))
        return h, B, n

    def forward(self, x, projected=False):
        h, B, n = self.forward_tokens(x)
        h = h.reshape(B, n, self.embed_dim)
        if projected:
            return self.clip_projector(h)
        return h[:, self.cls_token_num:].to(bf16)


def internvideo_next_base_patch14_224(pretrained=False, **kwargs):
    """InternVideo_next.py:541-549."""
    return InternVideo2(img_size=224, patch_size=14, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4,
                        attn_pool_num_heads=16, clip_embed_dim=768, **kwargs)


def internvideo_next_large_patch14_224(pretrained=False, **kwargs):
    """InternVideo_next.py:551-559."""
    return InternVideo2(img_size=224, patch_size=14, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4,
                        attn_pool_num_heads=16, clip_embed_dim=768, **kwargs)
