"""Frozen-teacher inference and the attention-guided mask of InternVideo2 stage-1 pre-training (SURVEY §8f-1), on the
same libivb200 kernels as the student.  Inference only: nothing is saved for backward.

Mirrors (constructor kwargs, parameter names / state_dict keys, forward contracts):
  InternVideo2/single_modality/models/internvl_clip_vision.py:336-465   `InternVL_CLIP`  (per-frame ViT-6B: RMSNorm,
        q/k-norm, LayerScale; attention-pooling projector that also returns its attention map)
  InternVideo2/single_modality/models/videomae.py:62-132,207-313        `VisionTransformer` (VideoMAEv2-g teacher: LayerNorm,
        q/v-bias attention, tubelet 2, fixed sinusoid table)
  InternVideo2/single_modality/engines/engine_for_pretraining.py:97-125 attention-guided mask + target selection

In the real recipe the two teachers cost ~30 TFLOP/clip against ~2.7 for the student step: end-to-end clips/s is
teacher-bound, which is why they run through the same wgmma GEMM / attention kernels.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import lowlevel as ll
from .modules import (LayerNormB, TubeletPatchEmbed, VideoMAEBlock, bf16, check_input, embed_tokens,
                      get_sinusoid_encoding_table, init_weights, run_blocks, to_2tuple, vit_stack)


# ------------------------------------------------------------------------------------------------ CLIP teacher
class FramePatchEmbed(nn.Module):
    """internvl_clip_vision.py:307-333 — Conv3d(k = s = (1, p, p)): every frame is embedded on its own."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, norm_layer=None, flatten=True):
        super().__init__()
        img_size, patch_size = to_2tuple(img_size), to_2tuple(patch_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.grid_size = (img_size[0] // patch_size[0], img_size[1] // patch_size[1])
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv3d(in_chans, embed_dim, kernel_size=(1, patch_size[0], patch_size[1]),
                              stride=(1, patch_size[0], patch_size[1]))
        self.norm = nn.Identity()


class InternVL_CLIP(nn.Module):
    """internvl_clip_vision.py:336-465.  forward(image[B,C,T,H,W]) -> (z[K,B,1+T*HW,C] L2-normalised tap features with
    the per-frame cls tokens averaged over time, x[B,clip_embed_dim] L2-normalised pooled feature, attn[B*T,HW] the
    pooling query's attention over the patches — the importance map of the attention-guided mask)."""

    def __init__(self, in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.2, embed_dim=3200,
                 num_heads=25, mlp_ratio=4, init_values=0.1, qk_normalization=True, depth=48, use_flash_attn=True,
                 use_fused_rmsnorm=True, use_fused_mlp=True, fused_mlp_heuristic=1, with_cp=False,
                 attn_pool_num_heads=16, clip_embed_dim=768, layerscale_no_force_fp32=True, clip_norm_type="l2",
                 return_attn=True, clip_return_layer=1, clip_return_interval=1):
        super().__init__()
        assert use_flash_attn == use_fused_rmsnorm == use_fused_mlp
        self.embed_dim = embed_dim
        self.clip_norm_type = clip_norm_type
        self.return_attn = return_attn
        self.return_index = [depth - int(i * clip_return_interval) - 1 for i in range(clip_return_layer)]
        self.patch_embed = FramePatchEmbed(img_size, patch_size, in_chans, embed_dim)
        self.num_patches = self.patch_embed.num_patches
        self.pos_embed = nn.Parameter(torch.zeros(1, self.num_patches + 1, embed_dim), requires_grad=False)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.blocks, self.clip_projector = vit_stack(
            embed_dim, depth, num_heads, mlp_ratio, drop_path_rate, attn_pool_num_heads, clip_embed_dim,
            qkv_bias=qkv_bias, init_values=init_values, use_flash_attn=use_flash_attn, use_fused_mlp=use_fused_mlp,
            fused_mlp_heuristic=fused_mlp_heuristic, qk_normalization=qk_normalization,
            layerscale_no_force_fp32=layerscale_no_force_fp32, use_fused_rmsnorm=use_fused_rmsnorm)

    @property
    def dtype(self):
        return self.patch_embed.proj.weight.dtype

    @torch.no_grad()
    def forward(self, image):
        check_input(self, image, self.dtype)
        B, C, T, H, W = image.shape
        D, L = self.embed_dim, self.num_patches
        n = L + 1
        frames = image.to(bf16).permute(0, 2, 1, 3, 4).reshape(B * T, C, 1, H, W).contiguous()   # one sequence per frame
        idx = torch.arange(0, n, device=image.device, dtype=torch.int32).repeat(B * T, 1).contiguous()
        h = embed_tokens(self.patch_embed, frames, idx, self.cls_token, self.pos_embed)
        # forward_infer: under no_grad in train mode forward_stream would draw DropPath factors
        h, taps = run_blocks(self.blocks, h, lambda i, blk, h: blk.forward_infer(h, B * T, n), self.return_index)
        z = list(taps.values())
        pooled, attn = self.clip_projector(h.reshape(B * T, n, D), return_attn=self.return_attn)
        if self.clip_norm_type == "l2":
            z = torch.stack(z).reshape(len(z), B, T, n, D)                       # fp32 stream taps
            cls = z[:, :, :, :1].mean(2)                                          # per-frame cls -> one per clip (:451)
            zt = torch.cat([cls, z[:, :, :, 1:].reshape(len(z), B, T * L, D)], dim=2)
            zt = zt / zt.norm(dim=-1, keepdim=True)
            x = pooled.float().view(B, T, -1).mean(1)
            x = x / x.norm(dim=-1, keepdim=True)
        elif self.clip_norm_type == "none":
            zt, x = torch.stack(z), pooled
        else:
            raise NotImplementedError
        if self.return_attn:
            return zt, x, attn[:, 1:]                                             # attn [B*T, n] over cls + patches
        return zt, x


# ------------------------------------------------------------------------------------------------ MAE teacher
class VisionTransformer(nn.Module):
    """videomae.py:207-313 — the VideoMAEv2 teacher.  forward(x[B,C,T,H,W]) -> [K, B, N, C] L2-normalised features of
    the last K blocks (the final LayerNorm is applied to the last block's output before it is tapped, :291-292)."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0,
                 qkv_bias=False, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.0,
                 norm_layer=nn.LayerNorm, init_values=0.0, all_frames=16, tubelet_size=2, mae_norm_type="l2",
                 mae_return_layer=1, mae_return_interval=1, head_axis_attention=True):
        super().__init__()
        # True = what the reference executes: videomae.py:94-97 hands flash_attn_func [B,H,N,d] tensors (FA2's layout is
        # [B,N,H,d]), so the softmax runs over the 16 heads of each token.  False = standard token-axis attention.
        self.head_axis_attention = bool(head_axis_attention)
        self.mae_norm_type = mae_norm_type
        self.return_index = [depth - int(i * mae_return_interval) - 1 for i in range(mae_return_layer)]
        self.tubelet_size, self.depth, self.embed_dim = tubelet_size, depth, embed_dim
        self.patch_embed = TubeletPatchEmbed(img_size, patch_size, in_chans, embed_dim, all_frames, tubelet_size)
        num_patches = self.patch_embed.num_patches
        pre = 2048 if patch_size == 14 else 1568
        if num_patches != pre:
            raise NotImplementedError("ivb200 VideoMAE teacher: only the recipe geometry (8 temporal positions, 14x14 "
                                      "or 16x16 grid) is built; other sizes interpolate the table in the reference")
        self.pos_embed = get_sinusoid_encoding_table(num_patches, embed_dim)        # fixed tensor, not a parameter
        ln = norm_layer if norm_layer is not nn.LayerNorm else nn.LayerNorm
        eps = getattr(ln(8), "eps", 1e-5)
        mk = lambda d: LayerNormB(d, eps=eps)  # noqa: E731
        self.blocks = nn.ModuleList([
            VideoMAEBlock(embed_dim, num_heads, mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale, norm_layer=mk,
                          init_values=init_values) for _ in range(depth)])
        self.norm = mk(embed_dim)
        self.apply(init_weights)

    def get_num_layers(self):
        return len(self.blocks)

    @torch.no_grad()
    def forward(self, x, mask=None):
        if mask is not None:
            raise NotImplementedError("the teacher sees the full clip (engine_for_pretraining.py:102)")
        check_input(self, x, self.patch_embed.proj.weight.dtype)
        B = x.shape[0]
        D, N = self.embed_dim, self.patch_embed.num_patches
        idx = torch.arange(0, N + 1, device=x.device, dtype=torch.int32).repeat(B, 1).contiguous()
        h = embed_tokens(self.patch_embed, x, idx, None, self.pos_embed.to(x.device).float())     # videomae.py:293

        def block(i, blk, h):
            h = blk.forward_infer(h, B, N, head_axis=self.head_axis_attention)
            return self.norm(h) if i == self.depth - 1 else h                     # bf16 [B*N, D] after the last

        h, taps = run_blocks(self.blocks, h, block, self.return_index)
        out = torch.stack([t.float().reshape(B, N, D) for t in taps.values()])
        if self.mae_norm_type == "l2":
            out = out / out.norm(dim=-1, keepdim=True)
        elif self.mae_norm_type != "none":
            raise NotImplementedError
        return out


# ------------------------------------------------------------------------------------------------ mask + targets
def attention_guided_mask(attn, B, mask_ratio, importance=None):
    """engine_for_pretraining.py:105-116.  attn [B*T, N] (teacher pooling attention over the patches of each frame).
    Per frame, N_vis = N - int(N * mask_ratio) patches are kept, drawn WITHOUT replacement with probability
    proportional to attn (torch.multinomial); the cls token is always visible.  Returns bool [B, 1 + T*N], True = masked,
    built on the device (the reference builds it on the host and pays a sync + upload every step, SURVEY App.B-19).
    `importance` ([B*T, N] permutation per frame) injects the draw for parity tests (SURVEY App.B-16)."""
    BT, N = attn.shape
    n_vis = N - int(N * mask_ratio)
    if importance is None:
        importance = torch.multinomial(attn.float(), N)
    masked = torch.ones((BT, N), device=attn.device, dtype=torch.bool)
    masked.scatter_(1, importance[:, :n_vis].to(attn.device), False)
    masked = masked.view(B, -1)
    return torch.cat([torch.zeros((B, 1), device=attn.device, dtype=torch.bool), masked], dim=1)


def select_targets(norm_clip_middle, norm_clip_final, norm_mae, bool_masked_pos, n_visible):
    """engine_for_pretraining.py:118-125: keep the teacher features of the student's visible tokens.
    norm_clip_middle [K,B,1+T*L,C], norm_mae [K',B,T*L,C'] -> ([K,B,n,C], [B,Cf], [K',B,n-1,C']) — one index build
    (bit-exact `x[~mask]` order) and two gathers, no host sync."""
    idx, err = ll.visible_indices(bool_masked_pos, n_visible)
    gi = idx.long()
    K, B, _, C = norm_clip_middle.shape
    tc = torch.gather(norm_clip_middle, 2, gi[None, :, :, None].expand(K, B, n_visible, C))
    Km, _, _, Cm = norm_mae.shape
    gm = (gi[:, 1:] - 1)
    tm = torch.gather(norm_mae, 2, gm[None, :, :, None].expand(Km, B, n_visible - 1, Cm))
    return tc, norm_clip_final, tm, err


class DistillationStep:
    """The body of train_one_epoch (engine_for_pretraining.py:97-166) for the bf16 recipe: frozen teachers -> attention-
    guided mask -> visible-token targets -> student forward + the three 2-2cos losses -> backward -> engine.step().
    Everything stays on the device: no `.item()`, no host-built mask (the reference syncs twice per step there), so
    the whole step can be captured into one CUDA graph (engine.GraphedStep).

      step = DistillationStep(student, engine, clip_teacher, mae_teacher, mask_ratio=0.8)
      loss = step(videos)          # videos [B,3,T_mae,H,W] bf16; the CLIP teacher / student see every td_ratio-th frame
    """

    def __init__(self, student, engine, clip_teacher, mae_teacher, mask_ratio=0.8, td_ratio=1,
                 clip_loss_ratio=(1.0, 1.0), mae_loss_ratio=1.0):
        self.student, self.engine = student, engine
        self.clip_teacher, self.mae_teacher = clip_teacher, mae_teacher
        self.mask_ratio, self.td_ratio = mask_ratio, td_ratio
        self.clip_loss_ratio, self.mae_loss_ratio = clip_loss_ratio, mae_loss_ratio

    @torch.no_grad()
    def targets(self, videos, importance=None):
        B = videos.shape[0]
        mae_videos = videos
        clip_videos = videos[:, :, ::self.td_ratio]                       # :108-110 (tubelet 2 vs 1)
        norm_clip_middle, norm_clip_final, attn = self.clip_teacher(clip_videos)
        norm_mae = self.mae_teacher(mae_videos)
        mask = attention_guided_mask(attn, B, self.mask_ratio, importance)
        N = attn.shape[1]
        n_vis = 1 + (attn.shape[0] // B) * (N - int(N * self.mask_ratio))
        tc, tf, tm, err = select_targets(norm_clip_middle, norm_clip_final, norm_mae, mask, n_vis)
        return clip_videos, mask, n_vis, tc, tf, tm

    def __call__(self, videos, importance=None):
        clip_videos, mask, n_vis, tc, tf, tm = self.targets(videos, importance)
        self.engine.zero_grad()
        lc, lf, lm = self.student.forward_loss(clip_videos.contiguous(), mask, tc, tf, tm, n_visible=n_vis)
        loss = lc * self.clip_loss_ratio[0] + lf * self.clip_loss_ratio[1] + lm * self.mae_loss_ratio
        loss.backward()
        self.engine.step()
        return loss
