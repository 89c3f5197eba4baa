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

from functools import partial

import numpy as np
import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .modules import AttentionPoolingBlock, Block, LayerNormB, RMSNorm, bf16, f32, to_2tuple, trunc_normal_


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
        dpr = [drop_path_rate * i / (depth - 1) if depth > 1 else 0.0 for i in range(depth)]
        self.blocks = nn.ModuleList([
            Block(embed_dim, num_heads, mlp_ratio, qkv_bias=qkv_bias, norm_layer=RMSNorm, drop_path=dpr[i],
                  init_values=init_values, attn_drop=0.0, use_flash_attn=use_flash_attn, use_fused_mlp=use_fused_mlp,
                  fused_mlp_heuristic=fused_mlp_heuristic, with_cp=False, qk_normalization=qk_normalization,
                  layerscale_no_force_fp32=layerscale_no_force_fp32, use_fused_rmsnorm=use_fused_rmsnorm)
            for i in range(depth)])
        self.clip_projector = AttentionPoolingBlock(dim=embed_dim, num_heads=attn_pool_num_heads, qkv_bias=True,
                                                    qk_scale=None, drop=0.0, attn_drop=0.0,
                                                    norm_layer=partial(nn.LayerNorm, eps=1e-5), out_dim=clip_embed_dim)

    @property
    def dtype(self):
        return self.patch_embed.proj.weight.dtype

    @torch.no_grad()
    def forward(self, image):
        if self.dtype != bf16 or not image.is_cuda:
            raise ll._lib.IvbError("ivb200 InternVL_CLIP: bf16 parameters and a CUDA input are required (no CPU path)")
        B, C, T, H, W = image.shape
        D, L = self.embed_dim, self.num_patches
        n = L + 1
        pe = self.patch_embed
        frames = image.to(bf16).permute(0, 2, 1, 3, 4).reshape(B * T, C, 1, H, W).contiguous()   # one sequence per frame
        idx = torch.arange(0, n, device=image.device, dtype=torch.int32).repeat(B * T, 1).contiguous()
        h = ops.EmbedFn.apply(frames, idx, pe.proj.weight, pe.proj.bias, self.cls_token, self.pos_embed, 1, pe.patch_size[0])
        z = []
        for i, blk in enumerate(self.blocks):
            h = blk.forward_infer(h, B * T, n)
            if i in self.return_index:
                z.append(h)
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
def get_sinusoid_encoding_table(n_position, d_hid):
    """videomae.py:152-205 for the recipe case n_position == pre_n_position (8 temporal positions, 14x14 or 16x16 grid):
    the plain 1-D sinusoid table [1, n_position, d_hid] (no interpolation branch)."""
    pos = np.arange(n_position, dtype=np.float64)[:, None]
    hid = np.arange(d_hid)[None, :]
    table = pos / np.power(10000, 2 * (hid // 2) / d_hid)
    table[:, 0::2] = np.sin(table[:, 0::2])
    table[:, 1::2] = np.cos(table[:, 1::2])
    return torch.tensor(table, dtype=torch.float).unsqueeze(0)


class TeacherAttention(nn.Module):
    """videomae.py:62-101 (parameter layout: qkv without bias + separate q_bias / v_bias)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0.0, proj_drop=0.0, attn_head_dim=None):
        super().__init__()
        self.num_heads = num_heads
        head_dim = attn_head_dim if attn_head_dim is not None else dim // num_heads
        all_head_dim = head_dim * num_heads
        self.scale = qk_scale or head_dim ** -0.5
        self.qkv = nn.Linear(dim, all_head_dim * 3, bias=False)
        if qkv_bias:
            self.q_bias = nn.Parameter(torch.zeros(all_head_dim))
            self.v_bias = nn.Parameter(torch.zeros(all_head_dim))
        else:
            self.q_bias = self.v_bias = None
        self.proj = nn.Linear(all_head_dim, dim)

    def qkv_bias_vector(self):
        if self.q_bias is None:
            return None
        return torch.cat((self.q_bias, torch.zeros_like(self.v_bias), self.v_bias))       # :86


class TeacherMlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features or in_features)
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features)


class TeacherBlock(nn.Module):
    """videomae.py:104-132: LayerNorm pre-norm block, optional gamma_1 / gamma_2."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, qk_scale=None, drop=0.0, attn_drop=0.0,
                 drop_path=0.0, init_values=None, act_layer=nn.GELU, norm_layer=nn.LayerNorm, attn_head_dim=None):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = TeacherAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale,
                                     attn_head_dim=attn_head_dim)
        self.norm2 = norm_layer(dim)
        self.mlp = TeacherMlp(dim, int(dim * mlp_ratio))
        if init_values and init_values > 0:
            self.gamma_1 = nn.Parameter(init_values * torch.ones(dim))
            self.gamma_2 = nn.Parameter(init_values * torch.ones(dim))
        else:
            self.gamma_1 = self.gamma_2 = None

    def forward_infer(self, x2d, B, n, head_axis_attention=True):
        """fp32 residual stream [B*n, D] -> same; 9 kernels, nothing saved."""
        a = self.attn
        return ops.block_forward_ln_infer(
            x2d, B, n, a.num_heads, a.scale, head_axis_attention=head_axis_attention, params=
            (self.norm1.weight, self.norm1.bias, self.norm1.eps, a.qkv.weight, a.qkv_bias_vector(), a.proj.weight,
             a.proj.bias, self.gamma_1, self.norm2.weight, self.norm2.bias, self.norm2.eps, self.mlp.fc1.weight,
             self.mlp.fc1.bias, self.mlp.fc2.weight, self.mlp.fc2.bias, self.gamma_2))


class TubeletPatchEmbed(nn.Module):
    """videomae.py:135-149."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, num_frames=16, tubelet_size=2):
        super().__init__()
        img_size, patch_size = to_2tuple(img_size), to_2tuple(patch_size)
        self.tubelet_size = int(tubelet_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.num_patches = (img_size[1] // patch_size[1]) * (img_size[0] // patch_size[0]) * (num_frames // self.tubelet_size)
        self.proj = nn.Conv3d(in_chans, embed_dim, kernel_size=(self.tubelet_size, patch_size[0], patch_size[1]),
                              stride=(self.tubelet_size, patch_size[0], patch_size[1]))


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
            TeacherBlock(embed_dim, num_heads, mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale, norm_layer=mk,
                         init_values=init_values) for _ in range(depth)])
        self.norm = mk(embed_dim)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def get_num_layers(self):
        return len(self.blocks)

    @torch.no_grad()
    def forward(self, x, mask=None):
        if mask is not None:
            raise NotImplementedError("the teacher sees the full clip (engine_for_pretraining.py:102)")
        w = self.patch_embed.proj.weight
        if w.dtype != bf16 or not x.is_cuda:
            raise ll._lib.IvbError("ivb200 VideoMAE teacher: bf16 parameters and a CUDA input are required (no CPU path)")
        B = x.shape[0]
        D, N = self.embed_dim, self.patch_embed.num_patches
        pe = self.patch_embed
        # EmbedFn embeds tokens idx[:, 1:] and puts `cls + pos[0]` in front: give it a zero cls row and drop it again
        idx = torch.arange(0, N + 1, device=x.device, dtype=torch.int32).repeat(B, 1).contiguous()
        pos = torch.cat([torch.zeros(1, 1, D, device=x.device), self.pos_embed.to(x.device).float()], 1).to(bf16)   # videomae.py:293
        zcls = torch.zeros(1, 1, D, device=x.device, dtype=bf16)
        h = ops.EmbedFn.apply(x.to(bf16), idx, pe.proj.weight, pe.proj.bias, zcls, pos, pe.tubelet_size, pe.patch_size[0])
        h = h.reshape(B, N + 1, D)[:, 1:].reshape(B * N, D).contiguous()
        z = []
        for i, blk in enumerate(self.blocks):
            h = blk.forward_infer(h, B, N, self.head_axis_attention)
            if i == self.depth - 1:
                h = self.norm(h)                                                   # bf16 [B*N, D]
            if i in self.return_index:
                z.append(h.float().reshape(B, N, D))
        out = torch.stack(z)
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
