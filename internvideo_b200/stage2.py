"""Stage-2 consumers of the tower (SURVEY §8 f-3): the multi-modality form of the student backbone, the unmasked-teacher
alignment loss, the hard-negative sampler of the video-text matching loss, and the retrieval score matrices.

  PretrainInternVideo2     multi_modality/models/backbones/internvideo2/internvideo2.py:380-668 — same ctor kwargs, same
                           state_dict keys, same forward contract:
                           forward(x[B,C,T,H,W], mask=None, use_image=False, x_vis_return_idx=-1, x_vis_only=False)
                             -> x_vis[B,n,D]                                        (x_vis_only)
                             -> (x_vis, x_pool_vis[B,Ce], x_clip_align[K,B,n,Ct], x_align[B,Cf])
                           The blocks, the embed gather, the pooling projector and the decoders are the libivb200 kernels
                           of modules.py; only the optional mask / image position tables / early exit are new.
  UTA_Loss                 criterions.py:345-385  (student vs unmasked-teacher alignment, l2 / mse / smooth_l1)
  vtm_negatives            criterions.py:133-153  (the sampling half of VTC_VTM_Loss.vtm_loss; the fusion encoder that consumes
                           the negatives is a BERT text tower and out of scope, DESIGN §9)
  retrieval_scores         tasks_clip/retrieval_utils.py:137-151 (dot-product scores + dual-softmax re-weighting)
  ensemble_clip_scores     tasks_clip/retrieval_utils.py:430-438 (mean / max / lse over the clips of one video)

The text tower (BERT), the MLM loss and the ITM head stay outside (DESIGN §9): they are consumers of `vision_embeds`, not part
of the video path.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import lowlevel as ll
from . import ops
from .modules import PretrainInternVideo2 as _SingleModalityTower
from .modules import _pos_tensor, get_3d_sincos_pos_embed, index_poison

bf16, f32 = torch.bfloat16, torch.float32


class PretrainInternVideo2(_SingleModalityTower):
    """internvideo2.py:380-668.  Differences to the single-modality tower (modules.PretrainInternVideo2): no MAE branch,
    `mask` is optional, images use the temporal mean of the video position table (or their own tables with
    `sep_image_video_pos_embed`), the block loop can stop early (`x_vis_return_idx`) and `x_vis` is returned."""

    pos_prefixes = ("", "clip_")         # the stage-2 tower has no MAE branch (keys must match the reference's)

    def __init__(self, in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.25, embed_dim=1408,
                 num_heads=16, mlp_ratio=4.3637, init_values=1e-5, qk_normalization=True, depth=40, use_flash_attn=True,
                 use_fused_rmsnorm=True, use_fused_mlp=True, fused_mlp_heuristic=1, attn_pool_num_heads=16,
                 clip_embed_dim=768, layerscale_no_force_fp32=False, num_frames=8, tubelet_size=1, sep_pos_embed=False,
                 sep_image_video_pos_embed=False, use_checkpoint=False, checkpoint_num=0, clip_teacher_embed_dim=3200,
                 clip_teacher_final_dim=768, clip_norm_type="l2", clip_return_layer=1, clip_student_return_interval=1):
        if sep_pos_embed:
            raise NotImplementedError          # internvideo2.py:449
        super().__init__(in_chans=in_chans, patch_size=patch_size, img_size=img_size, qkv_bias=qkv_bias,
                         drop_path_rate=drop_path_rate, embed_dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio,
                         init_values=init_values, qk_normalization=qk_normalization, depth=depth,
                         use_flash_attn=use_flash_attn, use_fused_rmsnorm=use_fused_rmsnorm, use_fused_mlp=use_fused_mlp,
                         fused_mlp_heuristic=fused_mlp_heuristic, attn_pool_num_heads=attn_pool_num_heads,
                         clip_embed_dim=clip_embed_dim, layerscale_no_force_fp32=layerscale_no_force_fp32,
                         num_frames=num_frames, tubelet_size=tubelet_size, sep_pos_embed=False,
                         use_checkpoint=use_checkpoint, checkpoint_num=checkpoint_num,
                         clip_teacher_embed_dim=clip_teacher_embed_dim, clip_teacher_final_dim=clip_teacher_final_dim,
                         clip_norm_type=clip_norm_type, clip_return_layer=clip_return_layer,
                         clip_student_return_interval=clip_student_return_interval, mae_return_layer=0)
        self.return_index = self.clip_return_index
        self.num_frames = num_frames
        self.tubelet_size = tubelet_size
        self.image_pos_groups = num_frames      # :601,663 — an image's table averages groups of frames, not tubelets
        self.sep_image_video_pos_embed = bool(sep_image_video_pos_embed)
        self.num_img_patches = self.patch_embed.grid_size[1] * self.patch_embed.grid_size[2]
        if self.sep_image_video_pos_embed:      # :455-460 — images get their own tables
            t = get_3d_sincos_pos_embed(embed_dim, self.patch_embed.grid_size[1], 1, cls_token=True)
            self.img_pos_embed = nn.Parameter(_pos_tensor(t))
            self.clip_img_pos_embed = nn.Parameter(_pos_tensor(t))

    @torch.jit.ignore
    def no_weight_decay(self):
        return super().no_weight_decay() | {"img_pos_embed", "clip_img_pos_embed"}

    def forward(self, x, mask=None, use_image=False, x_vis_return_idx=-1, x_vis_only=False):
        B, ntok = x.shape[0], 1 + (x.shape[2] // self.patch_embed.tubelet_size) * self.num_img_patches
        n_visible = None
        if mask is None:                                      # every token visible (:613-616)
            mask = torch.zeros((B, ntok), dtype=torch.bool, device=x.device)
            n_visible = ntok
        taps, h, idx, B, n = self.forward_features(x, mask, n_visible, use_image=use_image,
                                                   last=self.depth + x_vis_return_idx)      # early exit (:631-633)
        D = self.embed_dim
        x_vis = h.reshape(B, n, D).to(bf16)
        x_vis = x_vis + index_poison(self.index_error).to(bf16)   # ragged mask -> NaN (the reference's reshape raises)
        if x_vis_only:
            return x_vis
        x_pool_vis = self.clip_projector(h.reshape(B, n, D))
        x_align = self.final_clip_decoder(x_pool_vis)
        cpe = self._pos_table("clip_", use_image)
        # the reference stacks the taps in block order (x_clip.append inside the loop) and feeds decoder k with tap k
        clip_in = [ops.GatherAddFn.apply(taps[i], cpe, idx, B, n, 0, 0) for i in sorted(taps)]
        x_clip_align = torch.stack([dec(xi).reshape(B, n, -1) for dec, xi in zip(self.clip_decoder, clip_in)])
        return x_vis, x_pool_vis, x_clip_align, x_align


def pretrain_internvideo2_1b_patch14_224(config):
    """internvideo2.py:671-700 — built from `config.vision_encoder` like the reference factory."""
    ve = config.vision_encoder
    g = ve.get if hasattr(ve, "get") else (lambda k, d=None: getattr(ve, k, d))
    return PretrainInternVideo2(
        in_chans=3, img_size=224, patch_size=14, embed_dim=1408, depth=40, num_heads=16, mlp_ratio=48 / 11,
        clip_embed_dim=g("clip_embed_dim"), attn_pool_num_heads=16, qkv_bias=False, drop_path_rate=0.25, init_values=1e-5,
        qk_normalization=True, use_flash_attn=g("use_flash_attn", True), use_fused_rmsnorm=g("use_fused_rmsnorm", True),
        use_fused_mlp=g("use_fused_mlp", True), fused_mlp_heuristic=1, layerscale_no_force_fp32=False,
        num_frames=g("num_frames"), tubelet_size=g("tubelet_size"), sep_pos_embed=False,
        sep_image_video_pos_embed=g("sep_image_video_pos_embed"), use_checkpoint=g("use_checkpoint"),
        checkpoint_num=g("checkpoint_num"), clip_teacher_embed_dim=g("clip_teacher_embed_dim"),
        clip_teacher_final_dim=g("clip_teacher_final_dim"), clip_norm_type=g("clip_norm_type"),
        clip_return_layer=g("clip_return_layer"), clip_student_return_interval=g("clip_student_return_interval"))


class UTA_Loss(nn.Module):
    """criterions.py:345-385 — alignment of the student's decoder outputs with the unmasked teacher's features."""

    def __init__(self, uta_norm_type="l2", uta_loss_type="l2"):
        super().__init__()
        self.norm_type, self.loss_type = uta_norm_type, uta_loss_type
        if uta_loss_type == "mse":
            self.loss_func = nn.MSELoss()
        elif uta_loss_type == "smooth_l1":
            self.loss_func = nn.SmoothL1Loss()

    def _norm(self, t):
        if self.norm_type == "l2":
            return t / t.norm(dim=-1, keepdim=True)
        if self.norm_type == "none":
            return t
        raise NotImplementedError

    def uta_loss(self, student_output, clip_output):
        s, c = self._norm(student_output), self._norm(clip_output)
        if self.loss_type == "l2":
            return (2 - 2 * (s * c).sum(dim=-1)).mean()
        if self.loss_type in ("mse", "smooth_l1"):
            return self.loss_func(input=s, target=c)
        raise NotImplementedError

    def uta_vision_loss(self, student_v_output, clip_v_output):          # criterions.py:387-418
        if student_v_output.shape[1] != clip_v_output.shape[1]:
            student_v_output = student_v_output.mean(1, keepdim=True)
            clip_v_output = clip_v_output.mean(1, keepdim=True)
        return self.uta_loss(student_v_output, clip_v_output)

    def uta_all_loss(self, student_v_output, clip_v_output, student_t_output, clip_t_output):   # criterions.py:420-470
        lv = self.uta_vision_loss(student_v_output, clip_v_output)
        lt = self.uta_loss(student_t_output, clip_t_output)
        return (lv + lt) / 2.0


def positive_mask(sim, idx=None):
    """criterions.py:200-216 `get_mask`: 1 where (i, j) is a positive pair (same idx, or the diagonal without idx)."""
    if idx is not None:
        idx = idx.view(-1, 1)
        return torch.eq(idx, idx.T).to(sim.dtype)
    mask = torch.zeros_like(sim)
    mask.fill_diagonal_(1)
    return mask


def rand_indices(mask, k):
    """criterions.py:184-198 `get_rand_indices`: k random allowed (mask == 0) columns per row."""
    m = mask.float()
    m = m - 10000 * m
    m = m + torch.randn_like(m)
    _, indices = torch.sort(m, dim=1, descending=True)
    return indices[:, :k].contiguous()


@torch.no_grad()
def vtm_negatives(sim_v2t, sim_t2v, idx=None, hard=True):
    """criterions.py:133-153 — one negative video per text and one negative text per video.  hard: sampled from the
    softmax of the similarities with the positives masked out; else uniformly among the non-positives.
    Returns (vision_neg_indices[B], txt_neg_indices[B]).  Draws from the global RNG in the reference's order."""
    weights_v2t = F.softmax(sim_v2t + 1e-4, dim=1)
    weights_t2v = F.softmax(sim_t2v + 1e-4, dim=1)
    mask = positive_mask(sim_v2t, idx=idx).bool()
    weights_v2t.masked_fill_(mask, 0)
    weights_t2v.masked_fill_(mask, 0)
    weights_v2t = torch.nan_to_num_(weights_v2t, nan=1e-2, posinf=1e-2, neginf=1e-2)
    weights_t2v = torch.nan_to_num_(weights_t2v, nan=1e-2, posinf=1e-2, neginf=1e-2)
    if hard:
        vision_neg = torch.multinomial(weights_t2v, 1).squeeze()
        txt_neg = torch.multinomial(weights_v2t, 1).squeeze()
    else:
        vision_neg = rand_indices(mask, 1).squeeze()
        txt_neg = rand_indices(mask, 1).squeeze()
    return vision_neg, txt_neg


def vtm_triplets(vision_embeds, text_embeds, text_atts, vision_neg, txt_neg):
    """criterions.py:155-165 — the 3B (video, text) pairs handed to the fusion encoder: B positives, B with a negative video,
    B with a negative text, plus the labels (1 for the first B)."""
    vision_all = torch.cat([vision_embeds, vision_embeds[vision_neg], vision_embeds], dim=0)
    text_all = torch.cat([text_embeds, text_embeds, text_embeds[txt_neg]], dim=0)
    atts_all = torch.cat([text_atts, text_atts, text_atts[txt_neg]], dim=0)
    bs = vision_embeds.shape[0]
    labels = torch.ones(3 * bs, dtype=torch.long, device=vision_embeds.device)
    labels[bs:] = 0
    return vision_all, text_all, atts_all, labels


@torch.no_grad()
def get_sim(vision_proj, text_proj, temp=1.0, agg_method="mean"):
    """criterions.py:15-55 — cosine similarities / temp, both directions.  vision_proj [B,C] or [B,T,C] (per-frame), text
    [B,C] or [B,1/K,C].  CUDA bf16/fp32 inputs run the [B,B] product on the wgmma GEMM (fp32 accumulate)."""
    v = F.normalize(vision_proj.float(), dim=-1)
    t = F.normalize(text_proj.float(), dim=-1)
    if v.ndim == 3:
        sim_v2t = torch.einsum("mld,nd->mln", v, t) / temp
        sim_t2v = torch.einsum("nd,mld->nlm", t, v) / temp
        if agg_method == "mean":
            return sim_v2t.mean(1), sim_t2v.mean(1)
        if agg_method == "max":
            return sim_v2t.max(1)[0], sim_t2v.max(1)[0]
        raise ValueError(agg_method)
    if t.ndim == 3:
        sim_v2t = torch.einsum("nd,mld->nlm", v, t) / temp
        sim_t2v = torch.einsum("nld,md->nlm", t, v) / temp
        if agg_method == "mean":
            return sim_v2t.mean(1), sim_t2v.mean(1)
        if agg_method == "max":
            return sim_v2t.max(1)[0], sim_t2v.max(1)[0]
        raise ValueError(agg_method)
    if v.is_cuda and v.shape[1] % 8 == 0 and t.shape[0] % 8 == 0 and v.shape[0] >= 8:
        # fp32-faithful product on the bf16 tensor cores: x = hi + lo with both halves bf16 (|lo| <= 2^-9 |x|), the
        # lo*lo term (<= 2^-18) is dropped — rank order of near-ties matters for recall@k
        vh, th = v.to(bf16), t.to(bf16)
        vl, tl = (v - vh.float()).to(bf16), (t - th.float()).to(bf16)
        sim = ll.gemm(vh, th, epi=ll.EPI_F32) + ll.gemm(vh, tl, epi=ll.EPI_F32) + ll.gemm(vl, th, epi=ll.EPI_F32)
        sim = sim / temp
    else:
        sim = v @ t.T / temp
    return sim, sim.T


@torch.no_grad()
def retrieval_scores(image_feats, text_feats):
    """retrieval_utils.py:137-151 — dot-product scores of all (video, text) pairs and their dual-softmax re-weighting.
    Returns (i2t_dsl, t2i_dsl, i2t, t2i) as fp32 tensors ([Nv, Nt], [Nt, Nv], [Nv, Nt], [Nt, Nv])."""
    i2t, t2i = get_sim(image_feats, text_feats)
    i2t_dsl = i2t * i2t.softmax(dim=0)
    t2i_dsl = i2t.T * i2t.T.softmax(dim=0)
    return i2t_dsl.float(), t2i_dsl.float(), i2t.float(), i2t.T.float()


def ensemble_clip_scores(clip_scores, mode="mean"):
    """retrieval_utils.py:430-438 — combine the scores of the #clip views of one video ([#clip, k] -> [k])."""
    if mode == "mean":
        return clip_scores.mean(0)
    if mode == "max":
        return clip_scores.max(0)[0]
    if mode == "lse":
        return torch.logsumexp(clip_scores, dim=0)
    raise ValueError("config.evaluation.eval_frame_ensemble must in [mean, max, lse] when #clip > 1.")


@torch.no_grad()
def recall_at_k(scores_i2t, scores_t2i, txt2img, img2txt, ks=(1, 5, 10)):
    """retrieval_utils.py:463-520 `itm_eval` — recall@k of both directions from the score matrices.  txt2img[t] = the video
    of caption t (int or list), img2txt[i] = the captions of video i (int or list)."""
    import numpy as np
    s_i2t = scores_i2t.detach().float().cpu().numpy() if torch.is_tensor(scores_i2t) else np.asarray(scores_i2t)
    s_t2i = scores_t2i.detach().float().cpu().numpy() if torch.is_tensor(scores_t2i) else np.asarray(scores_t2i)

    def ranks_of(scores, gt):
        ranks = np.zeros(scores.shape[0])
        for i, row in enumerate(scores):
            inds = np.argsort(row)[::-1]
            g = gt[i]
            g = [g] if isinstance(g, (int, np.integer)) else list(g)
            ranks[i] = min(int(np.where(inds == j)[0][0]) for j in g)
        return ranks

    r_i2t, r_t2i = ranks_of(s_i2t, img2txt), ranks_of(s_t2i, txt2img)
    out = {}
    for k in ks:
        out[f"txt_r{k}"] = 100.0 * float((r_i2t < k).mean())      # the reference calls video->text recall "txt_r"
        out[f"img_r{k}"] = 100.0 * float((r_t2i < k).mean())
    out["txt_r_mean"] = sum(out[f"txt_r{k}"] for k in ks) / len(ks)
    out["img_r_mean"] = sum(out[f"img_r{k}"] for k in ks) / len(ks)
    out["r_mean"] = (out["txt_r_mean"] + out["img_r_mean"]) / 2
    return {k: round(v, 2) for k, v in out.items()}
