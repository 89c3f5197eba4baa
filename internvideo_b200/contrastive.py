"""Video-text contrastive loss with the cross-rank embedding all-gather (BASELINE cfg-3 hot path).

Mirrors InternVideo2/multi_modality/models/criterions.py (`get_sim` :15-55, `VTC_VTM_Loss.vtc_loss`
:65-103, `get_mask` :200-216) and models/utils.py `AllGather` (:193-212):

  * forward: ONE NCCL all-gather of a packed [B_loc, 2C+pad] buffer (vision | text | idx) instead of
    the reference's three collectives, then normalise -> wgmma sim GEMM -> fused two-direction
    soft-target cross-entropy (libivb200);
  * backward: NO collective — each rank keeps only the gradient rows of its own samples, exactly like
    `AllGather.backward` (models/utils.py:205-209); the usual gradient all-reduce of the data-parallel
    engine follows.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import ops


def pack_for_gather(vision_proj, text_proj, idx):
    """[B, C] x2 (+ int64 idx) -> one fp32 row-packed buffer [B, 2C + 2] (idx split into two exact
    24-bit halves so it survives the float transport bit-exactly for idx < 2^48)."""
    B, C = vision_proj.shape
    buf = torch.empty((B, 2 * C + 2), device=vision_proj.device, dtype=torch.float32)
    buf[:, :C] = vision_proj.detach().float()
    buf[:, C:2 * C] = text_proj.detach().float()
    if idx is None:
        idx = torch.full((B,), -1, device=vision_proj.device, dtype=torch.int64)
    i64 = idx.to(torch.int64)
    buf[:, 2 * C] = (i64 >> 24).float()
    buf[:, 2 * C + 1] = (i64 & 0xFFFFFF).float()
    return buf


def unpack_gathered(buf, C):
    v = buf[:, :C]
    t = buf[:, C:2 * C]
    idx = (buf[:, 2 * C].to(torch.int64) << 24) | buf[:, 2 * C + 1].to(torch.int64)
    return v, t, idx


def gather_embeddings(vision_proj, text_proj, idx, group=None):
    """All ranks' rows concatenated in rank order (== torch.cat(all_gather(...)) of AllGather.forward).
    Returns (v_all, t_all, idx_all, rank, b_local); the local rows are re-inserted WITH autograd so the
    loss back-propagates to this rank's samples only."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B, C = vision_proj.shape
    if world == 1:
        i = idx if idx is not None else torch.arange(B, device=vision_proj.device)
        return vision_proj, text_proj, i.to(torch.int64), 0, B
    packed = pack_for_gather(vision_proj, text_proj, idx)
    out = torch.empty((world * B, packed.shape[1]), device=packed.device, dtype=packed.dtype)
    dist.all_gather_into_tensor(out, packed, group=group)
    v_all, t_all, idx_all = unpack_gathered(out, C)
    if idx is None:
        idx_all = torch.arange(world * B, device=packed.device, dtype=torch.int64)
    lo, hi = rank * B, (rank + 1) * B
    v_all = torch.cat([v_all[:lo], vision_proj.float(), v_all[hi:]], dim=0)
    t_all = torch.cat([t_all[:lo], text_proj.float(), t_all[hi:]], dim=0)
    return v_all, t_all, idx_all, rank, B


class VTC_VTM_Loss(torch.nn.Module):
    """Drop-in for criterions.VTC_VTM_Loss (vtc_loss only; VTM/MLM need the BERT towers, out of scope)."""

    def __init__(self, vtm_hard_neg=False, process_group=None):
        super().__init__()
        self.vtm_hard_neg = vtm_hard_neg
        self.process_group = process_group

    def vtc_loss(self, vision_proj, text_proj, idx, temp=1.0, all_gather=True, agg_method="mean"):
        if vision_proj.ndim != 2 or text_proj.ndim != 2:
            raise NotImplementedError("ivb200 vtc_loss: only the [B,C] x [B,C] branch of get_sim (criterions.py:51-53)")
        if all_gather:
            v_all, t_all, idx_all, rank, bl = gather_embeddings(vision_proj, text_proj, idx, self.process_group)
        else:
            B = vision_proj.shape[0]
            v_all, t_all, rank, bl = vision_proj, text_proj, 0, B
            idx_all = idx if idx is not None else torch.arange(B, device=vision_proj.device)
        return ops.VtcLossFn.apply(v_all, t_all, idx_all.to(torch.int64), temp, rank, bl)
