"""Drop-in seams for a model that was CONSTRUCTED BY THE REFERENCE (SURVEY §8b, §7.1 step 2).

  FlashAttention            the reference's attention seam (single_modality/models/flash_attention_class.py:10-70): same
                            ctor and `forward(qkv[B,S,3,H,d], key_padding_mask=None, causal=False) -> (out[B,S,H,d], None)`
                            contract, on the wgmma attention kernels, differentiable.
  patch_flash_attention(m)  swap every `inner_attn` FlashAttention instance of a reference-built model for the one above
                            (the reference's own blocks then call libivb200 for attention and nothing else changes).
  from_reference(m)         rebuild a reference-built PretrainInternVideo2 as the ivb200 model with the same
                            hyper-parameters (read off the module) and the same weights (strict state_dict load): the whole
                            hot path then runs on libivb200.  Returns the new model; `m` is left untouched.

A reference training loop (engines/engine_for_pretraining.py:train_one_epoch) only calls `model(videos, mask)` and
`model.parameters()`: the object returned by from_reference() satisfies both, with the reference's state_dict keys.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .modules import PretrainInternVideo2

bf16 = torch.bfloat16


class FlashAttention(nn.Module):
    """flash_attention_class.py:10-70.  Only what the pre-training path uses is built: equal-length sequences
    (no key_padding_mask / cu_seqlens), non-causal, no dropout — anything else raises like the reference's asserts."""

    def __init__(self, softmax_scale=None, attention_dropout=0.0, device=None, dtype=None):
        super().__init__()
        self.softmax_scale = softmax_scale
        self.dropout_p = attention_dropout

    def forward(self, qkv, key_padding_mask=None, causal=False, cu_seqlens=None, max_s=None, need_weights=False):
        assert not need_weights
        assert qkv.dtype in (torch.float16, torch.bfloat16)
        assert qkv.is_cuda
        if key_padding_mask is not None or cu_seqlens is not None:
            raise NotImplementedError("ivb200 FlashAttention: variable-length batches are not on the pre-training path "
                                      "(internvideo2_pretrain.py:208-210 passes key_padding_mask=None)")
        if causal or (self.dropout_p and self.training):
            raise NotImplementedError("ivb200 FlashAttention: causal / dropout are not on the pre-training path")
        if qkv.dtype != bf16:
            raise ll._lib.IvbError("ivb200 FlashAttention computes in bf16 (the recipe's dtype)")
        B, S, three, H, d = qkv.shape
        assert three == 3
        flat = qkv.reshape(B * S, 3 * H * d)              # row = token, columns = q | k | v, each (h d): a view
        D = H * d
        scale = self.softmax_scale if self.softmax_scale is not None else d ** -0.5
        out = ops.AttnFn.apply(flat[:, :D], flat[:, D:2 * D], flat[:, 2 * D:], B, S, H, d, scale)
        return out.reshape(B, S, H, d), None


def patch_flash_attention(model: nn.Module) -> int:
    """Replace every sub-module attribute named `inner_attn` (the reference's FlashAttention instances,
    internvideo2_pretrain.py:166) by the ivb200 FlashAttention.  Returns how many were swapped."""
    n = 0
    for mod in model.modules():
        inner = getattr(mod, "inner_attn", None)
        if isinstance(inner, nn.Module) and not isinstance(inner, FlashAttention):
            mod.inner_attn = FlashAttention(softmax_scale=getattr(inner, "softmax_scale", None),
                                            attention_dropout=getattr(inner, "dropout_p", 0.0))
            n += 1
    return n


def reference_config(ref) -> dict:
    """Constructor kwargs of PretrainInternVideo2 read off a reference-built instance (shapes + attributes)."""
    sd = ref.state_dict()
    blk0 = ref.blocks[0]
    D = ref.embed_dim
    pe = ref.patch_embed
    depth = len(ref.blocks)
    Hd = sd["blocks.0.mlp.fc1.weight"].shape[0]
    cfg = dict(
        in_chans=pe.proj.weight.shape[1], patch_size=pe.patch_size[0], img_size=pe.img_size[0],
        qkv_bias=blk0.attn.qkv.bias is not None, embed_dim=D, num_heads=blk0.attn.num_heads, mlp_ratio=Hd / D,
        init_values=float(sd["blocks.0.ls1.gamma"].float().mean()) if "blocks.0.ls1.gamma" in sd else None,
        qk_normalization=bool(getattr(blk0.attn, "qk_normalization", False)), depth=depth,
        attn_pool_num_heads=ref.clip_projector.cross_attn.num_heads,
        clip_embed_dim=sd["clip_projector.cross_attn.proj.weight"].shape[0],
        num_frames=pe.grid_size[0] * pe.proj.weight.shape[2], tubelet_size=pe.proj.weight.shape[2],
        sep_pos_embed=bool(getattr(ref, "sep_pos_embed", False)),
        clip_teacher_embed_dim=sd["clip_decoder.0.head.weight"].shape[0],
        clip_teacher_final_dim=sd["final_clip_decoder.head.weight"].shape[0] if "final_clip_decoder.head.weight" in sd else 0,
        clip_norm_type=ref.clip_norm_type, clip_return_layer=len(ref.clip_return_index),
        mae_teacher_embed_dim=sd["mae_decoder.0.head.2.weight"].shape[0], mae_norm_type=ref.mae_norm_type,
        mae_return_layer=len(ref.mae_return_index),
        use_flash_attn=bool(ref.use_flash_attn), use_fused_rmsnorm=bool(ref.use_flash_attn), use_fused_mlp=bool(ref.use_flash_attn),
        use_checkpoint=any(getattr(b, "with_cp", False) for b in ref.blocks),
        checkpoint_num=sum(1 for b in ref.blocks if getattr(b, "with_cp", False)),
    )
    ci, mi = sorted(ref.clip_return_index, reverse=True), sorted(ref.mae_return_index, reverse=True)
    cfg["clip_student_return_interval"] = (ci[0] - ci[1]) if len(ci) > 1 else 1
    cfg["mae_student_return_interval"] = (mi[0] - mi[1]) if len(mi) > 1 else 1
    dp = [getattr(getattr(b, "drop_path1", None), "drop_prob", 0.0) or 0.0 for b in ref.blocks]
    cfg["drop_path_rate"] = float(dp[-1]) if dp else 0.0
    if cfg["init_values"] is None:
        cfg.pop("init_values")
    return cfg


def from_reference(ref, dtype=bf16, device="cuda") -> PretrainInternVideo2:
    """ivb200 PretrainInternVideo2 with the hyper-parameters and weights of the reference-built `ref`."""
    cfg = reference_config(ref)
    init = cfg.pop("init_values", 1e-5)
    model = PretrainInternVideo2(init_values=init, **cfg)
    model.load_state_dict(ref.state_dict(), strict=True)
    model.train(ref.training)
    return model.to(dtype=dtype, device=device) if device is not None else model.to(dtype=dtype)
