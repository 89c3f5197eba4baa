"""Video-text contrastive pre-training surface (BASELINE cfg-3): the unmasked InternVideo2 vision tower and the
InternVideo2_CLIP_small wrapper, on the same libivb200 kernels as the masked student.

Mirrors (constructor kwargs, attribute names, state_dict keys, forward contracts):
  InternVideo2/multi_modality/models/backbones/internvideo2/internvideo2_clip_vision.py:340-548  `InternVideo2`
  InternVideo2/multi_modality/models/internvideo2_clip_small.py:18-257                           `InternVideo2_CLIP_small`
  InternVideo2/multi_modality/models/internvideo2_clip.py:16-254                                  `InternVideo2_CLIP`
  InternVideo2/multi_modality/models/backbones/internvideo2/pos_embed.py:137-182                 `interpolate_pos_embed`

InternVideo2_CLIP_small takes any module/callable as `text_encoder`: text_modules.TextTransformer is the recipe's
MobileCLIP-B tower on the libivb200 kernels; the default accepts pre-computed text embeddings.  InternVideo2_CLIP (the
1B and 6B recipes) builds llama_modules.LLaMA, the frozen LLaMA-7B tower, unless it is given one.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .contrastive import VTC_VTM_Loss
from .llama_modules import LLaMA
from .modules import InternVideo2Tower, LayerNormB, check_input, embed_tokens, run_blocks


class InternVideo2(InternVideo2Tower):
    """internvideo2_clip_vision.py:340-548 — unmasked tower: every one of the 1 + T*L tokens goes through the
    blocks, then the attention-pooling projector.  forward(x[B,C,T,H,W], use_image=False) -> [B, clip_embed_dim]."""

    def __init__(self, in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.25,
                 head_drop_path_rate=0.0, embed_dim=1408, num_heads=16, mlp_ratio=48 / 11, init_values=1e-5,
                 qk_normalization=True, depth=40, use_flash_attn=True, use_fused_rmsnorm=True, use_fused_mlp=True,
                 fused_mlp_heuristic=1, attn_pool_num_heads=16, clip_embed_dim=768, layerscale_no_force_fp32=False,
                 num_frames=8, tubelet_size=1, sep_pos_embed=False, use_checkpoint=False, checkpoint_num=0):
        if head_drop_path_rate:
            raise NotImplementedError("ivb200 InternVideo2: head_drop_path_rate is 0 in every recipe")
        super().__init__(in_chans, patch_size, img_size, qkv_bias, drop_path_rate, embed_dim, num_heads, mlp_ratio,
                         init_values, qk_normalization, depth, use_flash_attn, use_fused_rmsnorm, use_fused_mlp,
                         fused_mlp_heuristic, attn_pool_num_heads, clip_embed_dim, layerscale_no_force_fp32, num_frames,
                         tubelet_size, sep_pos_embed, use_checkpoint, checkpoint_num)
        self.T = num_frames // tubelet_size
        self.num_frames, self.tubelet_size = num_frames, tubelet_size
        self.fc_norm = nn.Identity()
        self.init_tower()

    # ---- forward (:497-548)
    def forward_tokens(self, x, use_image=False):
        """-> fp32 residual stream [B*n, D] after the last block, B, n."""
        check_input(self, x, self.dtype)
        B = x.shape[0]
        pe = self.patch_embed
        n = 1 + (x.shape[2] // pe.tubelet_size) * pe.grid_size[1] * pe.grid_size[2]
        idx = torch.arange(0, n, device=x.device, dtype=torch.int32).repeat(B, 1).contiguous()   # nothing is masked
        h = embed_tokens(pe, x, idx, self.cls_token, self._pos_table("", use_image))
        h, _ = run_blocks(self.blocks, h, lambda i, blk, h: blk.forward_stream(h, B, n))
        return h, B, n

    def forward(self, x, use_image=False):
        h, B, n = self.forward_tokens(x, use_image)
        x = self.clip_projector(h.reshape(B, n, self.embed_dim))
        return self.fc_norm(x)


def _get(cfg, key, default=None):
    """config access for EasyDict / dict / namespace alike."""
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


class PrecomputedText(nn.Module):
    """Stand-in for the out-of-scope text tower: `text` is already a [B, C] embedding tensor."""

    def forward(self, text):
        if isinstance(text, dict):
            text = text["embeds"]
        return text


class InternVideo2_CLIP_small(nn.Module):
    """internvideo2_clip_small.py:18-142.  `config.model.vision_encoder.*`, `config.model.{temp,temp_min,
    freeze_vision,open_vision_clip_projector}` as in scripts/pretraining/clip/*/config.py.  forward(image[B,T,C,H,W],
    text, idx) -> dict(loss_vtc=...)."""

    def __init__(self, config, tokenizer=None, is_pretrain=True, text_encoder=None, process_group=None):
        super().__init__()
        self.config = config
        self.tokenizer = tokenizer
        self.is_pretrain = is_pretrain
        m = _get(config, "model")
        ve = _get(m, "vision_encoder")
        self.vision_encoder = self.build_vision_encoder()
        ced, ad = _get(ve, "clip_embed_dim"), _get(ve, "align_dim")
        self.vision_align = nn.Sequential(LayerNormB(ced), nn.Linear(ced, ad))
        self.text_encoder = text_encoder if text_encoder is not None else PrecomputedText()
        self.temp = nn.Parameter(torch.ones([]) * _get(m, "temp"))
        self.temp_min = _get(m, "temp_min")
        if _get(m, "freeze_vision", False):
            for name, p in self.vision_encoder.named_parameters():
                if not (_get(m, "open_vision_clip_projector", False) and name.startswith("clip_projector")):
                    p.requires_grad = False
        # The reference's loop (internvideo2_clip_small.py:55-58) logs "Freeze" but never sets requires_grad, so its text
        # tower keeps training; here freeze_text freezes it.  Leave freeze_text off to train the tower end to end.
        if _get(m, "freeze_text", False) and isinstance(self.text_encoder, nn.Module):
            for name, p in self.text_encoder.named_parameters():
                if not (_get(m, "open_text_projection", False) and name.startswith("projection_layer")):
                    p.requires_grad = False
        self.clip_loss = VTC_VTM_Loss(False, process_group=process_group)

    def no_weight_decay(self):
        ret = {"temp"}
        ret.update({"vision_encoder." + k for k in self.vision_encoder.no_weight_decay()})
        if isinstance(self.text_encoder, nn.Module):
            ret.update({"text_encoder." + k for k, _ in self.text_encoder.named_parameters()})
        return ret

    @torch.no_grad()
    def clip_contrastive_temperature(self):
        self.temp.clamp_(min=self.temp_min)        # in place on the device (:96-99), no host read

    def build_vision_encoder(self):
        ve = _get(_get(self.config, "model"), "vision_encoder")
        keys = ("in_chans", "patch_size", "img_size", "qkv_bias", "drop_path_rate", "head_drop_path_rate", "embed_dim",
                "num_heads", "mlp_ratio", "init_values", "qk_normalization", "depth", "use_flash_attn",
                "use_fused_rmsnorm", "use_fused_mlp", "fused_mlp_heuristic", "attn_pool_num_heads", "clip_embed_dim",
                "layerscale_no_force_fp32", "num_frames", "tubelet_size", "sep_pos_embed", "use_checkpoint",
                "checkpoint_num")
        return InternVideo2(**{k: _get(ve, k) for k in keys if _get(ve, k) is not None})

    def encode_vision(self, image, test=False):
        """image [B,T,C,H,W] -> [B, align_dim] (:125-142).  With the recipe's frozen tower the blocks run on the
        no-grad path (nothing saved) and only the attention-pooling projector + vision_align are differentiated."""
        v = tower_embeds(self.vision_encoder, image)
        ln, fc = self.vision_align[0], self.vision_align[1]
        return ops.linear(ln(v), fc.weight, fc.bias)

    def encode_text(self, text):
        return self.text_encoder(text)

    def forward(self, image, text, idx):
        self.clip_contrastive_temperature()
        vision_embeds = self.encode_vision(image)
        text_embeds = self.encode_text(text)
        loss_vtc = self.clip_loss.vtc_loss(vision_embeds, text_embeds, idx, self.temp, all_gather=True)
        return dict(loss_vtc=loss_vtc)

    # ---- checkpoint interop (:200-257)
    def load_checkpoint(self, vision_ckpt_path=None, text_ckpt_path=None, extra_ckpt_path=None):
        m = _get(self.config, "model")
        new_ckpt = {}
        if vision_ckpt_path is not None:
            ck = torch.load(vision_ckpt_path, map_location="cpu")
            new_ckpt.update(remap_vision_checkpoint(
                ck, self.vision_encoder, from_stage2=_get(m, "load_vision_ckpt_from_internvideo2_stage2", False),
                orig_t_size=_get(m, "vision_ckpt_t_size", 4)))
        if text_ckpt_path is not None and isinstance(self.text_encoder, nn.Module):
            tk = torch.load(text_ckpt_path, map_location="cpu")
            tk = tk.get("module", tk)
            new_ckpt.update({k: v for k, v in tk.items() if k.startswith("text_encoder.")})
        if extra_ckpt_path is not None:
            ek = torch.load(extra_ckpt_path, map_location="cpu")
            new_ckpt.update(ek.get("module", ek))
        return self.load_state_dict(new_ckpt, strict=False)


class InternVideo2_CLIP(nn.Module):
    """internvideo2_clip.py:16-192: the InternVideo2-CLIP 1B / 6B recipes.  `config.model.vision_encoder.*`,
    `config.model.text_encoder.{use_flash_attn,transformer_width,llama_path,use_lora}` and `config.model.{temp,temp_min,
    freeze_vision,open_vision_clip_projector,freeze_text,open_text_projection,open_text_lora}` as in
    scripts/pretraining/clip/{1B,6B}/config.py.  text_encoder: an llama_modules.LLaMA to use instead of building one
    from config.model.text_encoder.  forward(image[B,T,C,H,W], text ids [B, L], idx) -> dict(loss_vtc=...).

    The tokenizer stays host code: `text` is the id tensor the reference's Tokenizer returns.  The text tower has no
    LoRA parameters (llama_modules), so open_text_lora unfreezes nothing; the recipes leave it off."""

    def __init__(self, config, tokenizer=None, is_pretrain=True, text_encoder=None, process_group=None):
        super().__init__()
        self.config = config
        self.tokenizer = tokenizer
        self.is_pretrain = is_pretrain
        m = _get(config, "model")
        self.vision_encoder = InternVideo2_CLIP_small.build_vision_encoder(self)
        self.text_encoder = text_encoder if text_encoder is not None else self.build_text_encoder()
        self.temp = nn.Parameter(torch.ones([]) * _get(m, "temp"))
        self.temp_min = _get(m, "temp_min")
        if _get(m, "freeze_vision", False):
            for name, p in self.vision_encoder.named_parameters():
                if not (_get(m, "open_vision_clip_projector", False) and name.startswith("clip_projector")):
                    p.requires_grad = False
        if _get(m, "freeze_text", False):
            for name, p in self.text_encoder.named_parameters():
                if not (_get(m, "open_text_projection", False) and name.startswith("text_projection")):
                    p.requires_grad = False
        self.clip_loss = VTC_VTM_Loss(False, process_group=process_group)

    def build_text_encoder(self):
        te = _get(_get(self.config, "model"), "text_encoder")
        return LLaMA(use_flash_attn=_get(te, "use_flash_attn", True), transformer_width=_get(te, "transformer_width"),
                     llama_path=_get(te, "llama_path"), use_lora=_get(te, "use_lora", True))

    def no_weight_decay(self):
        ret = {"temp"}
        ret.update({"vision_encoder." + k for k in self.vision_encoder.no_weight_decay()})
        ret.update({"text_encoder." + k for k, _ in self.text_encoder.named_parameters()})
        return ret

    clip_contrastive_temperature = InternVideo2_CLIP_small.clip_contrastive_temperature

    def encode_vision(self, image, test=False):
        """image [B,T,C,H,W] -> the tower's [B, clip_embed_dim] (:115-131), on tower_embeds' frozen-tower path."""
        return tower_embeds(self.vision_encoder, image)

    def encode_text(self, text):
        return self.text_encoder(text)

    forward = InternVideo2_CLIP_small.forward

    def load_checkpoint(self, vision_ckpt_path=None, text_ckpt_path=None, extra_ckpt_path=None):
        """:194-254: the vision side through remap_vision_checkpoint, the text side through remap_text_checkpoint, then
        the extra checkpoint's keys as they are; loaded with strict=False."""
        m = _get(self.config, "model")
        new_ckpt = {}
        if vision_ckpt_path is not None:
            ck = torch.load(vision_ckpt_path, map_location="cpu")
            new_ckpt.update(remap_vision_checkpoint(
                ck, self.vision_encoder, from_stage2=_get(m, "load_vision_ckpt_from_internvideo2_stage2", False),
                orig_t_size=_get(m, "vision_ckpt_t_size", 4)))
        if text_ckpt_path is not None:
            new_ckpt.update(remap_text_checkpoint(torch.load(text_ckpt_path, map_location="cpu")))
        if extra_ckpt_path is not None:
            ek = torch.load(extra_ckpt_path, map_location="cpu")
            new_ckpt.update(ek.get("module", ek))
        return self.load_state_dict(new_ckpt, strict=False)


def tower_embeds(enc, image):
    """The frozen-tower path of both wrappers: image [B,T,C,H,W] -> the vision tower's [B, clip_embed_dim].  While no
    parameter before the projector trains (the recipes' freeze_vision with open_vision_clip_projector), the blocks run
    without autograd (nothing saved) and only the attention-pooling projector is differentiated."""
    use_image = image.shape[1] == 1
    image = image.permute(0, 2, 1, 3, 4)
    trainable = any(p.requires_grad for n, p in enc.named_parameters() if not n.startswith("clip_projector"))
    if trainable and torch.is_grad_enabled():
        return enc(image, use_image=use_image)
    with torch.no_grad():
        h, B, n = enc.forward_tokens(image.contiguous(), use_image)
    return enc.fc_norm(enc.clip_projector(h.reshape(B, n, enc.embed_dim)))


def remap_text_checkpoint(ckpt):
    """Text-side key surgery of InternVideo2_CLIP.load_checkpoint (internvideo2_clip.py:231-241): unwrap DeepSpeed
    'module', keep `transformer.*` and `text_projection` under 'text_encoder.'.  LLaMA's load hook then maps a use_lora
    checkpoint's keys."""
    if "module" in ckpt:
        ckpt = ckpt["module"]
    return {"text_encoder." + k: v for k, v in ckpt.items() if k.startswith("transformer.") or k == "text_projection"}


def interpolate_pos_embed(checkpoint_model, model, orig_t_size=4, pos_name="vision_encoder.pos_embed"):
    """pos_embed.py:137-182 — linear interpolation over time, bicubic over space, cls token untouched."""
    if pos_name not in checkpoint_model:
        return
    pe = checkpoint_model[pos_name]
    C = pe.shape[-1]
    num_patches = model.patch_embed.num_patches
    extra = model.pos_embed.shape[-2] - num_patches
    new_t = model.T
    orig_size = int(((pe.shape[-2] - extra) // orig_t_size) ** 0.5)
    new_size = int((num_patches // new_t) ** 0.5)
    if orig_t_size != new_t:
        ext, tok = pe[:, :extra], pe[:, extra:]
        tok = tok.view(1, orig_t_size, -1, C).permute(0, 2, 3, 1).reshape(-1, C, orig_t_size)
        tok = torch.nn.functional.interpolate(tok, size=new_t, mode="linear")
        tok = tok.view(1, -1, C, new_t).permute(0, 3, 1, 2).reshape(1, -1, C)
        pe = torch.cat((ext, tok), dim=1)
        checkpoint_model[pos_name] = pe
    if orig_size != new_size:
        ext, tok = pe[:, :extra], pe[:, extra:]
        tok = tok.reshape(-1, new_t, orig_size, orig_size, C).reshape(-1, orig_size, orig_size, C).permute(0, 3, 1, 2)
        tok = torch.nn.functional.interpolate(tok, size=(new_size, new_size), mode="bicubic", align_corners=False)
        tok = tok.permute(0, 2, 3, 1).reshape(-1, new_t, new_size, new_size, C).flatten(1, 3)
        checkpoint_model[pos_name] = torch.cat((ext, tok), dim=1)


def remap_vision_checkpoint(ckpt, vision_encoder, from_stage2=False, orig_t_size=4):
    """Key surgery of InternVideo2_CLIP_small.load_checkpoint (:207-231): unwrap DeepSpeed 'module' / 'model', drop the
    stage-1 decoders and decoder position tables, prefix the tower's keys with 'vision_encoder.'; a stage-2
    checkpoint keeps its prefix and has its position table interpolated to this tower's frame count."""
    if "module" in ckpt:
        ckpt = ckpt["module"]
    elif "model" in ckpt:
        ckpt = ckpt["model"]
    out = {}
    if from_stage2:
        ckpt = dict(ckpt)
        interpolate_pos_embed(ckpt, vision_encoder, orig_t_size=orig_t_size)
        for k, v in ckpt.items():
            if not k.startswith("vision_encoder."):
                continue
            if "clip_decoder" in k or "final_clip_decoder" in k:
                continue
            if "clip_pos_embed" in k or "clip_img_pos_embed" in k or "img_pos_embed" in k:
                continue
            out[k] = v
        return out
    for k, v in ckpt.items():
        if k.startswith("clip_decoder.") or k.startswith("mae_decoder.") or k.startswith("final_clip_decoder."):
            continue
        if k in ("clip_pos_embed", "mae_pos_embed"):
            continue
        out["vision_encoder." + k] = v
    return out
