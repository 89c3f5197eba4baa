"""InternVideo-MM, InternVideo1's multimodal video-text model (InternVideo1/Pretrain/Multi-Modalities-Pretraining), on
the libivb200 kernels.  Forward only: the reference ships the architecture, the loader and a zero-shot demo, not a
training recipe.

Mirrors (constructors, attribute names, state_dict keys and order, init draws, forward contracts):
  InternVideo/clip_utils/utils/clip_vit_only_global.py:94-459   `Extractor`, `Transformer`, `VisionTransformer`,
                                                                 `vit_only_global_b16`, `vit_only_global_l14`
  InternVideo/clip_utils/model.py:86-328                        `VideoIntern`, `build_model`
  InternVideo/internvideo.py:17-21                              `load_model`
so that a released checkpoint loads with strict=True.

Vision tower.  A per-frame OpenAI-CLIP ViT: conv1 (ops.EmbedFn, im2col + wgmma GEMM) with the class embedding and the
position table, ln_pre (ivb_norm_fwd), whose bf16 output widened to fp32 is the residual stream, and the blocks as fused
LayerNorm blocks with QuickGELU (viclip.ResidualAttentionBlock) over the N*T frames' sequences of 1 + H*W tokens.  The
stream's row (n*T + t)*(1 + H*W) + l is token l of frame t of clip n.

Global extractor, at each backbone layer in return_list (tap j):
  - ivb_dpe_ln_fwd: the depthwise 3x3x3 position conv `dpe[j]` over (T, H, W) added to the patch tokens, then `ln_3`,
    in one kernel that reads the fp32 stream and writes bf16 keys' inputs (the cls rows: ln_3 alone);
  - one GEMM for k and v (in_proj rows C .. 3C, with bias) over all N*T*(1 + H*W) rows; the q GEMM on the N query rows
    after ln_1;
  - ivb_pool_attn_fwd: one query per clip over its T*(1 + H*W) keys, in the reference's (t, l) order;
  - out_proj as a GEMM with the residual add; ln_2 -> c_fc with the QuickGELU epilogue -> c_proj with the residual add.
Head: feats = (1 - sigmoid(balance)) * cls + sigmoid(balance) * mean_t(stream cls rows) (O(N*C) torch glue), then
visual_ln_post and the GEMM with visual_proj.

Text tower: ivb_token_embed_fwd, the causal fused blocks, ln_final on the EOT rows (text.argmax(-1)) and the GEMM with
text_projection.  masked_indices replaces the token rows it names by text_mask_embedding before the position add (torch
glue).  Tokenization is host code outside the library: encode_text takes token ids.

Refused, each with a message: a forward in training mode or of an input that requires a gradient (the extractor MLP's
Dropout(0.5) is live in training), an extractor attn_mask, a video whose T is not t_size in video mode, and weights
that would be downloaded (pretrained is a local checkpoint path or False).
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .modules import check_input, index_poison
from .viclip import QuickGELU, ResidualAttentionBlock, Transformer as _BlockStack, _load_local

bf16, f32 = torch.bfloat16, torch.float32

__all__ = ["Extractor", "Transformer", "VisionTransformer", "VideoIntern", "vit_only_global_b16",
           "vit_only_global_l14", "build_model", "load_model"]


def _refuse_training(module, *inputs):
    if module.training:
        raise ll._lib.IvbError(f"ivb200 {type(module).__name__} is forward only (no training recipe is built): call "
                               f".eval() first")
    if any(torch.is_tensor(t) and t.requires_grad for t in inputs):
        raise ll._lib.IvbError(f"ivb200 {type(module).__name__} is forward only: its input must not require a gradient")


class Extractor(nn.Module):
    """clip_vit_only_global.py:94-149: one learnable query per clip that cross-attends over the clip's ln_3-normed
    tokens, then an MLP, each with a residual add.  ln_3 runs inside ivb_dpe_ln_fwd (Transformer.forward)."""

    def __init__(self, d_model, n_head, attn_mask=None, mlp_factor=4.0, dropout=0.0, drop_path=0.0):
        super().__init__()
        if attn_mask is not None:
            raise NotImplementedError("ivb200 Extractor: attn_mask is not supported (the reference asserts it is None)")
        self.drop_path = nn.Identity()     # DropPath acts only in training, which is refused
        self.attn = nn.MultiheadAttention(d_model, n_head)
        self.ln_1 = nn.LayerNorm(d_model)
        d_mlp = round(mlp_factor * d_model)
        self.mlp = nn.Sequential(OrderedDict([
            ("c_fc", nn.Linear(d_model, d_mlp)),
            ("gelu", QuickGELU()),
            ("dropout", nn.Dropout(dropout)),
            ("c_proj", nn.Linear(d_mlp, d_model)),
        ]))
        self.ln_2 = nn.LayerNorm(d_model)
        self.ln_3 = nn.LayerNorm(d_model)
        self.attn_mask = attn_mask
        nn.init.xavier_uniform_(self.attn.in_proj_weight)
        nn.init.constant_(self.attn.out_proj.weight, 0.)
        nn.init.constant_(self.attn.out_proj.bias, 0.)
        nn.init.xavier_uniform_(self.mlp[0].weight)
        nn.init.constant_(self.mlp[-1].weight, 0.)
        nn.init.constant_(self.mlp[-1].bias, 0.)

    def forward_rows(self, x, keys, n):
        """x: the fp32 query stream [N, C]; keys: bf16 [N*n, C], ln_3 of each clip's n tokens -> fp32 [N, C]."""
        if self.attn_mask is not None:
            raise NotImplementedError("ivb200 Extractor: attn_mask is not supported")
        a = self.attn
        C, H = x.shape[1], a.num_heads
        d = C // H
        w, b = a.in_proj_weight, a.in_proj_bias
        kv = ll.gemm(keys, w[C:], bias=b[C:])                                   # bf16 [N*n, 2C]
        q = ll.gemm(ops.layernorm(x, self.ln_1.weight, self.ln_1.bias, self.ln_1.eps), w[:C], bias=b[:C])
        o, _ = ll.pool_attn_fwd(q, kv[:, :C], kv[:, C:], x.shape[0], n, H, d, d ** -0.5)
        x = ll.gemm(o, a.out_proj.weight, epi=ll.EPI_RESID, bias=a.out_proj.bias, aux=x)
        h = ll.gemm(ops.layernorm(x, self.ln_2.weight, self.ln_2.bias, self.ln_2.eps), self.mlp.c_fc.weight,
                    epi=ll.EPI_BIAS_GELU, flags=ll.FLAG_GELU_QUICK, bias=self.mlp.c_fc.bias)
        return ll.gemm(h, self.mlp.c_proj.weight, epi=ll.EPI_RESID, bias=self.mlp.c_proj.bias, aux=x)


class Transformer(nn.Module):
    """clip_vit_only_global.py:152-240: the backbone blocks, the position convs `dpe`, the extractors `dec`, the query
    `temporal_cls_token` and the `balance` of the two clip features."""

    def __init__(self, width, layers, heads, attn_mask=None, backbone_drop_path_rate=0., use_checkpoint=False,
                 checkpoint_num=[0], t_size=8, return_list=[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], n_layers=12,
                 n_dim=768, n_head=12, mlp_factor=4.0, drop_path_rate=0., mlp_dropout=[0.5] * 12, cls_dropout=0.5,
                 num_classes=400):
        super().__init__()
        if attn_mask is not None:
            raise NotImplementedError("ivb200 InternVideo-MM Transformer: the backbone takes no attn_mask")
        if n_layers != len(return_list):
            raise ValueError(f"ivb200 InternVideo-MM Transformer: n_layers {n_layers} != len(return_list) "
                             f"{len(return_list)}")
        if n_dim != width:
            raise NotImplementedError(f"ivb200 InternVideo-MM Transformer: n_dim {n_dim} must equal the backbone width "
                                      f"{width} (the extractor reads the backbone's tokens)")
        self.T = t_size
        self.return_list = return_list
        b_dpr = [x.item() for x in torch.linspace(0, backbone_drop_path_rate, layers)]
        self.resblocks = nn.ModuleList([ResidualAttentionBlock(width, heads, drop_path=b_dpr[i])
                                        for i in range(layers)])
        self.use_checkpoint = use_checkpoint
        self.checkpoint_num = checkpoint_num
        self.temporal_cls_token = nn.Parameter(torch.zeros(1, 1, n_dim))
        self.dpe = nn.ModuleList([nn.Conv3d(n_dim, n_dim, kernel_size=3, stride=1, padding=1, bias=True, groups=n_dim)
                                  for _ in range(n_layers)])
        for m in self.dpe:
            nn.init.constant_(m.bias, 0.)
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, n_layers)]
        self.dec = nn.ModuleList([Extractor(n_dim, n_head, mlp_factor=mlp_factor, dropout=mlp_dropout[i],
                                            drop_path=dpr[i]) for i in range(n_layers)])
        self.balance = nn.Parameter(torch.zeros((n_dim)))
        self.sigmoid = nn.Sigmoid()

    def forward_stream(self, h, N, T, Hg, Wg):
        """h: the fp32 stream [N*T*(1 + Hg*Wg), C] after ln_pre -> (clip features fp32 [N, C], the stream after the last
        block)."""
        L = 1 + Hg * Wg
        C = h.shape[1]
        cls = self.temporal_cls_token.reshape(1, C).float().expand(N, C).contiguous()
        j = -1
        for i, blk in enumerate(self.resblocks):
            h = blk.forward_stream(h, N * T, L)
            if i in self.return_list:
                j += 1
                dpe, dec = self.dpe[j], self.dec[j]
                keys = ll._dpe_ln_fwd(h, dpe.weight, dpe.bias, dec.ln_3.weight, dec.ln_3.bias, dec.ln_3.eps, N, T, Hg, Wg)
                cls = dec.forward_rows(cls, keys, T * L)
        weight = torch.sigmoid(self.balance.float())
        residual = h.reshape(N, T, L, C)[:, :, 0].mean(1)
        return (1 - weight) * cls + weight * residual, h

    def forward(self, x, mode="video", return_all_feats=False):
        """x: [L, N*T, C] in the reference's layout (fp32 or bf16, on the GPU)."""
        _refuse_training(self, x)
        L, NT, C = x.shape
        T = self.T if mode == "video" else 1
        Hg = Wg = int((L - 1) ** 0.5)
        if Hg * Wg != L - 1 or NT % T:
            raise ll._lib.IvbError(f"ivb200 InternVideo-MM Transformer: {L} tokens of {NT} frames are not clips of "
                                   f"{T} frames of a square grid")
        with torch.no_grad():
            h = x.float().permute(1, 0, 2).reshape(NT * L, C).contiguous()
            feats, h = self.forward_stream(h, NT // T, T, Hg, Wg)
        if return_all_feats:
            return feats, h.reshape(NT // T, T, L, C).permute(2, 0, 1, 3)
        return feats


class VisionTransformer(nn.Module):
    """clip_vit_only_global.py:243-286.  forward(x [N, 3, T, H, W], mode="video", return_all_feats=False) -> the clip
    features fp32 [N, C] (and with return_all_feats the stream after the last block in the reference's [L, N, T, C]
    layout).  mode "video": clips of t_size frames; any other mode: every frame is its own clip (T_down = 1).
    Parameters must be bf16 (model.bfloat16()), the input on the GPU, the module in eval mode."""

    def __init__(self, input_resolution, patch_size, width, layers, heads, output_dim, backbone_drop_path_rate=0.,
                 use_checkpoint=False, checkpoint_num=[0], t_size=8, return_list=[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11],
                 n_layers=12, n_dim=768, n_head=12, mlp_factor=4.0, drop_path_rate=0., mlp_dropout=[0.5] * 12,
                 cls_dropout=0.5, num_classes=400):
        super().__init__()
        self.input_resolution = input_resolution
        self.output_dim = output_dim
        self.conv1 = nn.Conv3d(3, width, (1, patch_size, patch_size), (1, patch_size, patch_size), (0, 0, 0),
                               bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = Transformer(
            width, layers, heads, backbone_drop_path_rate=backbone_drop_path_rate, use_checkpoint=use_checkpoint,
            checkpoint_num=checkpoint_num, t_size=t_size, return_list=return_list, n_layers=n_layers, n_dim=n_dim,
            n_head=n_head, mlp_factor=mlp_factor, drop_path_rate=drop_path_rate, mlp_dropout=mlp_dropout,
            cls_dropout=cls_dropout, num_classes=num_classes)

    def forward(self, x, mode="video", return_all_feats=False):
        _refuse_training(self, x)
        N, _, T, H, W = x.shape
        if mode == "video" and T != self.transformer.T:
            raise ll._lib.IvbError(f"ivb200 InternVideo-MM: the video has {T} frames, the model t_size "
                                   f"{self.transformer.T} (mode='video')")
        check_input(self, x, self.conv1.weight.dtype)
        p = self.conv1.weight.shape[-1]
        Hg, Wg = H // p, W // p
        L = 1 + Hg * Wg
        if L != self.positional_embedding.shape[0]:
            raise ll._lib.IvbError(f"ivb200 InternVideo-MM: a {H}x{W} input gives {L - 1} patches, the position table "
                                   f"has {self.positional_embedding.shape[0] - 1}")
        with torch.no_grad():
            frames = x.to(bf16).permute(0, 2, 1, 3, 4).reshape(N * T, 3, 1, H, W).contiguous()
            idx = torch.arange(L, device=x.device, dtype=torch.int32).repeat(N * T, 1)
            w = self.conv1.weight
            zero_bias = torch.zeros(w.shape[0], device=w.device, dtype=w.dtype)
            h = ops.EmbedFn.apply(frames, idx, w, zero_bias, self.class_embedding, self.positional_embedding, 1, p)
            h = ops.layernorm(h, self.ln_pre.weight, self.ln_pre.bias, self.ln_pre.eps).float()
            Tc = T if mode == "video" else 1
            feats, h = self.transformer.forward_stream(h, N * T // Tc, Tc, Hg, Wg)
        if return_all_feats:
            return feats, h.reshape(N * T // Tc, Tc, L, -1).permute(2, 0, 1, 3)
        return feats


def _vision_factory(resolution, patch, width, layers, heads, output_dim, pretrained, **kw):
    model = VisionTransformer(input_resolution=resolution, patch_size=patch, width=width, layers=layers, heads=heads,
                              output_dim=output_dim, **kw)
    if pretrained:
        # load_state_dict (:301-311): a tensor of another shape is skipped (<= 2 dims) or inflated in time (the 2D
        # patch embed: its centre frame)
        sd = _load_local(pretrained, "vit_only_global")
        own = model.state_dict()
        for k in list(sd):
            if k in own and sd[k].shape != own[k].shape:
                if own[k].ndim <= 2:
                    del sd[k]
                else:
                    w3 = torch.zeros(*sd[k].shape).unsqueeze(2).repeat(1, 1, own[k].shape[2], 1, 1)
                    w3[:, :, own[k].shape[2] // 2] = sd[k]
                    sd[k] = w3
        model.load_state_dict(sd, strict=False)
    return model.eval()


def vit_only_global_b16(pretrained=False, use_checkpoint=False, checkpoint_num=[0], t_size=16,
                        backbone_drop_path_rate=0., return_list=[8, 9, 10, 11], n_layers=4, n_dim=768, n_head=12,
                        mlp_factor=4.0, drop_path_rate=0., mlp_dropout=[0.5, 0.5, 0.5, 0.5], cls_dropout=0.5,
                        num_classes=400):
    """clip_vit_only_global.py:351-385 (no download: pretrained is a local CLIP ViT-B/16 checkpoint path or False)."""
    return _vision_factory(224, 16, 768, 12, 12, 512, pretrained, use_checkpoint=use_checkpoint,
                           checkpoint_num=checkpoint_num, t_size=t_size, backbone_drop_path_rate=backbone_drop_path_rate,
                           return_list=return_list, n_layers=n_layers, n_dim=n_dim, n_head=n_head,
                           mlp_factor=mlp_factor, drop_path_rate=drop_path_rate, mlp_dropout=mlp_dropout,
                           cls_dropout=cls_dropout, num_classes=num_classes)


def vit_only_global_l14(pretrained=False, use_checkpoint=False, checkpoint_num=[0], t_size=16,
                        backbone_drop_path_rate=0., return_list=[20, 21, 22, 23], n_layers=4, n_dim=1024, n_head=16,
                        mlp_factor=4.0, drop_path_rate=0., mlp_dropout=[0.5, 0.5, 0.5, 0.5], cls_dropout=0.5,
                        num_classes=400):
    """clip_vit_only_global.py:388-422 (no download: pretrained is a local CLIP ViT-L/14 checkpoint path or False)."""
    return _vision_factory(224, 14, 1024, 24, 16, 768, pretrained, use_checkpoint=use_checkpoint,
                           checkpoint_num=checkpoint_num, t_size=t_size, backbone_drop_path_rate=backbone_drop_path_rate,
                           return_list=return_list, n_layers=n_layers, n_dim=n_dim, n_head=n_head,
                           mlp_factor=mlp_factor, drop_path_rate=drop_path_rate, mlp_dropout=mlp_dropout,
                           cls_dropout=cls_dropout, num_classes=num_classes)


# the backbones VideoIntern builds by name, as the reference looks them up in its `utils` package
BACKBONES = {"vit_only_global_b16": vit_only_global_b16, "vit_only_global_l14": vit_only_global_l14}


class VideoIntern(nn.Module):
    """model.py:86-245.  encode_video(video [N, 3, T, H, W], return_all_feats=False, masked_indices=None, mode="video")
    -> bf16 [N, embed_dim]; encode_text(token ids [B, context_length], masked_indices=None, return_all_feats=False) ->
    bf16 [B, embed_dim].  Forward only: eval mode, bf16 parameters (model.bfloat16()), inputs on the GPU.  As in the
    reference, positional_embedding, text_projection and text_mask_embedding are drawn by initialize_parameters, and
    the model has no forward() of its own."""

    def __init__(self, embed_dim, vision_width, context_length, vocab_size, transformer_width, transformer_heads,
                 transformer_layers, n_layers=4, n_dim=768, n_head=12, drop_path_rate=0.0,
                 mlp_dropout=[0.5, 0.5, 0.5, 0.5], cls_dropout=0.5, t_size=8, use_image_attnmap=True,
                 backbone='vit_2plus1d_dw_bias_b16', return_list=[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11],
                 use_checkpoint=False, checkpoint_num=[0]):
        super().__init__()
        if backbone not in BACKBONES:
            raise NotImplementedError(f"ivb200 VideoIntern: backbone {backbone!r} (built: {sorted(BACKBONES)})")
        self.vision_width = n_dim
        self.context_length = context_length
        self.visual = BACKBONES[backbone](
            pretrained=False, t_size=t_size, mlp_dropout=mlp_dropout, cls_dropout=cls_dropout, n_dim=n_dim,
            n_head=n_head, return_list=return_list, drop_path_rate=drop_path_rate,
            backbone_drop_path_rate=drop_path_rate, use_checkpoint=use_checkpoint, checkpoint_num=checkpoint_num)
        self.visual_ln_post = nn.LayerNorm(n_dim)
        scale = n_dim ** -0.5
        self.visual_proj = nn.Parameter(scale * torch.randn(n_dim, embed_dim))
        self.return_qk = use_image_attnmap
        self.return_num = n_layers
        self.transformer = _BlockStack(transformer_width, transformer_layers, transformer_heads, causal=True)
        self.vocab_size = vocab_size
        self.token_embedding = nn.Embedding(vocab_size, transformer_width)
        self.positional_embedding = nn.Parameter(torch.empty(self.context_length, transformer_width))
        self.ln_final = nn.LayerNorm(transformer_width)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]) * np.log(1 / 0.07))
        self.embed_dim = embed_dim
        self.text_mask_embedding = nn.Parameter(torch.empty(1, 1, transformer_width))
        self.initialize_parameters()

    def initialize_parameters(self):
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.positional_embedding, std=0.01)
        nn.init.normal_(self.text_mask_embedding, std=0.02)
        proj_std = (self.transformer.width ** -0.5) * ((2 * self.transformer.layers) ** -0.5)
        attn_std = self.transformer.width ** -0.5
        fc_std = (2 * self.transformer.width) ** -0.5
        for block in self.transformer.resblocks:
            nn.init.normal_(block.attn.in_proj_weight, std=attn_std)
            nn.init.normal_(block.attn.out_proj.weight, std=proj_std)
            nn.init.normal_(block.mlp.c_fc.weight, std=fc_std)
            nn.init.normal_(block.mlp.c_proj.weight, std=proj_std)
        nn.init.normal_(self.text_projection, std=self.transformer.width ** -0.5)
        nn.init.constant_(self.visual_ln_post.weight, 1.0)
        nn.init.constant_(self.visual_ln_post.bias, 0.0)

    def build_attention_mask(self):
        mask = torch.empty(self.context_length, self.context_length)
        mask.fill_(float("-inf"))
        mask.triu_(1)
        return mask

    @property
    def dtype(self):
        return self.visual.conv1.weight.dtype

    def encode_video(self, video, return_all_feats=False, masked_indices=None, mode="video"):
        """video [N, 3, T, H, W] -> bf16 [N, embed_dim]; with return_all_feats also the backbone stream [L, N, T, C]
        (fp32).  masked_indices is accepted and unused, as in the reference."""
        _refuse_training(self, video)
        out = self.visual(video, return_all_feats=return_all_feats, mode=mode)
        x, feats = out if return_all_feats else (out, None)
        with torch.no_grad():
            ln = self.visual_ln_post
            x = ops.linear(ops.layernorm(x, ln.weight, ln.bias, ln.eps), self.visual_proj, w_t=True)
        return (x, feats) if return_all_feats else x

    def encode_text(self, text, masked_indices=None, return_all_feats=False):
        """token ids [B, context_length] (EOT: the largest id of each row) -> bf16 [B, embed_dim]; with
        return_all_feats also ln_final of every token, bf16 [B, context_length, width].  masked_indices: any index of
        a [B, context_length] tensor (a bool mask, or index tensors); those token rows become text_mask_embedding.  An
        id outside [0, vocab_size) makes the output NaN (a device flag, no host read)."""
        _refuse_training(self, text)
        check_input(self, text, self.token_embedding.weight.dtype)
        B, L = text.shape
        if L != self.context_length:
            raise ll._lib.IvbError(f"ivb200 VideoIntern.encode_text: sequence length {L} != context_length "
                                   f"{self.context_length}")
        with torch.no_grad():
            if masked_indices is None:
                h, err = ops.TokenEmbedFn.apply(text.long(), self.token_embedding.weight, self.positional_embedding)
            else:
                # the token rows through the same kernel (an out-of-range id sets the flag, as above) with a zero
                # position table, the masked rows replaced, then the position add
                D = self.token_embedding.weight.shape[1]
                zero = torch.zeros((L, D), device=text.device, dtype=bf16)
                h, err = ll._token_embed_fwd(text.long().contiguous(), self.token_embedding.weight, zero)
                h = h.reshape(B, L, D)
                h[masked_indices] = self.text_mask_embedding.reshape(-1).float()
                h = (h + self.positional_embedding.float()).reshape(B * L, D)
            for blk in self.transformer.resblocks:
                h = blk.forward_stream(h, B, L)
            ln = self.ln_final
            rows = h.reshape(B, L, -1)[torch.arange(B, device=h.device), text.argmax(dim=-1)]
            feats = ops.linear(ops.layernorm(rows, ln.weight, ln.bias, ln.eps), self.text_projection, w_t=True)
            feats = feats + index_poison(err).to(feats.dtype)
            if return_all_feats:
                every = ops.layernorm(h, ln.weight, ln.bias, ln.eps).reshape(B, L, -1)
                return feats, every + index_poison(err).to(every.dtype)
        return feats


def build_model(state_dict: dict, n_layers=4, n_dim=768, n_head=12, mlp_factor=4.0, drop_path_rate=0.0,
                mlp_dropout=[0.5, 0.5, 0.5, 0.5], cls_dropout=0.5, t_size=8, spatial_size=14, use_t_conv=True,
                use_image_attnmap=True, use_t_pos_embed=True, no_pretrain=False, init_zero=True, use_checkpoint=False,
                checkpoint_num=[0]):
    """model.py:248-329: the configuration inferred from the state dict's shapes, then the weights loaded.  Returns the
    fp32 model in eval mode (call .bfloat16().cuda() to run it)."""
    embed_dim = state_dict["text_projection"].shape[1]
    context_length = state_dict["positional_embedding"].shape[0]
    vocab_size = state_dict["token_embedding.weight"].shape[0]
    transformer_width = state_dict["ln_final.weight"].shape[0]
    transformer_heads = transformer_width // 64
    transformer_layers = len(set(k.split(".")[2] for k in state_dict if k.startswith("transformer.resblocks")))
    vision_width = state_dict["visual_proj"].shape[0]
    n_dim = vision_width
    if vision_width == 768:
        backbone, n_head, return_list = "vit_only_global_b16", 12, [8, 9, 10, 11]
    elif vision_width == 1024:
        backbone, n_head, return_list = "vit_only_global_l14", 16, [20, 21, 22, 23]
    else:
        raise NotImplementedError(f"ivb200 build_model: vision width {vision_width} (built: 768, 1024)")
    model = VideoIntern(embed_dim, vision_width, context_length, vocab_size, transformer_width, transformer_heads,
                        transformer_layers, n_layers=n_layers, n_dim=n_dim, n_head=n_head,
                        drop_path_rate=drop_path_rate, mlp_dropout=mlp_dropout, cls_dropout=cls_dropout, t_size=t_size,
                        use_image_attnmap=use_image_attnmap, backbone=backbone, return_list=return_list,
                        use_checkpoint=use_checkpoint, checkpoint_num=checkpoint_num)
    # The reference loads with strict=False.  Its modules' keys are this model's keys one for one (the checkpoint is a
    # VideoIntern state_dict), so nothing is left to skip; strict=True turns a checkpoint of another configuration into
    # an error instead of a model with some weights left at their random init.
    model.load_state_dict(state_dict, strict=True)
    return model.eval()


def load_model(path):
    """internvideo.py:17-21: the `clip.`-prefixed entries of the checkpoint's state_dict, built by build_model."""
    state = torch.load(path, map_location="cpu")["state_dict"]
    state = {k[len("clip."):]: v for k, v in state.items() if k.startswith("clip.")}
    return build_model(state_dict=state)
