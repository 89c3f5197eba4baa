"""ViCLIP, InternVideo1's video-text contrastive model (InternVideo1/Pretrain/ViCLIP), on the libivb200 kernels.

Mirrors (constructors, attribute names, state_dict keys and order, init draws, forward contracts):
  models/backbones/clip/clip_vision.py:28-177, 256-303   `ResidualAttentionBlock`, `Transformer`, `VisionTransformer`,
                                                          `clip_joint_b16`, `clip_joint_l14`
  models/backbones/clip/clip_text.py:25-178, 181-255      `CLIP_TEXT`, `clip_text_b16`, `clip_text_l14`
  models/viclip.py:10-207                                 `ViCLIP`
so that a released ViCLIP checkpoint loads with strict=True.

The blocks are OpenAI-CLIP blocks: pre-norm LayerNorm (eps 1e-5), nn.MultiheadAttention with its full qkv bias, and an
MLP whose activation is QuickGELU, x * sigmoid(1.702 x).  Each runs as one fused LayerNorm block (ops.BlockFn /
ops.block_forward with BlockSpec(layernorm=True, gelu_quick=True)): QuickGELU and its derivative are computed in the fc1
and dh GEMM epilogues (IVB_FLAG_GELU_QUICK).  The text tower's blocks add causal=True.

The vision front end:
  - the kept patches are embedded by ops.EmbedFn (an im2col + wgmma GEMM over the kept tokens only).  The reference
    orders the patch tokens `(n t)`, patch-major; the library's patch index is `(t n)`, frame-major.  Each kept token's
    index row entry names its `(t n)` patch, and the rows stay in the reference's order, so the token order of every
    output (return_embed included) is the reference's.  EmbedFn gathers by index and accepts any order;
  - the position table (cls row, then patch s of frame t: positional_embedding[1+s] + temporal_positional_embedding[t],
    or the temporal mean for a single frame) is O(T*L*D) torch glue built each call, so its gradient reaches all three
    parameters;
  - masking_prob draws the reference's mask on the host (torch.rand_like on a CPU tensor, mask_tokens :121-135), so a
    torch seed gives the reference's kept tokens bit for bit; the index rows are then copied to the device;
  - ln_pre's output is the blocks' fp32 residual stream.  The library's LayerNorm writes bf16 rows (ops.layernorm), so
    the stream is that bf16 row widened to fp32: one bf16 rounding of the block input, no new kernel path.

DropPath: the reference runs its blocks on the [N, B, D] layout, so timm's DropPath draws one factor per TOKEN
POSITION, shared by every clip of the batch (not one per clip).  The port keeps that draw and applies it as the
residual epilogues' per-row factors.  The library's DropPath plans skip the attention work of whole clips, which this
draw never drops, so the ViCLIP blocks run without plans.

Refused: dropout > 0, kernel_size other than 1 (weight inflation is out of scope), encoder names other than vit_b16 /
vit_l14, pretrained weights that would be downloaded (pass a local path or False), and string captions (tokenization
stays host code: encode_text takes token ids).
"""
from __future__ import annotations

import os
from collections import OrderedDict

import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .clip_modules import _get
from .contrastive import VTC_VTM_Loss
from .modules import Fp8Block, block_attn_fp8, block_precision, check_input, index_poison

bf16, f32 = torch.bfloat16, torch.float32


class QuickGELU(nn.Module):
    """clip_vision.py:28-30 (the fused block computes it in the fc1 epilogue; this form is for standalone use)."""

    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


class _InProj:
    """The `.weight` of nn.MultiheadAttention's packed qkv projection, read live (Fp8InferenceWeights re-reads it)."""

    def __init__(self, attn):
        self.attn = attn

    @property
    def weight(self):
        return self.attn.in_proj_weight


class ResidualAttentionBlock(Fp8Block, nn.Module):
    """clip_vision.py:33-61 (clip_text.py:38-59 without drop_path is the same block): x + attn(ln_1(x)), then
    x + mlp(ln_2(x)), mlp = c_fc -> QuickGELU -> c_proj.  `attn` is the nn.MultiheadAttention parameter container
    (in_proj_weight / in_proj_bias / out_proj); the block runs fused.  causal: the text tower's -inf upper triangle
    (its attn_mask).  drop_path: the rate of this block's two DropPath draws (VisionTransformer draws them)."""

    def __init__(self, d_model, n_head, drop_path=0.0, attn_mask=None, dropout=0.0, causal=False):
        super().__init__()
        if dropout:
            raise NotImplementedError("ivb200 ResidualAttentionBlock: dropout must be 0 (ViCLIP's recipes use 0)")
        if d_model % n_head:
            raise NotImplementedError(f"ivb200 ResidualAttentionBlock: {n_head} heads do not split width {d_model}")
        self.drop_prob = float(drop_path)
        self.attn = nn.MultiheadAttention(d_model, n_head, dropout=dropout)
        self.ln_1 = nn.LayerNorm(d_model)
        self.mlp = nn.Sequential(OrderedDict([
            ("c_fc", nn.Linear(d_model, d_model * 4)),
            ("gelu", QuickGELU()),
            ("c_proj", nn.Linear(d_model * 4, d_model)),
        ]))
        self.ln_2 = nn.LayerNorm(d_model)
        self.causal = bool(causal)
        self.checkpoint = False       # set by the tower from its checkpoint_num

    def _spec(self, B, n, training=False):
        return ops.BlockSpec(B, n, self.attn.num_heads, layernorm=True, gelu_quick=True, eps1=self.ln_1.eps,
                             eps2=self.ln_2.eps, checkpoint=self.checkpoint, causal=self.causal,
                             precision=block_precision(self, training),
                             attn_fp8=block_attn_fp8(self) and not self.causal)

    def _fp8_linears(self):
        return (_InProj(self.attn), self.attn.out_proj, self.mlp.c_fc, self.mlp.c_proj)

    def _param_tuple(self):
        a = self.attn
        return ops.BlockParams(n1w=self.ln_1.weight, n1b=self.ln_1.bias, qkvw=a.in_proj_weight, qkvb=a.in_proj_bias,
                               qnw=None, knw=None, projw=a.out_proj.weight, projb=a.out_proj.bias, g1=None,
                               n2w=self.ln_2.weight, n2b=self.ln_2.bias, fc1w=self.mlp.c_fc.weight,
                               fc1b=self.mlp.c_fc.bias, fc2w=self.mlp.c_proj.weight, fc2b=self.mlp.c_proj.bias, g2=None)

    def forward_stream(self, x2d, B, n, rowscale=(None, None)):
        """fp32 residual stream [B*n, D] -> same.  Differentiated (ops.BlockFn) when grad mode is on and the stream or a
        parameter needs a gradient; otherwise the no-grad block forward.  rowscale: the two branches' DropPath factors,
        fp32 [B*n] or None."""
        if torch.is_grad_enabled() and (x2d.requires_grad or any(p.requires_grad for p in self.parameters())):
            return ops.BlockFn.apply(x2d, self._spec(B, n, training=True), rowscale[0], rowscale[1],
                                     *self._param_tuple())
        with torch.no_grad():
            out, _ = ops.block_forward(x2d, self._spec(B, n), self._param_tuple(), rowscale[0], rowscale[1],
                                       save=False)
        return out

    def forward(self, x):
        """x [N, B, D] (the reference's layout) -> same."""
        N, B, D = x.shape
        h = x.permute(1, 0, 2).reshape(B * N, D).float().contiguous()
        return self.forward_stream(h, B, N).reshape(B, N, D).permute(1, 0, 2).to(x.dtype)


class Transformer(nn.Module):
    """clip_vision.py:64-80 / clip_text.py:62-78: `resblocks`, DropPath rates linspace(0, drop_path, layers).
    checkpointed: how many leading blocks keep only their input and recompute their forward in the backward."""

    def __init__(self, width, layers, heads, drop_path=0.0, checkpoint_num=0, dropout=0.0, causal=False,
                 checkpointed=None):
        super().__init__()
        dpr = [x.item() for x in torch.linspace(0, drop_path, layers)]
        self.width, self.layers = width, layers
        self.resblocks = nn.ModuleList([ResidualAttentionBlock(width, heads, drop_path=dpr[i], dropout=dropout,
                                                               causal=causal) for i in range(layers)])
        self.checkpoint_num = checkpoint_num
        for i, blk in enumerate(self.resblocks):
            blk.checkpoint = i < (checkpoint_num if checkpointed is None else checkpointed)


def _load_local(path, what):
    if path is True or (isinstance(path, str) and not os.path.isfile(path)):
        raise ValueError(f"ivb200 {what}: pretrained must be a local checkpoint path or False (nothing is downloaded), "
                         f"got {path!r}")
    return torch.load(path, map_location="cpu")


class VisionTransformer(nn.Module):
    """clip_vision.py:83-177.  forward(x [B, 3, T, H, W], masking_prob=0.0, return_embed=False) -> [B, output_dim] (the
    ln_post of the cls token times proj), or with return_embed the ln_post of every token, [B, n, width], in the
    reference's token order.  Parameters must be bf16 (model.bfloat16()) and the input on the GPU.

    drop_path_factors (port only): fp32 [2 * layers, n], the DropPath factor of every token position of each block
    branch (rows 2i, 2i+1: block i's attention and MLP branch), used instead of a fresh draw."""

    def __init__(self, input_resolution, patch_size, width, layers, heads, output_dim=None, kernel_size=1,
                 num_frames=8, drop_path=0, checkpoint_num=0, dropout=0.0, temp_embed=True):
        super().__init__()
        if kernel_size != 1:
            raise NotImplementedError("ivb200 VisionTransformer: kernel_size must be 1 (ViCLIP's recipe; the "
                                      "temporal weight inflation of kernel_size > 1 is not built)")
        if dropout:
            raise NotImplementedError("ivb200 VisionTransformer: dropout must be 0")
        self.output_dim = output_dim
        self.patch_size = patch_size
        self.conv1 = nn.Conv3d(3, width, (kernel_size, patch_size, patch_size), (kernel_size, patch_size, patch_size),
                               (0, 0, 0), bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        if temp_embed:
            self.temporal_positional_embedding = nn.Parameter(torch.zeros(1, num_frames, width))
        self.transformer = Transformer(width, layers, heads, drop_path=drop_path, checkpoint_num=checkpoint_num,
                                       dropout=dropout)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(torch.empty(width, output_dim)) if output_dim is not None else None
        self.dropout = nn.Dropout(dropout)

    def get_num_layers(self):
        return len(self.transformer.resblocks)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"positional_embedding", "class_embedding", "temporal_positional_embedding"}

    @staticmethod
    def mask_tokens(B, L, masking_prob):
        """The kept positions of mask_tokens (:121-135) over the B clips' L patch tokens: int64 [B, L - int(p L)],
        ascending, drawn on the host exactly as the reference draws them (the same torch RNG calls)."""
        Lm = int(masking_prob * L)
        masked_indices = torch.zeros(B, L)
        indices = torch.argsort(torch.rand_like(masked_indices), dim=-1)[:, :Lm]
        batch_indices = torch.arange(masked_indices.shape[0]).unsqueeze(-1).expand_as(indices)
        masked_indices[batch_indices, indices] = 1
        return (~masked_indices.bool()).nonzero()[:, 1].reshape(B, L - Lm)

    @staticmethod
    def token_index(B, T, L, masking_prob=0.0):
        """int32 [B, 1 + kept] host index rows for ops.EmbedFn: column 0 the cls slot (0), then each kept token, in the
        reference's `(n t)` order, as 1 + its library `(t n)` patch index."""
        kept = VisionTransformer.mask_tokens(B, T * L, masking_prob) if masking_prob > 0.0 else \
            torch.arange(T * L).expand(B, T * L)
        s, t = kept // T, kept % T
        return torch.cat([torch.zeros(B, 1, dtype=torch.int64), 1 + t * L + s], 1).to(torch.int32)

    def _pos_table(self, T, L):
        """[1 + T*L, width]: the cls row, then patch s of frame t at row 1 + t*L + s (:140-154)."""
        pe = self.positional_embedding
        if hasattr(self, "temporal_positional_embedding"):
            tpe = self.temporal_positional_embedding
            tpe = tpe.mean(1) if T == 1 else tpe.reshape(-1, pe.shape[-1])
            patches = (pe[1:].unsqueeze(0) + tpe.reshape(-1, 1, pe.shape[-1])).reshape(T * L, -1)
        else:
            patches = pe[1:].repeat(T, 1)
        return torch.cat([pe[:1], patches], 0)

    def _drop_path_rows(self, B, n, device, factors=None):
        """The DropPath factors of every block branch as per-row epilogue factors: a list of (rs1, rs2) fp32 [B*n] or
        None per block.  The reference's draw (timm DropPath on [N, B, D]): Bernoulli(keep) / keep per token position,
        branch by branch in block order, in training only."""
        blocks = self.transformer.resblocks
        if factors is not None:
            f = factors.to(device=device, dtype=f32)
            return [(f[2 * i].repeat(B).contiguous(), f[2 * i + 1].repeat(B).contiguous()) for i in range(len(blocks))]
        out = []
        for blk in blocks:
            if not self.training or blk.drop_prob == 0.0:
                out.append((None, None))
                continue
            keep = 1.0 - blk.drop_prob
            out.append(tuple((torch.empty(n, device=device, dtype=f32).bernoulli_(keep) / keep).repeat(B)
                             for _ in range(2)))
        return out

    def forward_tokens(self, x, masking_prob=0.0, drop_path_factors=None):
        """-> (fp32 stream [B*n, width] after the last block, B, n)."""
        check_input(self, x, self.conv1.weight.dtype)
        B, _, T, H, W = x.shape
        p = self.patch_size
        L = (H // p) * (W // p)
        idx = self.token_index(B, T, L, masking_prob).to(x.device, non_blocking=True)
        w = self.conv1.weight
        zero_bias = torch.zeros(w.shape[0], device=w.device, dtype=w.dtype)
        table = self._pos_table(T, L).to(bf16)
        h = ops.EmbedFn.apply(x.to(bf16).contiguous(), idx, w, zero_bias, self.class_embedding, table, 1, p)
        n = idx.shape[1]
        h = ops.layernorm(h, self.ln_pre.weight, self.ln_pre.bias, self.ln_pre.eps).float()
        for blk, rs in zip(self.transformer.resblocks, self._drop_path_rows(B, n, h.device, drop_path_factors)):
            h = blk.forward_stream(h, B, n, rs)
        return h, B, n

    def forward(self, x, masking_prob=0.0, return_embed=False, drop_path_factors=None):
        h, B, n = self.forward_tokens(x, masking_prob, drop_path_factors)
        D = h.shape[1]
        ln = self.ln_post
        if return_embed or self.proj is None:
            return ops.layernorm(h, ln.weight, ln.bias, ln.eps).reshape(B, n, D)
        cls = ops.layernorm(h.reshape(B, n, D)[:, 0], ln.weight, ln.bias, ln.eps)
        return ops.linear(cls, self.proj, w_t=True)


def _vision_factory(width, layers, heads, output_dim, patch_size, pretrained, input_resolution, kernel_size,
                    center, num_frames, drop_path, checkpoint_num, dropout):
    model = VisionTransformer(input_resolution=input_resolution, patch_size=patch_size, width=width, layers=layers,
                              heads=heads, output_dim=output_dim, kernel_size=kernel_size, num_frames=num_frames,
                              drop_path=drop_path, checkpoint_num=checkpoint_num, dropout=dropout)
    if pretrained:
        sd = _load_local(pretrained, "clip_joint")
        # load_state_dict (:198-233) at kernel_size 1: a 2D patch-embed weight gains its time axis; other shape
        # mismatches of 1D / 2D tensors are skipped, and a position table of another grid is refused, as there
        own = model.state_dict()
        for k in list(sd):
            if k in own and sd[k].shape != own[k].shape:
                if own[k].ndim <= 2:
                    del sd[k]
                elif sd[k].ndim == own[k].ndim - 1:
                    sd[k] = sd[k].unsqueeze(2)
        if sd["positional_embedding"].shape != own["positional_embedding"].shape:
            raise ValueError("clip_joint: the checkpoint's position table is for another input resolution")
        model.load_state_dict(sd, strict=False)
    return model.eval()


def clip_joint_b16(pretrained=False, input_resolution=224, kernel_size=1, center=True, num_frames=8, drop_path=0.0,
                   checkpoint_num=0, dropout=0.0):
    """clip_vision.py:236-259 (no download: pretrained is a local path or False)."""
    return _vision_factory(768, 12, 12, 512, 16, pretrained, input_resolution, kernel_size, center, num_frames,
                           drop_path, checkpoint_num, dropout)


def clip_joint_l14(pretrained=False, input_resolution=224, kernel_size=1, center=True, num_frames=8, drop_path=0.0,
                   checkpoint_num=0, dropout=0.0):
    """clip_vision.py:262-285 (no download: pretrained is a local path or False)."""
    return _vision_factory(1024, 24, 16, 768, 14, pretrained, input_resolution, kernel_size, center, num_frames,
                           drop_path, checkpoint_num, dropout)


class CLIP_TEXT(nn.Module):
    """clip_text.py:81-178.  forward(text int [B, context_length], return_embed=False) -> [B, embed_dim]: the ln_final
    of each caption's EOT token (the largest id of its row) times text_projection; with return_embed the pair
    (every token times text_projection [B, L, embed_dim], that pooled output).  Causal blocks.  As in the reference,
    positional_embedding and text_projection are allocated uninitialised (they come from the checkpoint).  Frozen
    (requires_grad False, ViCLIP's freeze_text) the tower runs its no-grad forward.  An id outside [0, vocab_size)
    makes the output NaN (a device flag, no host read).  Parameters must be bf16 and the ids on the GPU; tokenization
    (`tokenize`) is host code that is not built here."""

    def __init__(self, embed_dim, context_length, vocab_size, transformer_width, transformer_heads, transformer_layers,
                 checkpoint_num):
        super().__init__()
        self.context_length = context_length
        self._tokenizer = None
        # checkpoint_sequential(resblocks, segments) checkpoints every segment but the last (clip_text.py:72-76)
        segments = min(checkpoint_num, transformer_layers)
        checkpointed = (transformer_layers // segments) * (segments - 1) if segments > 0 else 0
        self.transformer = Transformer(transformer_width, transformer_layers, transformer_heads, causal=True,
                                       checkpoint_num=checkpoint_num, checkpointed=checkpointed)
        self.vocab_size = vocab_size
        self.token_embedding = nn.Embedding(vocab_size, transformer_width)
        self.positional_embedding = nn.Parameter(torch.empty(self.context_length, transformer_width))
        self.ln_final = nn.LayerNorm(transformer_width)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, embed_dim))

    def no_weight_decay(self):
        return {"token_embedding", "positional_embedding"}

    def tokenize(self, texts, context_length=77, truncate=True):
        raise NotImplementedError("ivb200 CLIP_TEXT: tokenization is host code outside the library; pass token ids")

    def forward_tokens(self, text):
        """-> (fp32 stream [B*L, width] after the last block, B, L, int32[1] bad-id flag)."""
        B, L = text.shape
        if L != self.context_length:
            raise ll._lib.IvbError(f"ivb200 CLIP_TEXT: sequence length {L} != context_length {self.context_length}")
        check_input(self, text, self.token_embedding.weight.dtype)
        h, err = ops.TokenEmbedFn.apply(text.long(), self.token_embedding.weight, self.positional_embedding)
        for blk in self.transformer.resblocks:
            h = blk.forward_stream(h, B, L)
        return h, B, L, err

    def forward(self, text, return_embed=False):
        h, B, L, err = self.forward_tokens(text)
        ln = self.ln_final
        # EOT pooling: LayerNorm is per row, so normalising the B pooled rows only is the reference's arithmetic
        rows = h.reshape(B, L, -1)[torch.arange(B, device=h.device), text.argmax(dim=-1)]
        pooled = ops.linear(ops.layernorm(rows, ln.weight, ln.bias, ln.eps), self.text_projection, w_t=True)
        pooled = pooled + index_poison(err)
        if not return_embed:
            return pooled
        every = ops.linear(ops.layernorm(h, ln.weight, ln.bias, ln.eps), self.text_projection, w_t=True)
        return every.reshape(B, L, -1) + index_poison(err), pooled


def _text_factory(embed_dim, context_length, vocab_size, width, heads, layers, checkpoint_num, pretrained):
    model = CLIP_TEXT(embed_dim, context_length, vocab_size, width, heads, layers, checkpoint_num)
    if pretrained:
        sd = _load_local(pretrained, "clip_text")
        pe = sd["positional_embedding"]
        if context_length < pe.shape[0]:           # clip_text.py:207-217
            sd["positional_embedding"] = pe[:context_length]
        elif context_length > pe.shape[0]:
            sd["positional_embedding"] = torch.nn.functional.pad(pe, (0, 0, 0, context_length - pe.shape[0]))
        model.load_state_dict(sd, strict=False)
    return model.eval()


def clip_text_b16(embed_dim=512, context_length=77, vocab_size=49408, transformer_width=512, transformer_heads=8,
                  transformer_layers=12, checkpoint_num=0, pretrained=False):
    """clip_text.py:181-222 (no download: pretrained is a local path or False)."""
    return _text_factory(embed_dim, context_length, vocab_size, transformer_width, transformer_heads,
                         transformer_layers, checkpoint_num, pretrained)


def clip_text_l14(embed_dim=768, context_length=77, vocab_size=49408, transformer_width=768, transformer_heads=12,
                  transformer_layers=12, checkpoint_num=0, pretrained=False):
    """clip_text.py:225-258 (no download: pretrained is a local path or False)."""
    return _text_factory(embed_dim, context_length, vocab_size, transformer_width, transformer_heads,
                         transformer_layers, checkpoint_num, pretrained)


_VISION = {"vit_b16": clip_joint_b16, "vit_l14": clip_joint_l14}
_TEXT = {"vit_b16": clip_text_b16, "vit_l14": clip_text_l14}


def _local_or_false(p):
    """A config's `pretrained` as the factories take it: a local file path, else False (the recipe's text value
    "bert-base-uncased" names no file; weights then come from a ViCLIP checkpoint)."""
    return p if isinstance(p, str) and os.path.isfile(p) else False


class ViCLIP(nn.Module):
    """viclip.py:10-207.  forward(image [B,T,C,H,W], text, raw_text, idx) -> dict(loss_vtc=...): the vision-text
    contrastive loss (contrastive.VTC_VTM_Loss with its packed all-gather; ViCLIP's criterions.py vtc_loss, get_sim
    and get_mask are InternVideo2's statement for statement).  raw_text: the captions' token ids [B, max_txt_l] (the
    reference tokenizes strings there; here tokenization is host code: a callable `tokenizer(texts, context_length=)`
    is used for strings when given)."""

    def __init__(self, config, tokenizer=None, is_pretrain=True):
        super().__init__()
        self.config = config
        self.tokenizer = tokenizer
        self.is_pretrain = is_pretrain
        m = _get(config, "model")
        self.vision_width = _get(_get(m, "vision_encoder"), "d_model")
        self.text_width = _get(_get(m, "text_encoder"), "d_model")
        self.embed_dim = _get(m, "embed_dim")
        self.vision_encoder = self.build_vision_encoder()
        self.text_encoder = self.build_text_encoder()
        self.temp = nn.Parameter(torch.ones([]) * _get(m, "temp"))
        self.temp_min = _get(m, "temp_min")
        self.clip_loss = VTC_VTM_Loss(False)
        if _get(m, "freeze_text"):
            self.freeze_text()

    def freeze_text(self):
        for p in self.text_encoder.parameters():
            p.requires_grad = False

    def no_weight_decay(self):
        ret = {"temp"}
        ret.update({"vision_encoder." + k for k in self.vision_encoder.no_weight_decay()})
        ret.update({"text_encoder." + k for k in self.text_encoder.no_weight_decay()})
        return ret

    def forward(self, image, text, raw_text, idx, log_generation=None, return_sims=False):
        if return_sims:
            raise NotImplementedError("ivb200 ViCLIP: return_sims belongs to retrieval, which is not built")
        self.clip_contrastive_temperature()
        vision_embeds = self.encode_vision(image)
        text_embeds = self.encode_text(raw_text)
        loss_vtc = self.clip_loss.vtc_loss(vision_embeds, text_embeds, idx, self.temp, all_gather=True)
        return dict(loss_vtc=loss_vtc)

    def encode_vision(self, image, test=False):
        """image [B,T,C,H,W] (or an image [B,C,H,W]) -> [B, embed_dim]; masking_prob applies unless test (:98-120)."""
        image = image.permute(0, 2, 1, 3, 4).contiguous() if image.ndim == 5 else image.unsqueeze(2)
        p = _get(_get(_get(self.config, "model"), "vision_encoder"), "masking_prob", 0.0)
        if not test and p > 0.0:
            return self.vision_encoder(image, masking_prob=p)
        return self.vision_encoder(image)

    def encode_text(self, text):
        """token ids [B, max_txt_l] (or strings, with a tokenizer) -> [B, embed_dim]."""
        if not torch.is_tensor(text):
            if self.tokenizer is None:
                raise NotImplementedError("ivb200 ViCLIP.encode_text: pass token ids; tokenization is host code "
                                          "(give ViCLIP a tokenizer to encode strings)")
            text = self.tokenizer(text, context_length=_get(self.config, "max_txt_l"))
        device = next(self.text_encoder.parameters()).device
        return self.text_encoder(text.to(device))

    @torch.no_grad()
    def clip_contrastive_temperature(self, min_val=0.001, max_val=0.5):
        self.temp.clamp_(min=self.temp_min)        # in place on the device, no host read

    def build_vision_encoder(self):
        ve = _get(_get(self.config, "model"), "vision_encoder")
        name = _get(ve, "name")
        if name not in _VISION:
            raise NotImplementedError(f"ivb200 ViCLIP: vision encoder {name!r} (built: {sorted(_VISION)})")
        inputs = _get(self.config, "inputs")
        return _VISION[name](pretrained=_local_or_false(_get(ve, "pretrained")),
                             input_resolution=_get(inputs, "image_res"), kernel_size=_get(ve, "kernel_size", 1),
                             center=_get(ve, "center", True),
                             num_frames=_get(_get(inputs, "video_input"), "num_frames"),
                             drop_path=_get(ve, "drop_path_rate", 0.0), checkpoint_num=_get(ve, "checkpoint_num", 0))

    def build_text_encoder(self):
        te = _get(_get(self.config, "model"), "text_encoder")
        name = _get(te, "name")
        if name not in _TEXT:
            raise NotImplementedError(f"ivb200 ViCLIP: text encoder {name!r} (built: {sorted(_TEXT)})")
        return _TEXT[name](pretrained=_local_or_false(_get(te, "pretrained")), embed_dim=_get(te, "d_model"),
                           context_length=_get(self.config, "max_txt_l"), vocab_size=_get(te, "vocab_size"),
                           checkpoint_num=_get(te, "checkpoint_num", 0))

    def get_text_encoder(self):
        return self.text_encoder
