"""The MobileCLIP text tower of the video-text contrastive recipe (BASELINE cfg-3, `text_encoder.name = "mobileclip_b"`)
on the libivb200 kernels.

Mirrors (constructor, attribute names, state_dict keys, init draws, forward contract):
  InternVideo2/multi_modality/models/backbones/internvideo2/mobileclip/text_encoder.py:18-245   `TextTransformer`
  InternVideo2/multi_modality/models/backbones/internvideo2/mobileclip/transformer.py:89-125,142-450
      `LearnablePositionalEmbedding`, `MultiHeadAttention`, `TransformerEncoder`
so that the `text_encoder.` keys of a MobileCLIP checkpoint (mobileclip_blt.pt) load unchanged.

The path: token embedding + position table into the fp32 residual stream (ops.TokenEmbedFn), pre-norm LayerNorm blocks
with causal attention (ops.BlockFn / block_forward with BlockSpec(layernorm=True, causal=True): full qkv bias, erf
GELU, no LayerScale), the final LayerNorm, EOT pooling and the projection GEMM.  Tokenization stays host code: the
tower takes token ids.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .modules import Fp8Block, block_attn_fp8, block_precision, check_input, index_poison

# text_cfg and embed_dim of mobileclip/configs/mobileclip_b.json
MOBILECLIP_B = {"context_length": 77, "vocab_size": 49408, "dim": 512, "ffn_multiplier_per_layer": 4.0,
                "n_heads_per_layer": 8, "n_transformer_layers": 12, "norm_layer": "layer_norm_fp32",
                "causal_masking": True, "model_name": "base"}
MOBILECLIP_B_PROJECTION_DIM = 512


class LearnablePositionalEmbedding(nn.Module):
    """transformer.py:89-138: pos_embed [1, 1, L, D], truncated-normal init with std D ** -0.5."""

    def __init__(self, num_embeddings, embedding_dim):
        super().__init__()
        self.pos_embed = nn.Parameter(torch.empty(1, 1, num_embeddings, embedding_dim))
        self.embedding_dim, self.num_embeddings = embedding_dim, num_embeddings
        nn.init.trunc_normal_(self.pos_embed, mean=0, std=embedding_dim ** -0.5)


class PositionalEmbedding(nn.Module):
    """transformer.py:57-86 (the learnable form, the only one the reference builds)."""

    def __init__(self, num_embeddings, embedding_dim):
        super().__init__()
        self.pos_embed = LearnablePositionalEmbedding(num_embeddings, embedding_dim)


class MultiHeadAttention(nn.Module):
    """transformer.py:142-330, self-attention form: parameter container of qkv_proj ([3D, D], bias) and out_proj."""

    def __init__(self, embed_dim, num_heads):
        super().__init__()
        self.qkv_proj = nn.Linear(embed_dim, 3 * embed_dim, bias=True)
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=True)
        self.head_dim = embed_dim // num_heads
        self.scaling = self.head_dim ** -0.5
        self.num_heads, self.embed_dim = num_heads, embed_dim


class TransformerEncoder(Fp8Block, nn.Module):
    """transformer.py:333-450: pre-norm block, LayerNorm (eps 1e-5, fp32 statistics) -> MHA -> residual, LayerNorm ->
    Linear -> GELU (erf) -> Linear -> residual, no LayerScale, dropout 0.  Runs as one fused block (ops.BlockFn, or
    ops.block_forward without saving anything when no gradient is needed), at the precision modules.set_fp8 and
    modules.set_fp8_inference choose; causal attention stays bf16 in every precision."""

    def __init__(self, embed_dim, ffn_latent_dim, num_heads=8):
        super().__init__()
        attn_unit = MultiHeadAttention(embed_dim, num_heads)    # built first, as in the reference: the init draw order
        self.pre_norm_mha = nn.Sequential(nn.LayerNorm(embed_dim), attn_unit, nn.Dropout(p=0.0))
        self.pre_norm_ffn = nn.Sequential(nn.LayerNorm(embed_dim), nn.Linear(embed_dim, ffn_latent_dim), nn.GELU(),
                                          nn.Dropout(p=0.0), nn.Linear(ffn_latent_dim, embed_dim), nn.Dropout(p=0.0))
        self.embed_dim, self.ffn_dim = embed_dim, ffn_latent_dim

    def _spec(self, B, n, causal, training=False):
        ln1, a, ln2 = self.pre_norm_mha[0], self.pre_norm_mha[1], self.pre_norm_ffn[0]
        return ops.BlockSpec(B, n, a.num_heads, layernorm=True, eps1=ln1.eps, eps2=ln2.eps, scale=a.scaling,
                             causal=causal, precision=block_precision(self, training),
                             attn_fp8=block_attn_fp8(self) and not causal)

    def _fp8_linears(self):
        a = self.pre_norm_mha[1]
        return (a.qkv_proj, a.out_proj, self.pre_norm_ffn[1], self.pre_norm_ffn[4])

    def _param_tuple(self):
        ln1, a, ln2 = self.pre_norm_mha[0], self.pre_norm_mha[1], self.pre_norm_ffn[0]
        fc1, fc2 = self.pre_norm_ffn[1], self.pre_norm_ffn[4]
        return ops.BlockParams(n1w=ln1.weight, n1b=ln1.bias, qkvw=a.qkv_proj.weight, qkvb=a.qkv_proj.bias, qnw=None,
                               knw=None, projw=a.out_proj.weight, projb=a.out_proj.bias, g1=None, n2w=ln2.weight,
                               n2b=ln2.bias, fc1w=fc1.weight, fc1b=fc1.bias, fc2w=fc2.weight, fc2b=fc2.bias, g2=None)

    def forward_stream(self, x2d, B, n, causal=True):
        """fp32 residual stream [B*n, D] -> same.  Differentiated (ops.BlockFn) when grad mode is on and the stream or a
        parameter of the block needs a gradient; otherwise the no-grad block forward."""
        if torch.is_grad_enabled() and (x2d.requires_grad or any(p.requires_grad for p in self.parameters())):
            return ops.BlockFn.apply(x2d, self._spec(B, n, causal, training=True), None, None, *self._param_tuple())
        with torch.no_grad():
            out, _ = ops.block_forward(x2d, self._spec(B, n, causal), self._param_tuple(), save=False)
        return out


class TextTransformer(nn.Module):
    """text_encoder.py:18-245, the "base" variant.  forward(text_tokens int64 [B, context_length], key_padding_mask=None,
    return_all_tokens=False) -> [B, projection_dim] (the final LayerNorm of each caption's EOT token, the largest id of
    its row, times projection_layer), or with return_all_tokens the final LayerNorm of every token, [B, L, dim].

    As in the reference, key_padding_mask is ignored under causal masking, the embedding is not scaled by embed_scale,
    and projection_layer is allocated uninitialised (torch.empty: it comes from the checkpoint).  Refused: the "mct"
    variant (the reference raises too), a sequence length other than context_length (the reference would interpolate
    the position table; its tokenizer always pads to context_length), no_pos_embedding, dropout, and a
    key_padding_mask without causal masking.  An id outside [0, vocab_size) makes the output NaN (a device flag, no
    host read).  Parameters must be bf16 (model.bfloat16()) and the ids on the GPU."""

    def __init__(self, cfg, projection_dim, *args, **kwargs):
        super().__init__()
        model_dim = cfg["dim"]
        variant = cfg["model_name"]
        if variant == "mct":
            raise NotImplementedError("TextTransformer: the mct variant is not implemented (nor is it in the reference)")
        if variant != "base":
            raise ValueError(f"Unrecognized text encoder variant {variant}")
        if cfg.get("no_pos_embedding", False) or cfg.get("embed_dropout", 0.0):
            raise NotImplementedError("ivb200 TextTransformer: needs the position table and embed_dropout 0 "
                                      "(MobileCLIP-B's configuration)")
        if cfg["norm_layer"] not in ("layer_norm", "layer_norm_fp32"):
            raise NotImplementedError(f"Option: {cfg['norm_layer']} not supported.")
        self.vocab_size = cfg["vocab_size"]
        self.projection_dim = projection_dim
        self.embedding_layer = nn.Embedding(embedding_dim=model_dim, num_embeddings=self.vocab_size)
        self.embed_scale = 1.0 if cfg.get("no_scale_embedding", False) else model_dim ** -0.5
        self.context_length = cfg["context_length"]
        self.positional_embedding = PositionalEmbedding(self.context_length, model_dim)
        self.embedding_dropout = nn.Dropout(p=0.0)
        n_layers = cfg["n_transformer_layers"]
        ffn_mult = cfg["ffn_multiplier_per_layer"]
        ffn_mult = [ffn_mult] * n_layers if isinstance(ffn_mult, (float, int)) else ffn_mult
        heads = cfg["n_heads_per_layer"]
        heads = [heads] * n_layers if isinstance(heads, int) else heads
        ffn_dims = [int(math.ceil(model_dim * m / 16.0) * 16.0) for m in ffn_mult]
        self.transformer = nn.ModuleList([TransformerEncoder(model_dim, ffn_dims[i], heads[i]) for i in range(n_layers)])
        self.final_layer_norm = nn.LayerNorm(model_dim)
        self.projection_layer = nn.Parameter(torch.empty(model_dim, self.projection_dim))
        self.model_dim = model_dim
        self.causal_masking = cfg["causal_masking"]

    def forward_tokens(self, text_tokens, key_padding_mask=None):
        """-> (fp32 residual stream [B*L, dim] after the last block, B, L, int32[1] bad-id flag)."""
        B, L = text_tokens.shape
        if L != self.context_length:
            raise ll._lib.IvbError(f"ivb200 TextTransformer: sequence length {L} != context_length "
                                   f"{self.context_length} (pad the tokens to the context length)")
        if key_padding_mask is not None and not self.causal_masking:
            raise NotImplementedError("ivb200 TextTransformer: key_padding_mask is supported only under causal masking, "
                                      "where the reference ignores it")
        check_input(self, text_tokens, self.embedding_layer.weight.dtype)
        h, err = ops.TokenEmbedFn.apply(text_tokens.long(), self.embedding_layer.weight,
                                        self.positional_embedding.pos_embed.pos_embed)
        for layer in self.transformer:
            h = layer.forward_stream(h, B, L, self.causal_masking)
        return h, B, L, err

    def encode_text(self, text_tokens, key_padding_mask=None, return_all_tokens=False, *args, **kwargs):
        h, B, L, err = self.forward_tokens(text_tokens, key_padding_mask)
        ln = self.final_layer_norm
        if return_all_tokens:
            return ops.layernorm(h, ln.weight, ln.bias, ln.eps).reshape(B, L, self.model_dim) + index_poison(err)
        # EOT pooling (the EOT id is the largest of each row): LayerNorm is per row, so normalising the B pooled rows
        # only is the reference's arithmetic
        rows = h.reshape(B, L, self.model_dim)[torch.arange(B, device=h.device), text_tokens.argmax(dim=-1)]
        x = ops.layernorm(rows, ln.weight, ln.bias, ln.eps)
        return ops.linear(x, self.projection_layer, w_t=True) + index_poison(err)

    def forward(self, text_tokens, key_padding_mask=None, return_all_tokens=False, *args, **kwargs):
        return self.encode_text(text_tokens, key_padding_mask, return_all_tokens)
