"""The BERT-large text encoder of the stage-2 recipes (`text_enc = "bert_large"`) in text mode, on the libivb200 kernels.
Inference only.

Mirrors (constructor, attribute names, state_dict keys, order and shapes, forward contract of mode="text"):
  InternVideo2/multi_modality/models/backbones/bert/xbert.py:272-334, 337-811, 1013-1288
      `BertEmbeddings`, `BertSelfAttention`, `BertSelfOutput`, `BertAttention`, `BertIntermediate`, `BertOutput`,
      `BertLayer`, `BertEncoder`, `BertModel(config, add_pooling_layer=False)`
so that the `text_encoder.bert.` keys of a stage-2 checkpoint, with that prefix stripped, load with strict=True (the
model's get_text_encoder() returns `text_encoder.bert`, internvideo2_stage2_visual.py:358-361).  The cross-attention
weights of the layers from `fusion_layer` on are registered as in the reference and never run.

The path of forward(input_ids, attention_mask, mode="text"), the reference's encode_text
(internvideo2_stage2_visual.py:269-289), which runs layers [0, fusion_layer):
  embedding  word row + (position row + token-type row 0) into an fp32 row (ivb_token_embed_fwd; the position and
             token-type tables are summed once per call, an O(L*D) table), then LayerNorm (eps 1e-12) to bf16
  layer      post-LN BERT layer: qkv (three bias GEMMs) -> attention with per-caption key lengths
             (ivb_attn_fwd_keylen) -> h1 = LN(h + a Wo^T + bo) -> g = GELU_erf(h1 W1^T + b1) (fused epilogue) ->
             LN(h1 + g W2^T + b2)
Precision of the residual path: bf16, as the reference keeps it when it runs in bf16.  Each LayerNorm writes its row in
bf16, and the next residual sum is formed in the GEMM epilogue in fp32 (acc + bias + the bf16 residual) and rounded to
bf16 once, in place over the residual; the LayerNorm statistics are fp32.  modules.set_fp8_inference switches the text
layers to FP8 GEMMs (BertLayer.forward_text); the residual path stays as above.

Key lengths come from attention_mask on the device: kv_len[b] = attention_mask[b].sum().  The reference masks the
padded keys with an additive -10000, which underflows to the same zero probability as the kernel's -inf; padded
queries are computed as in the reference.  A caption whose mask is not a prefix of ones (the tokenizer pads on the
right) or has no ones gets key length 0, which makes the attention kernel write NaN rows for it, so that caption's
output is NaN; an id outside [0, vocab_size) makes the whole output NaN (a device flag).  Nothing is read by the host
except for token_type_ids, when given, so a call without them is capturable in a CUDA graph.

Refused with NotImplementedError: modes "fusion" and "multi_modal" (cross-attention), position_embedding_type other
than "absolute", a hidden_act other than "gelu", non-zero token_type_ids, training mode with a dropout probability > 0
(the reference's BERT-large config has 0.1: call .eval()), and a call with grad enabled while a parameter requires grad
(the module has no backward).  Parameters must be bf16 (model.bfloat16()) and the ids on the GPU.
"""
from __future__ import annotations

import types
from typing import NamedTuple

import torch
import torch.nn as nn

from . import lowlevel as ll
from .modules import Fp8InferenceSwitch, block_precision, check_input, index_poison

# configs/config_bert_large.json of the multi-modality recipes (fusion_layer 19: the text layers are 0..18)
BERT_LARGE = {"architectures": ["BertForMaskedLM"], "attention_probs_dropout_prob": 0.1, "gradient_checkpointing": False,
              "hidden_act": "gelu", "hidden_dropout_prob": 0.1, "hidden_size": 1024, "initializer_range": 0.02,
              "intermediate_size": 4096, "layer_norm_eps": 1e-12, "max_position_embeddings": 512, "model_type": "bert",
              "num_attention_heads": 16, "num_hidden_layers": 24, "pad_token_id": 0,
              "position_embedding_type": "absolute", "type_vocab_size": 2, "use_cache": True, "vocab_size": 30522,
              "fusion_layer": 19, "encoder_width": 768, "cross_module": "ca"}


def _config(config):
    """An attribute view of an xbert-style config: a dict of the config_bert_large.json fields plus fusion_layer, or
    an object with those attributes (xbert.BertConfig)."""
    return types.SimpleNamespace(**config) if isinstance(config, dict) else config


class BertEmbeddings(nn.Module):
    """xbert.py:272-334: word, position and token-type tables, LayerNorm, and the position_ids buffer."""

    def __init__(self, config):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size, padding_idx=config.pad_token_id)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.register_buffer("position_ids", torch.arange(config.max_position_embeddings).expand((1, -1)))


class BertSelfAttention(nn.Module):
    """xbert.py:337-371: query, key, value (key and value read encoder_width columns in a cross-attention)."""

    def __init__(self, config, is_cross_attention):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError(f"The hidden size ({config.hidden_size}) is not a multiple of the number of attention "
                             f"heads ({config.num_attention_heads})")
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = config.hidden_size // config.num_attention_heads
        self.all_head_size = self.num_attention_heads * self.attention_head_size
        width = config.encoder_width if is_cross_attention else config.hidden_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(width, self.all_head_size)
        self.value = nn.Linear(width, self.all_head_size)


class BertSelfOutput(nn.Module):
    """xbert.py:501-512: dense, then LayerNorm of (dense output + residual)."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=config.layer_norm_eps)


class BertAttention(nn.Module):
    """xbert.py:515-567."""

    def __init__(self, config, is_cross_attention=False):
        super().__init__()
        self.self = BertSelfAttention(config, is_cross_attention)
        self.output = BertSelfOutput(config)


class BertIntermediate(nn.Module):
    """xbert.py:570-582: dense, then erf GELU (ACT2FN["gelu"])."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)


class BertOutput(nn.Module):
    """xbert.py:585-596: dense, then LayerNorm of (dense output + residual)."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=config.layer_norm_eps)


def layer_norm(x, ln, fp8):
    """A post-LN LayerNorm of the bf16 rows x: (bf16 rows, None), or with fp8 (the next GEMM runs in FP8) the same bf16
    rows and, from the same read of each row, their E4M3 rows with per-row scales (lowlevel.norm_fwd_fp8, save=True;
    its statistics are not used)."""
    if not fp8:
        return ll.norm_fwd(x, ln.weight, ln.bias, eps=ln.eps, layernorm=True, want_stats=False)[0], None
    q, s, y, _, _ = ll.norm_fwd_fp8(x, ln.weight, ln.bias, eps=ln.eps, layernorm=True, save=True)
    return y, (q, s)


class BertLayer(Fp8InferenceSwitch, nn.Module):
    """xbert.py:599-687; the cross-attention of layers >= fusion_layer is a parameter container only.  A text layer
    (below fusion_layer) runs in FP8 under modules.set_fp8_inference."""

    def __init__(self, config, layer_num):
        super().__init__()
        self.attention = BertAttention(config)
        self.has_cross_attention = layer_num >= config.fusion_layer
        if self.has_cross_attention:
            self.crossattention = BertAttention(config, is_cross_attention=True)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)

    def _fp8_linears(self):
        """The six GEMM weights of a text layer: query, key, value, attention output, intermediate, output; none for a
        fusion layer, which text mode never runs."""
        if self.has_cross_attention:
            return ()
        sa = self.attention.self
        return (sa.query, sa.key, sa.value, self.attention.output.dense, self.intermediate.dense, self.output.dense)

    def forward_text(self, h, B, L, kv_len, h8=None, fp8_out=False):
        """The self-attention layer over h, bf16 [B*L, D] (overwritten: it holds the first residual sum afterwards),
        with per-caption key lengths kv_len int32 [B] -> (the layer output, bf16 [B*L, D], and with fp8_out its E4M3
        rows and row scales, else None).  7 library calls in bf16.

        Under set_fp8_inference the six GEMMs run on the FP8 tensor cores (lowlevel.gemm_fp8) with per-token
        activation scales and the per-output-channel weight copies, each keeping its bf16 epilogue (bias, GELU, the
        in-place residual sum); h8: h's E4M3 rows and scales as the previous LayerNorm wrote them (None: cast here),
        the attention output and g are cast row by row, and the first LayerNorm writes the intermediate GEMM's E4M3
        rows with the residual.  Attention stays bf16."""
        sa, so = self.attention.self, self.attention.output
        M, D = h.shape
        H, d = sa.num_attention_heads, sa.attention_head_size
        w8 = None if self.fp8_inference is None else block_precision(self)

        def linear(act, act8, i, lin, **epilogue):
            if w8 is None:
                return ll.gemm(act, lin.weight, bias=lin.bias, **epilogue)
            q, s = act8 if act8 is not None else ll.fp8_quantize_rows(act)
            return ll.gemm_fp8(q, s, *w8[i], bias=lin.bias, **epilogue)
        if w8 is not None and h8 is None:
            h8 = ll.fp8_quantize_rows(h)
        qkv = torch.empty((M, 3 * D), device=h.device, dtype=torch.bfloat16)
        for i, lin in enumerate((sa.query, sa.key, sa.value)):
            linear(h, h8, i, lin, out0=qkv[:, i * D:(i + 1) * D])
        a, _ = ll.attn_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B, L, H, d, d ** -0.5, want_lse=False,
                           kv_len=kv_len)
        linear(a, None, 3, so.dense, flags=ll.FLAG_ACCUM, out0=h)                        # h + a Wo^T + bo
        h1, h1_8 = layer_norm(h, so.LayerNorm, w8 is not None)
        g = linear(h1, h1_8, 4, self.intermediate.dense, epi=ll.EPI_BIAS_GELU)
        linear(g, None, 5, self.output.dense, flags=ll.FLAG_ACCUM, out0=h1)             # h1 + g W2^T + b2
        return layer_norm(h1, self.output.LayerNorm, fp8_out)


class BertEncoder(nn.Module):
    """xbert.py:690-811: the layer stack."""

    def __init__(self, config):
        super().__init__()
        self.layer = nn.ModuleList([BertLayer(config, i) for i in range(config.num_hidden_layers)])


class BertTextOutput(NamedTuple):
    """What forward returns: last_hidden_state bf16 [B, L, hidden_size] (the reference's BaseModelOutput field)."""
    last_hidden_state: torch.Tensor


def key_lengths(attention_mask, B, L, device):
    """int32 [B] key lengths of a right-padded [B, L] mask (None: every key), computed on the device: the number of
    ones of each row, or 0 for a row that is not a prefix of ones or has none (the attention then writes NaN rows)."""
    if attention_mask is None:
        return torch.full((B,), L, device=device, dtype=torch.int32)
    if attention_mask.shape != (B, L):
        raise NotImplementedError(f"ivb200 BertModel: attention_mask must be a [B, L] = [{B}, {L}] padding mask, got "
                                  f"{tuple(attention_mask.shape)}")
    m = attention_mask.to(device=device, dtype=torch.int32)
    kv = m.sum(1, dtype=torch.int32)
    prefix = (torch.arange(L, device=device, dtype=torch.int32)[None, :] < kv[:, None]).to(torch.int32)
    return torch.where((m == prefix).all(1), kv, torch.zeros_like(kv))


class BertModel(nn.Module):
    """xbert.BertModel(config, add_pooling_layer=False) in text mode; see the module docstring."""

    def __init__(self, config, add_pooling_layer=False):
        super().__init__()
        config = _config(config)
        if add_pooling_layer:
            raise NotImplementedError("ivb200 BertModel: the pooler is not implemented (the stage-2 recipes build "
                                      "BertModel with add_pooling_layer=False)")
        if getattr(config, "position_embedding_type", "absolute") != "absolute":
            raise NotImplementedError("ivb200 BertModel: only absolute position embeddings are implemented")
        if config.hidden_act != "gelu":
            raise NotImplementedError(f"ivb200 BertModel: hidden_act {config.hidden_act!r}; only 'gelu' (erf) is "
                                      "implemented")
        self.config = config
        self.embeddings = BertEmbeddings(config)
        self.encoder = BertEncoder(config)
        self.apply(self._init_weights)

    def _init_weights(self, module):
        """xbert.py:909-919 (BertPreTrainedModel._init_weights)."""
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    def _check_call(self, input_ids, token_type_ids, mode):
        cfg = self.config
        if mode in ("fusion", "multi_modal"):
            raise NotImplementedError(f"ivb200 BertModel: mode {mode!r} runs the cross-attention layers, which are not "
                                      "implemented; only mode='text' ('temporal') is")
        if mode not in ("text", "temporal"):
            raise ValueError(f"BertModel: unknown mode {mode!r}")
        if self.training and (cfg.hidden_dropout_prob > 0 or cfg.attention_probs_dropout_prob > 0):
            raise NotImplementedError("ivb200 BertModel: dropout is not implemented; call .eval() (inference only)")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("ivb200 BertModel is forward-only: call it under torch.no_grad() or freeze its "
                                      "parameters")
        if token_type_ids is not None and bool((token_type_ids != 0).any()):
            raise NotImplementedError("ivb200 BertModel: token type ids other than 0 are not implemented")
        check_input(self, input_ids, self.embeddings.word_embeddings.weight.dtype)
        if input_ids.dim() != 2 or input_ids.shape[1] > cfg.max_position_embeddings:
            raise ll._lib.IvbError(f"ivb200 BertModel: input_ids must be [B, L] with L <= "
                                   f"{cfg.max_position_embeddings}, got {tuple(input_ids.shape)}")

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, return_dict=True, mode="text"):
        """input_ids int64 [B, L], attention_mask [B, L] (1 = token, 0 = right padding; None: no padding) ->
        BertTextOutput(last_hidden_state bf16 [B, L, hidden_size]) after layers [0, fusion_layer)."""
        self._check_call(input_ids, token_type_ids, mode)
        B, L = input_ids.shape
        emb = self.embeddings
        pos = (emb.position_embeddings.weight[:L].float() + emb.token_type_embeddings.weight[0].float()).to(torch.bfloat16)
        x, err = ll._token_embed_fwd(input_ids.long().contiguous(), emb.word_embeddings.weight, pos)
        layers = self.encoder.layer[:self.config.fusion_layer]
        fp8 = [layer.fp8_inference is not None for layer in layers] + [False]
        h, h8 = layer_norm(x, emb.LayerNorm, fp8[0])     # each LayerNorm also writes E4M3 rows for an FP8 layer after it
        kv_len = key_lengths(attention_mask, B, L, input_ids.device)
        for i, layer in enumerate(layers):
            h, h8 = layer.forward_text(h, B, L, kv_len, h8, fp8_out=fp8[i + 1])
        return BertTextOutput(h.reshape(B, L, -1) + index_poison(err))
