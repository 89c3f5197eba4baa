"""The frozen LLaMA-7B text tower of InternVideo2-CLIP (the 1B and 6B recipes, scripts/pretraining/clip/{1B,6B}) on the
libivb200 kernels.  Inference only, except for text_projection.

Mirrors (constructor, attribute names, state_dict keys, order and shapes, forward contract):
  InternVideo2/multi_modality/models/backbones/internvideo2/internvideo2_clip_text.py:14-52   `LLaMA`
with `transformer` transformers' `LlamaModel` (embed_tokens, layers.i.{self_attn.{q,k,v,o}_proj, mlp.{gate,up,down}_proj,
input_layernorm, post_attention_layernorm}, norm), so that the `transformer.*` and `text_projection` keys of an
InternVL-C checkpoint load unchanged.  The model config is read from `<llama_path>/config.json` with json, or given as a
dict; transformers is not needed.

The path of forward(text), ids int64 [B, L] (pad id 0, right-padded):
  embedding  the token rows into the fp32 residual stream (ivb_token_embed_fwd with a cached zero position table)
  layer      10 launches: RMSNorm -> q, k, v GEMMs into the column slots of one [B*L, 3D] buffer -> RoPE on q and k in
             place (ivb_rope_qk, HF's rotate_half pairing, cos / sin tables built once per (L, head_dim, theta,
             device) as HF's LlamaRotaryEmbedding builds them, in fp32) -> causal attention -> o_proj accumulated into the
             stream -> RMSNorm -> gate and up in one SwiGLU GEMM (IVB_EPI_SWIGLU) -> down_proj accumulated into the stream
  output     each caption's last kept token, at (text > 0).sum(1) - 1, gathered on the device; the final RMSNorm of
             those B rows and the projection GEMM text_projection ([width, clip_embed_dim], read transposed).  The
             projection is differentiable (open_text_projection); nothing else is.
Nothing is read by the host, so a forward is capturable in a CUDA graph once a first call has built the cached tables
and joined each layer's gate and up weights.

Why causal attention alone is exact: the reference also masks the padded keys (attention_mask = text > 0), but with
right padding a kept token never attends to a later position, so that mask changes no output the tower returns.  A
caption whose nonzero ids are not a prefix, or that has none, gets a NaN output row here (as bert_modules.key_lengths
does); the reference returns a value for it.  An id outside [0, vocab_size) makes the whole output NaN (a device flag).

Gate and up weights: the SwiGLU GEMM reads them as the two halves of one contiguous [2I, D] tensor.  The first forward
of a layer rebinds both parameters' .data to views of one buffer (once the old tensors are freed this costs no memory,
and load_state_dict still copies in place); no second copy is kept.

LoRA: use_lora=True is accepted.  The reference's adapters (peft, r = 16 on q_proj and v_proj) are the identity at
initialisation (lora_B = 0) and frozen in every recipe, so the output is the same; the module has the use_lora=False
keys.  Loading maps `*.base_layer.weight` to `*.weight`, drops the adapters, refuses a nonzero lora_B tensor, and
ignores the `rotary_emb.inv_freq` buffers older transformers saved.

Refused with NotImplementedError: rope_scaling, num_key_value_heads != num_attention_heads (GQA), hidden_act other than
"silu", attention_bias or mlp_bias, a head_dim the RoPE kernel does not take (a multiple of 16 in [16, 128]), L >
max_position_embeddings, and a call with grad enabled while a parameter other than text_projection requires grad.
Parameters must be bf16 (model.bfloat16()) and the ids on the GPU.  modules.set_fp8_inference does not reach these
layers: they stay bf16.

Initialisation uses the distributions of transformers' LlamaPreTrainedModel._init_weights (Linear and Embedding weights
N(0, initializer_range), the padding row zero, RMSNorm weights 1) but is not draw-for-draw the reference's: the order of
draws depends on the transformers version.  text_projection is torch.empty, as in the reference.
"""
from __future__ import annotations

import json
import os
import types

import torch
import torch.nn as nn

from . import lowlevel as ll
from . import ops
from .modules import check_input, index_poison

# Chinese-Alpaca-7B (the recipes' llama_path): LLaMA-7B with the extended Chinese vocabulary
LLAMA_7B = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "vocab_size": 49954, "hidden_size": 4096,
            "intermediate_size": 11008, "num_hidden_layers": 32, "num_attention_heads": 32, "num_key_value_heads": 32,
            "hidden_act": "silu", "max_position_embeddings": 2048, "rms_norm_eps": 1e-6, "rope_theta": 10000.0,
            "rope_scaling": None, "attention_bias": False, "mlp_bias": False, "initializer_range": 0.02,
            "pad_token_id": 0, "bos_token_id": 1, "eos_token_id": 2, "tie_word_embeddings": False}

_DEFAULTS = {"num_key_value_heads": None, "hidden_act": "silu", "max_position_embeddings": 2048, "rms_norm_eps": 1e-6,
             "rope_theta": 10000.0, "rope_scaling": None, "attention_bias": False, "mlp_bias": False,
             "initializer_range": 0.02, "pad_token_id": None, "head_dim": None}


def _config(config):
    """An attribute view of a LLaMA config.json dict (transformers' LlamaConfig defaults for the fields it omits)."""
    c = dict(_DEFAULTS, **config)
    if c["num_key_value_heads"] is None:
        c["num_key_value_heads"] = c["num_attention_heads"]
    if c["head_dim"] is None:
        c["head_dim"] = c["hidden_size"] // c["num_attention_heads"]
    return types.SimpleNamespace(**c)


def check_config(cfg):
    """The LLaMA variants the tower runs: refuses the others with NotImplementedError."""
    if cfg.rope_scaling is not None:
        raise NotImplementedError("ivb200 LLaMA: rope_scaling is not implemented")
    if cfg.num_key_value_heads != cfg.num_attention_heads:
        raise NotImplementedError("ivb200 LLaMA: grouped-query attention (num_key_value_heads != num_attention_heads) "
                                  "is not implemented")
    if cfg.hidden_act != "silu":
        raise NotImplementedError(f"ivb200 LLaMA: hidden_act {cfg.hidden_act!r}; only 'silu' is implemented")
    if cfg.attention_bias or cfg.mlp_bias:
        raise NotImplementedError("ivb200 LLaMA: attention_bias / mlp_bias are not implemented")
    d = cfg.head_dim
    if d % 16 or not 16 <= d <= 128:
        raise NotImplementedError(f"ivb200 LLaMA: head_dim {d}; the RoPE kernel takes a multiple of 16 in [16, 128]")


class LlamaRMSNorm(nn.Module):
    """transformers LlamaRMSNorm: weight [D] (ones), variance_epsilon."""

    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps


class LlamaAttention(nn.Module):
    """transformers LlamaAttention: q, k, v, o projections without bias."""

    def __init__(self, cfg):
        super().__init__()
        D, Hd = cfg.hidden_size, cfg.num_attention_heads * cfg.head_dim
        self.num_heads, self.head_dim = cfg.num_attention_heads, cfg.head_dim
        self.q_proj = nn.Linear(D, Hd, bias=False)
        self.k_proj = nn.Linear(D, Hd, bias=False)
        self.v_proj = nn.Linear(D, Hd, bias=False)
        self.o_proj = nn.Linear(Hd, D, bias=False)


class LlamaMLP(nn.Module):
    """transformers LlamaMLP: down(silu(gate(x)) * up(x)), no bias."""

    def __init__(self, cfg):
        super().__init__()
        self.gate_proj = nn.Linear(cfg.hidden_size, cfg.intermediate_size, bias=False)
        self.up_proj = nn.Linear(cfg.hidden_size, cfg.intermediate_size, bias=False)
        self.down_proj = nn.Linear(cfg.intermediate_size, cfg.hidden_size, bias=False)

    def gate_up(self):
        """gate_proj.weight and up_proj.weight as the halves of one contiguous [2I, D] tensor (the SwiGLU GEMM's B).  The
        first call rebinds both parameters to views of one buffer; later calls only check they still are."""
        g, u = self.gate_proj.weight, self.up_proj.weight
        I, D = g.shape
        joined = (g.is_contiguous() and u.is_contiguous() and g.device == u.device and g.dtype == u.dtype
                  and g.untyped_storage().data_ptr() == u.untyped_storage().data_ptr()
                  and u.storage_offset() == g.storage_offset() + g.numel())
        if not joined:
            buf = torch.cat([g.detach(), u.detach()])
            g.data, u.data = buf[:I], buf[I:]
        return g.detach().as_strided((2 * I, D), (D, 1))


class LlamaDecoderLayer(nn.Module):
    """transformers LlamaDecoderLayer: pre-norm attention and SwiGLU MLP branches on the residual stream."""

    def __init__(self, cfg):
        super().__init__()
        self.self_attn = LlamaAttention(cfg)
        self.mlp = LlamaMLP(cfg)
        self.input_layernorm = LlamaRMSNorm(cfg.hidden_size, eps=cfg.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNorm(cfg.hidden_size, eps=cfg.rms_norm_eps)

    def forward_stream(self, x, B, L, cos, sin):
        """The layer over the fp32 residual stream x [B*L, D], in place: 10 library calls."""
        at, mlp = self.self_attn, self.mlp
        H, d = at.num_heads, at.head_dim
        Hd = H * d
        ln1, ln2 = self.input_layernorm, self.post_attention_layernorm
        n1 = ll.norm_fwd(x, ln1.weight, eps=ln1.variance_epsilon, want_stats=False)[0]
        qkv = torch.empty((x.shape[0], 3 * Hd), device=x.device, dtype=torch.bfloat16)
        for i, lin in enumerate((at.q_proj, at.k_proj, at.v_proj)):
            ll.gemm(n1, lin.weight, out0=qkv[:, i * Hd:(i + 1) * Hd])
        q, k, v = qkv[:, :Hd], qkv[:, Hd:2 * Hd], qkv[:, 2 * Hd:]
        ll._rope_qk(q, k, B, L, H, d, cos, sin)
        a, _ = ll.attn_fwd(q, k, v, B, L, H, d, d ** -0.5, want_lse=False, causal=True)
        ll.gemm(a, at.o_proj.weight, epi=ll.EPI_F32, flags=ll.FLAG_ACCUM, out0=x)        # x + a Wo^T
        n2 = ll.norm_fwd(x, ln2.weight, eps=ln2.variance_epsilon, want_stats=False)[0]
        g = ll.gemm(n2, mlp.gate_up(), epi=ll.EPI_SWIGLU)                                 # silu(n2 Wg^T) * (n2 Wu^T)
        ll.gemm(g, mlp.down_proj.weight, epi=ll.EPI_F32, flags=ll.FLAG_ACCUM, out0=x)     # x + g Wd^T
        return x


class LlamaModel(nn.Module):
    """transformers LlamaModel: embed_tokens, layers, norm (the rotary tables are derived, not parameters)."""

    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        self.padding_idx = cfg.pad_token_id
        self.embed_tokens = nn.Embedding(cfg.vocab_size, cfg.hidden_size, padding_idx=cfg.pad_token_id)
        self.layers = nn.ModuleList([LlamaDecoderLayer(cfg) for _ in range(cfg.num_hidden_layers)])
        self.norm = LlamaRMSNorm(cfg.hidden_size, eps=cfg.rms_norm_eps)


_TABLES = {}


def rope_tables(L, d, theta, device):
    """(cos, sin) fp32 [L, d/2] for positions 0 .. L-1, as transformers' LlamaRotaryEmbedding builds them (default rope
    type, attention_scaling 1): inv_freq = 1 / theta^(arange(0, d, 2) / d) and freqs = pos (x) inv_freq in fp32.  Built
    once per (L, d, theta, device) and cached."""
    key = (L, d, float(theta), str(torch.device(device)))
    if key not in _TABLES:
        inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.int64).to(device=device, dtype=torch.float) / d))
        freqs = torch.outer(torch.arange(L, device=device, dtype=torch.float), inv_freq)
        _TABLES[key] = (freqs.cos().contiguous(), freqs.sin().contiguous())
    return _TABLES[key]


def _zero_pos(L, D, device):
    key = ("pos", L, D, str(torch.device(device)))
    if key not in _TABLES:
        _TABLES[key] = torch.zeros((L, D), device=device, dtype=torch.bfloat16)
    return _TABLES[key]


def last_token_poison(text):
    """(index int64 [B] of each caption's last kept token, fp32 [B] 0 or NaN): NaN where the nonzero ids are not a prefix
    of the row or there are none.  On the device; nothing is read by the host."""
    B, L = text.shape
    keep = text > 0
    n = keep.sum(1)
    prefix = torch.arange(L, device=text.device)[None, :] < n[:, None]
    ok = (keep == prefix).all(1) & (n > 0)
    z = torch.zeros((B,), device=text.device, dtype=torch.float32)
    return (n - 1).clamp(min=0), torch.where(ok, z, torch.full_like(z, float("nan")))


class LLaMA(nn.Module):
    """internvideo2_clip_text.py:14-52; see the module docstring.  config: a config.json dict (LLAMA_7B, say), used when
    llama_path is None."""

    def __init__(self, use_flash_attn=True, transformer_width=4096, llama_path=None, use_lora=True, clip_embed_dim=768,
                 config=None):
        super().__init__()
        if llama_path is not None:
            with open(os.path.join(llama_path, "config.json")) as f:
                config = json.load(f)
        if config is None:
            raise ValueError("LLaMA: give llama_path (a directory holding config.json) or a config dict")
        cfg = _config(config)
        check_config(cfg)
        self.use_flash_attn = use_flash_attn
        self.transformer_width = transformer_width
        self.use_lora = use_lora
        self.transformer = LlamaModel(cfg)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, clip_embed_dim))
        self.transformer.apply(self._init_weights)
        self._register_load_state_dict_pre_hook(self._map_lora_keys)

    def _init_weights(self, module):
        std = self.transformer.config.initializer_range
        if isinstance(module, nn.Linear):
            module.weight.data.normal_(mean=0.0, std=std)
        elif isinstance(module, nn.Embedding):
            module.weight.data.normal_(mean=0.0, std=std)
            if module.padding_idx is not None:
                module.weight.data[module.padding_idx].zero_()
        elif isinstance(module, LlamaRMSNorm):
            module.weight.data.fill_(1.0)

    @staticmethod
    def _map_lora_keys(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        """A use_lora=True checkpoint (peft) in the use_lora=False keys: `*.base_layer.weight` -> `*.weight`, adapters
        dropped (a nonzero lora_B refused: its update is not the identity), `rotary_emb.inv_freq` buffers dropped."""
        for k in [k for k in state_dict if k.startswith(prefix)]:
            rest = k[len(prefix):]
            if ".lora_B." in rest and bool((state_dict[k] != 0).any()):
                raise NotImplementedError(f"ivb200 LLaMA: {k} is nonzero; trained LoRA adapters are not implemented")
            if ".lora_A." in rest or ".lora_B." in rest or rest.endswith("rotary_emb.inv_freq"):
                del state_dict[k]
            elif rest.endswith(".base_layer.weight"):
                state_dict[k[:-len(".base_layer.weight")] + ".weight"] = state_dict.pop(k)

    def _check_call(self, text):
        if torch.is_grad_enabled() and any(p.requires_grad for n, p in self.named_parameters()
                                           if n != "text_projection"):
            raise NotImplementedError("ivb200 LLaMA is forward-only except for text_projection: freeze the other "
                                      "parameters or call it under torch.no_grad()")
        cfg = self.transformer.config
        if text.dim() != 2:
            raise ll._lib.IvbError(f"ivb200 LLaMA: text must be ids [B, L], got {tuple(text.shape)}")
        if text.shape[1] > cfg.max_position_embeddings:
            raise NotImplementedError(f"ivb200 LLaMA: L = {text.shape[1]} > max_position_embeddings = "
                                      f"{cfg.max_position_embeddings}")
        bf16 = all(p.dtype == torch.bfloat16 for p in self.parameters())
        check_input(self, text, torch.bfloat16 if bf16 else torch.float32)

    def forward(self, text):
        """text int64 [B, L] -> [B, clip_embed_dim] bf16: the last kept token's final-norm row @ text_projection."""
        self._check_call(text)
        B, L = text.shape
        tr = self.transformer
        cfg = tr.config
        ids = text.long().contiguous()
        x, err = ll._token_embed_fwd(ids, tr.embed_tokens.weight, _zero_pos(L, cfg.hidden_size, text.device))
        cos, sin = rope_tables(L, cfg.head_dim, cfg.rope_theta, text.device)
        for layer in tr.layers:
            layer.forward_stream(x, B, L, cos, sin)
        last, poison = last_token_poison(ids)
        rows = x.view(B, L, -1)[torch.arange(B, device=text.device), last] + (poison + index_poison(err))[:, None]
        y = ll.norm_fwd(rows, tr.norm.weight, eps=tr.norm.variance_epsilon, want_stats=False)[0]
        return ops.linear(y, self.text_projection, w_t=True)
