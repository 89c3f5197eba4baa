"""TEST / BASELINE INFRASTRUCTURE ONLY — the oracle of InternVideo2-CLIP's LLaMA text tower.

  stage()        copies the unmodified internvideo2_clip_text.py into the git-ignored oracle/_ref/reference/ (same
                 layout as the reference tree; __graft_entry__.build() runs it)
  reference()    imports that unmodified file behind a `peft` stand-in (peft is not installed; only the use_lora=False
                 path runs, which never calls it)
  build_reference(cfg)  the reference LLaMA(use_lora=False) with cfg written as config.json into a temporary directory
  restate()      the tower's forward in functional fp32 torch
  make()         writes tests/golden/llama_text.npz by executing the unmodified reference module:
                 python oracle/llama_text.py

The fixture stores no parameters: each is drawn from a generator seeded by its name (draw_param).  Nothing here reads
the reference at import time; only tests/, tools/ and the build import this module.
"""
from __future__ import annotations

import importlib
import json
import os
import shutil
import sys
import tempfile
import types
import zlib
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
IV2 = "InternVideo2/multi_modality/models/backbones/internvideo2"
FILE = "internvideo2_clip_text.py"
STAGED = Path(__file__).resolve().parent / "_ref" / "reference"

# two layers of head_dim 128 (LLaMA-7B's); intermediate 688 = 2 * 344, so the SwiGLU GEMM's 128-wide N tiles have a tail
CFG = dict(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
           num_key_value_heads=2, hidden_act="silu", max_position_embeddings=64, rms_norm_eps=1e-6, rope_theta=10000.0,
           rope_scaling=None, attention_bias=False, mlp_bias=False, initializer_range=0.02, pad_token_id=0,
           bos_token_id=1, eos_token_id=2, tie_word_embeddings=False, model_type="llama",
           architectures=["LlamaForCausalLM"])
EMBED = 64          # clip_embed_dim
L = 24
LENGTHS = (L, 13, 1, 7)


def _source_root():
    from oracle import ref_shim
    return Path(ref_shim.REF_ROOT)


def stage(verbose=True) -> bool:
    src = Path("/root/reference") / IV2 / FILE
    try:
        mounted = src.is_file()
    except OSError:
        mounted = False
    if not mounted:
        return (STAGED / IV2 / FILE).is_file()
    (STAGED / IV2).mkdir(parents=True, exist_ok=True)
    shutil.copyfile(src, STAGED / IV2 / FILE)
    if verbose:
        print(f"llama_text.stage: {FILE} -> {STAGED / IV2}")
    return True


def available() -> bool:
    return (_source_root() / IV2 / FILE).is_file()


def _peft_stub():
    """peft's three names; the use_lora=False path never calls them."""
    m = types.ModuleType("peft")

    def get_peft_model(*args, **kwargs):
        raise NotImplementedError("the oracle runs LLaMA(use_lora=False) only")
    m.get_peft_model = get_peft_model
    m.LoraConfig = get_peft_model
    m.TaskType = types.SimpleNamespace(CAUSAL_LM="CAUSAL_LM")
    return m


def reference():
    """The unmodified internvideo2_clip_text.py, imported on its own (the package __init__ would import the vision
    tower's flash-attention dependencies)."""
    sys.modules.setdefault("peft", _peft_stub())
    pkg = "_ivref_llama"
    if pkg not in sys.modules:
        m = types.ModuleType(pkg)
        m.__path__ = [str(_source_root() / IV2)]
        sys.modules[pkg] = m
    return importlib.import_module(pkg + ".internvideo2_clip_text")


def build_reference(cfg=CFG, clip_embed_dim=EMBED):
    """LLaMA(use_flash_attn=False, transformer_width=hidden, llama_path=<tmp with cfg as config.json>, use_lora=False)."""
    mod = reference()
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "config.json"), "w") as f:
            json.dump(cfg, f)
        return mod.LLaMA(use_flash_attn=False, transformer_width=cfg["hidden_size"], llama_path=tmp, use_lora=False,
                         clip_embed_dim=clip_embed_dim)


def draw_param(name, shape):
    """The fixture's value of one parameter, bf16-representable, from a generator seeded by its name alone: RMSNorm
    weights 1 + N(0, 0.1^2), the token table N(0, 1), every other tensor N(0, 1 / fan_in) (text_projection: its rows)."""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    r = torch.randn(shape, generator=g)
    if name.endswith("norm.weight"):
        v = 1 + 0.1 * r
    elif name.endswith("embed_tokens.weight"):
        v = r
    elif name == "text_projection":
        v = r * shape[0] ** -0.5
    else:
        v = r * shape[1] ** -0.5
    return v.to(torch.bfloat16).float()


def draw_state(module):
    """{name: draw_param(name, shape)} for every parameter of `module`, in its state_dict order."""
    return {k: draw_param(k, tuple(v.shape)) for k, v in module.state_dict().items()}


def caption_ids():
    """Right-padded captions of LENGTHS ids in L slots (ids in [1, V), BOS 1 first), then zeros.  int64 [B, L]."""
    g = torch.Generator().manual_seed(43)
    ids = torch.zeros(len(LENGTHS), L, dtype=torch.int64)
    for b, n in enumerate(LENGTHS):
        ids[b, :n] = torch.randint(3, CFG["vocab_size"], (n,), generator=g)
        ids[b, 0] = 1
    return ids


def rope_tables(L_, d, theta):
    """transformers LlamaRotaryEmbedding (default type): inv_freq = 1 / theta^(arange(0, d, 2) / d), freqs = pos (x)
    inv_freq, in fp32."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.int64).float() / d))
    freqs = torch.outer(torch.arange(L_, dtype=torch.float), inv_freq)
    return freqs.cos(), freqs.sin()


def restate(sd, ids, cfg=CFG, dtype=torch.float32):
    """LLaMA.forward(ids) (internvideo2_clip_text.py:45-52) through transformers' LlamaModel: embed_tokens; per layer
    (LlamaDecoderLayer) x += o_proj(attn(rope(q), rope(k), v)) over RMSNorm(x), causal and masked on the padded keys
    (attention_mask = ids > 0), then x += down(silu(gate(h)) * up(h)) over RMSNorm(x); the final norm; the last kept
    token's row at (ids > 0).sum(1) - 1; @ text_projection.  RMSNorm: w * x / sqrt(mean(x^2) + eps).  RoPE:
    rotate_half, x' = x cos + rotate_half(x) sin with cos, sin = cat(freqs, freqs).  sd: the module's state_dict;
    dtype: the compute type (fp32; bf16 gives the restatement's own bf16 error, the yardstick of the GPU tests)."""
    B, n = ids.shape
    D, H, eps = cfg["hidden_size"], cfg["num_attention_heads"], cfg["rms_norm_eps"]
    d = D // H
    w = {k: v.to(dtype) for k, v in sd.items()}
    dev = ids.device

    def rms(t, k):
        tf = t.float()
        return (w[k].float() * (tf * torch.rsqrt(tf.pow(2).mean(-1, keepdim=True) + eps))).to(dtype)

    c, s = rope_tables(n, d, cfg["rope_theta"])
    c, s = torch.cat([c, c], -1).to(dev, dtype), torch.cat([s, s], -1).to(dev, dtype)

    def rope(t):
        t1, t2 = t[..., :d // 2], t[..., d // 2:]
        return t * c + torch.cat([-t2, t1], -1) * s
    keep = ids > 0
    allowed = torch.tril(torch.ones(n, n, dtype=torch.bool, device=dev))[None, None] & keep[:, None, None, :]
    x = w["transformer.embed_tokens.weight"][ids]
    for i in range(cfg["num_hidden_layers"]):
        p = f"transformer.layers.{i}."
        h = rms(x, p + "input_layernorm.weight")
        q, k, v = (F.linear(h, w[p + f"self_attn.{m}_proj.weight"]).reshape(B, n, H, d).transpose(1, 2)
                   for m in ("q", "k", "v"))
        q, k = rope(q), rope(k)
        sc = (q @ k.transpose(-1, -2)).float() * d ** -0.5
        pr = torch.softmax(sc.masked_fill(~allowed, float("-inf")), -1).to(dtype)
        a = (pr @ v).transpose(1, 2).reshape(B, n, D)
        x = x + F.linear(a, w[p + "self_attn.o_proj.weight"])
        h = rms(x, p + "post_attention_layernorm.weight")
        g = F.silu(F.linear(h, w[p + "mlp.gate_proj.weight"])) * F.linear(h, w[p + "mlp.up_proj.weight"])
        x = x + F.linear(g, w[p + "mlp.down_proj.weight"])
    x = rms(x, "transformer.norm.weight")
    x = x[torch.arange(B, device=dev), keep.sum(1) - 1]
    return x @ w["text_projection"]


def load(path):
    """(cfg, {name: fp32 parameter} in state_dict order, the npz itself) of a fixture make() wrote."""
    z = np.load(path)
    cfg = json.loads(bytes(z["cfg"]).decode())
    shapes = json.loads(bytes(z["shapes"]).decode())
    return cfg, {k: draw_param(k, tuple(s)) for k, s in shapes.items()}, z


def make(path=ROOT / "tests" / "golden" / "llama_text.npz"):
    """The unmodified reference LLaMA at CFG, fp32 on the CPU, every parameter from draw_param; the captions of
    caption_ids(); its output."""
    torch.manual_seed(0)
    model = build_reference().eval()
    sd = draw_state(model)
    model.load_state_dict(sd, strict=True)
    ids = caption_ids()
    with torch.no_grad():
        out = model(ids)
    blob = {"cfg": np.frombuffer(json.dumps(dict(CFG, clip_embed_dim=EMBED)).encode(), dtype=np.uint8),
            "shapes": np.frombuffer(json.dumps({k: list(v.shape) for k, v in sd.items()}).encode(), dtype=np.uint8),
            "ids": ids.numpy(), "out": out.numpy()}
    np.savez_compressed(path, **blob)
    print(f"llama_text: out {tuple(out.shape)}, {len(sd)} parameters, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    assert available(), "reference not mounted"
    make()
