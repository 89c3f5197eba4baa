"""TEST / BASELINE INFRASTRUCTURE ONLY — the oracle of the MobileCLIP text tower (BASELINE cfg-3's text encoder).

  stage()        copies the unmodified mobileclip text_encoder.py / transformer.py into the git-ignored
                 oracle/_ref/reference/ (same layout as the reference tree; __graft_entry__.build() runs it), so that
                 tools/text_tower_table.py can time the reference module on the GPU box
  reference()    imports those two unmodified files (from the reference tree where it is mounted, else the staged
                 copies)
  restate()      a CPU restatement of the tower in functional torch
  loss_weights() the fixed weights of the scalar loss whose gradients the fixture stores
  make()         writes tests/golden/text_tower.npz by executing the unmodified reference TextTransformer:
                 python oracle/text_tower.py

Nothing here reads the reference at import time; only tests/, tools/ and the build import this module.
"""
from __future__ import annotations

import importlib
import json
import os
import shutil
import sys
import types
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
MC = "InternVideo2/multi_modality/models/backbones/internvideo2/mobileclip"
FILES = ("text_encoder.py", "transformer.py")
STAGED = Path(__file__).resolve().parent / "_ref" / "reference"

# a narrow tower: vocabulary 512, width 32, 2 layers of 2 heads of 16, the real context length 77
CFG = dict(context_length=77, vocab_size=512, dim=32, ffn_multiplier_per_layer=4.0, n_heads_per_layer=2,
           n_transformer_layers=2, norm_layer="layer_norm_fp32", causal_masking=True, model_name="base")
PROJ = 16
ALL_TOKENS_ROWS = 3     # the return_all_tokens output is stored for the first captions only (EOT at 4, 11 and 76)


def _source_root():
    from oracle import ref_shim
    return Path(ref_shim.REF_ROOT)


def stage(verbose=True) -> bool:
    src = Path("/root/reference") / MC
    try:
        mounted = src.is_dir()
    except OSError:
        mounted = False
    if not mounted:
        return (STAGED / MC / FILES[0]).is_file()
    (STAGED / MC).mkdir(parents=True, exist_ok=True)
    for f in FILES:
        shutil.copyfile(src / f, STAGED / MC / f)
    if verbose:
        print(f"text_tower.stage: {len(FILES)} mobileclip files -> {STAGED / MC}")
    return True


def available() -> bool:
    return (_source_root() / MC / FILES[0]).is_file()


def reference():
    """The reference module mobileclip/text_encoder.py (with its sibling transformer.py), imported without the package
    __init__, which would also import the tokenizer and its vocabulary file."""
    pkg = "_ivref_mobileclip"
    if pkg not in sys.modules:
        m = types.ModuleType(pkg)
        m.__path__ = [str(_source_root() / MC)]
        sys.modules[pkg] = m
    return importlib.import_module(pkg + ".text_encoder")


def restate(sd, ids, n_layers, n_heads, return_all_tokens=False, eps=1e-5):
    """TextTransformer.encode_text — {MC}/text_encoder.py:131-219 with TransformerEncoder.forward and
    MultiHeadAttention._forward_impl ({MC}/transformer.py:200-294, 420-450), causal masking: token embedding plus the
    position table (no embed_scale), pre-norm blocks (LayerNorm, qkv with bias, (q * d^-0.5) k^T plus the -inf upper
    triangle, softmax, out_proj; LayerNorm, Linear, erf GELU, Linear), the final LayerNorm, then the EOT row
    (ids.argmax) times projection_layer, or every row with return_all_tokens.  sd: the tower's state_dict keys."""
    B, L = ids.shape
    x = sd["embedding_layer.weight"][ids] + sd["positional_embedding.pos_embed.pos_embed"].reshape(L, -1)
    D = x.shape[-1]
    d = D // n_heads
    mask = torch.full((L, L), float("-inf"), dtype=x.dtype).triu(1)
    for i in range(n_layers):
        p = lambda k: sd[f"transformer.{i}.{k}"]  # noqa: E731
        h = F.layer_norm(x, (D,), p("pre_norm_mha.0.weight"), p("pre_norm_mha.0.bias"), eps)
        qkv = F.linear(h, p("pre_norm_mha.1.qkv_proj.weight"), p("pre_norm_mha.1.qkv_proj.bias"))
        q, k, v = qkv.reshape(B, L, 3, n_heads, d).permute(2, 0, 3, 1, 4)
        a = torch.softmax((q * d ** -0.5) @ k.transpose(-2, -1) + mask, -1) @ v
        x = x + F.linear(a.transpose(1, 2).reshape(B, L, D), p("pre_norm_mha.1.out_proj.weight"),
                         p("pre_norm_mha.1.out_proj.bias"))
        h = F.layer_norm(x, (D,), p("pre_norm_ffn.0.weight"), p("pre_norm_ffn.0.bias"), eps)
        h = F.gelu(F.linear(h, p("pre_norm_ffn.1.weight"), p("pre_norm_ffn.1.bias")))
        x = x + F.linear(h, p("pre_norm_ffn.4.weight"), p("pre_norm_ffn.4.bias"))
    x = F.layer_norm(x, (D,), sd["final_layer_norm.weight"], sd["final_layer_norm.bias"], eps)
    if return_all_tokens:
        return x
    return x[torch.arange(B), ids.argmax(-1)] @ sd["projection_layer"]


def loss_weights(pooled_shape, all_shape):
    """(wp, wa): the loss is sum(pooled * wp) + sum(all_tokens * wa).  A closed form, so the fixture need not store
    them."""
    def w(shape, f):
        i = torch.arange(int(np.prod(shape)), dtype=torch.float64)
        return torch.cos(f * i + 0.3).reshape(shape).float()
    return w(tuple(pooled_shape), 0.71), w(tuple(all_shape), 0.37)


def caption_ids(B=8, L=77, V=512, seed=23):
    """Caption ids as the tokenizer lays them out: SOT (V - 2), words, EOT (V - 1, the largest id of the row), then
    zero padding, with the EOT at a different position in every row (the last slot included) and repeated word ids
    inside and across rows."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(B, L, dtype=torch.int64)
    for b in range(B):
        n = [3, 10, 75, 20, 1, 40, 7, 55][b % 8]           # words; the EOT lands at n + 1 (75 words: the last slot)
        ids[b, 0] = V - 2
        ids[b, 1:n + 1] = torch.randint(1, 12 if b % 2 else V - 2, (n,), generator=g)   # odd rows: few distinct ids
        ids[b, n + 1] = V - 1
    return ids


def _bf16_bits(t):
    return t.detach().to(torch.bfloat16).view(torch.int16).numpy()


def load(path):
    """(cfg, fp32 state_dict, the npz itself: ids, outputs and gradients) of a fixture make() wrote."""
    z = np.load(path)
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {k[2:]: torch.from_numpy(z[k]).view(torch.bfloat16).float() for k in z.files if k.startswith("w/")}
    return cfg, sd, z


def make(path=ROOT / "tests" / "golden" / "text_tower.npz"):
    """The unmodified reference tower at CFG, fp32 on the CPU: bf16-representable parameters (stored as bf16 bits;
    projection_layer, uninitialised in the reference, drawn here), caption_ids(); the pooled output of every caption,
    the return_all_tokens output of the first ALL_TOKENS_ROWS, and every parameter gradient of the loss_weights loss
    over the two."""
    torch.manual_seed(2468)
    tower = reference().TextTransformer(CFG, PROJ)
    g = torch.Generator().manual_seed(29)
    with torch.no_grad():
        tower.projection_layer.copy_(torch.randn(tower.projection_layer.shape, generator=g) * CFG["dim"] ** -0.5)
        for name, p in tower.named_parameters():
            if name.endswith("bias"):
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
            elif "norm" in name and name.endswith("weight"):
                p.add_(torch.randn(p.shape, generator=g) * 0.1)
            elif name == "embedding_layer.weight":
                p.mul_(0.5)
            p.copy_(p.to(torch.bfloat16).float())
    ids = caption_ids(V=CFG["vocab_size"])
    pooled = tower(ids)
    every = tower(ids[:ALL_TOKENS_ROWS], return_all_tokens=True)
    wp, wa = loss_weights(pooled.shape, every.shape)
    ((pooled * wp).sum() + (every * wa).sum()).backward()
    blob = {"cfg": np.frombuffer(json.dumps(dict(CFG, projection_dim=PROJ)).encode(), dtype=np.uint8),
            "ids": ids.numpy(), "pooled": pooled.detach().numpy(), "all_tokens": every.detach().numpy()}
    for k, t in tower.state_dict().items():
        blob["w/" + k] = _bf16_bits(t)
    for k, p in tower.named_parameters():
        blob["g/" + k] = p.grad.numpy()
    np.savez_compressed(path, **blob)
    print(f"text_tower: pooled {tuple(pooled.shape)}, all tokens {tuple(every.shape)}, {len(blob)} arrays, "
          f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    assert available(), "reference not mounted"
    make()
