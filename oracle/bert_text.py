"""TEST / BASELINE INFRASTRUCTURE ONLY — the oracle of the stage-2 BERT text encoder in text mode.

  stage()        copies the unmodified xbert.py into the git-ignored oracle/_ref/reference/ (same layout as the
                 reference tree; __graft_entry__.build() runs it), so that tools/bert_text_table.py can time the
                 reference module on the GPU box
  reference()    imports that unmodified file (from the reference tree where it is mounted, else the staged copy)
                 under the stubs of install_stubs()
  restate()      a CPU restatement of BertModel(..., mode="text") in functional torch
  make()         writes tests/golden/bert_text.npz by executing the unmodified reference BertModel:
                 python oracle/bert_text.py

xbert.py was written against an older transformers.  install_stubs() supplies exactly the names it needs that the
installed transformers no longer has, and only where they are missing; none of them touches the math of text mode:
  transformers.modeling_utils.apply_chunking_to_forward   transformers.pytorch_utils' function (moved there)
  transformers.modeling_utils.prune_linear_layer          transformers.pytorch_utils' function (moved there)
  transformers.modeling_utils.find_pruneable_heads_and_indices   raises: head pruning is never called here
  BertPreTrainedModel.all_tied_weights_keys               {}: init_weights() ties weights through it, and it is
                                                          set only by post_init(), which BertModel never calls
  BertPreTrainedModel.get_head_mask                       [None] * layers for head_mask None, the only form
                                                          BertModel.forward passes here (it raises otherwise)
The reference's init draws are therefore not relied on: make() draws every weight from its own seed, and the tests
compare keys, order and shapes against the reference, not init bytes.

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
BERT = "InternVideo2/multi_modality/models/backbones/bert"
FILE = "xbert.py"
STAGED = Path(__file__).resolve().parent / "_ref" / "reference"

# a narrow BERT: vocabulary 512, width 128, 2 heads of 64 (BERT-large's head dim), 3 layers of which the first 2 are
# text layers (fusion_layer 2: layer 2 carries the cross-attention weights), 64 positions; captions of max_txt_l = 40
CFG = dict(vocab_size=512, hidden_size=128, num_hidden_layers=3, num_attention_heads=2, intermediate_size=256,
           hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, max_position_embeddings=64,
           type_vocab_size=2, initializer_range=0.02, layer_norm_eps=1e-12, pad_token_id=0,
           position_embedding_type="absolute", fusion_layer=2, encoder_width=96, cross_module="ca")
L = 40
LENGTHS = (2, 17, 39, 40)
PROJ = 64       # text_proj: hidden_size -> the stage-2 embed_dim (narrowed)


def _source_root():
    from oracle import ref_shim
    return Path(ref_shim.REF_ROOT)


def stage(verbose=True) -> bool:
    src = Path("/root/reference") / BERT / FILE
    try:
        mounted = src.is_file()
    except OSError:
        mounted = False
    if not mounted:
        return (STAGED / BERT / FILE).is_file()
    (STAGED / BERT).mkdir(parents=True, exist_ok=True)
    shutil.copyfile(src, STAGED / BERT / FILE)
    if verbose:
        print(f"bert_text.stage: {FILE} -> {STAGED / BERT}")
    return True


def available() -> bool:
    return (_source_root() / BERT / FILE).is_file()


def install_stubs():
    """The names of the module docstring's list that the installed transformers lacks (the BertPreTrainedModel ones
    are set by reference(), after the import)."""
    import transformers.modeling_utils as mu
    import transformers.pytorch_utils as pu
    for name in ("apply_chunking_to_forward", "prune_linear_layer"):
        if not hasattr(mu, name):
            setattr(mu, name, getattr(pu, name))
    if not hasattr(mu, "find_pruneable_heads_and_indices"):
        def find_pruneable_heads_and_indices(*args, **kwargs):
            raise NotImplementedError("head pruning is not part of the oracle")
        mu.find_pruneable_heads_and_indices = find_pruneable_heads_and_indices


def _get_head_mask(self, head_mask, num_hidden_layers, is_attention_chunked=False):
    if head_mask is not None:
        raise NotImplementedError("head masks are not part of the oracle")
    return [None] * num_hidden_layers


def reference():
    """The reference module xbert.py, imported without the package __init__ (which would also import the tokenizer)."""
    install_stubs()
    pkg = "_ivref_bert"
    if pkg not in sys.modules:
        m = types.ModuleType(pkg)
        m.__path__ = [str(_source_root() / BERT)]
        sys.modules[pkg] = m
    xb = importlib.import_module(pkg + ".xbert")
    base = xb.BertPreTrainedModel
    if not hasattr(base, "all_tied_weights_keys"):
        base.all_tied_weights_keys = {}
    if not hasattr(base, "get_head_mask"):
        base.get_head_mask = _get_head_mask
    return xb


def build_reference(cfg=CFG):
    """xbert.BertModel(BertConfig(**cfg), add_pooling_layer=False), as the stage-2 recipes build the text encoder."""
    xb = reference()
    return xb.BertModel(xb.BertConfig(**cfg), add_pooling_layer=False)


def restate(sd, ids, mask, cfg=CFG):
    """BertModel.forward(ids, attention_mask=mask, mode="text").last_hidden_state — xbert.py:1122-1288 with
    BertEmbeddings.forward (:298-334) and the layers [0, fusion_layer) of BertEncoder (:690-811): word + token-type 0
    + absolute position rows, LayerNorm; per layer q, k, v Linear, q k^T / sqrt(d) plus (1 - mask) * -10000 on the
    keys, softmax, context, dense, LayerNorm(dense + x); Linear, erf GELU, Linear, LayerNorm(+ residual).  sd: the
    model's state_dict keys; dropout off (eval)."""
    B, n = ids.shape
    D, H, eps = cfg["hidden_size"], cfg["num_attention_heads"], cfg["layer_norm_eps"]
    d = D // H
    ln = lambda t, k: F.layer_norm(t, (D,), sd[k + ".weight"], sd[k + ".bias"], eps)  # noqa: E731
    x = (sd["embeddings.word_embeddings.weight"][ids] + sd["embeddings.token_type_embeddings.weight"][0]
         + sd["embeddings.position_embeddings.weight"][:n])
    x = ln(x, "embeddings.LayerNorm")
    ext = (1.0 - mask[:, None, None, :].to(x.dtype)) * -10000.0
    for i in range(cfg["fusion_layer"]):
        p = f"encoder.layer.{i}."
        lin = lambda t, k: F.linear(t, sd[p + k + ".weight"], sd[p + k + ".bias"])  # noqa: E731
        q, k, v = (lin(x, "attention.self." + w).reshape(B, n, H, d).transpose(1, 2) for w in ("query", "key", "value"))
        a = torch.softmax(q @ k.transpose(-1, -2) / d ** 0.5 + ext, -1) @ v
        x = ln(lin(a.transpose(1, 2).reshape(B, n, D), "attention.output.dense") + x, p + "attention.output.LayerNorm")
        h = F.gelu(lin(x, "intermediate.dense"))
        x = ln(lin(h, "output.dense") + x, p + "output.LayerNorm")
    return x


def caption_ids(V=CFG["vocab_size"]):
    """Right-padded BERT captions of LENGTHS tokens in L slots: [CLS] (1), words, [SEP] (2), then zeros, with repeated
    word ids inside every caption (odd captions: a vocabulary of 10 words) and across captions.  Returns (ids int64
    [B, L], attention_mask int64 [B, L])."""
    g = torch.Generator().manual_seed(41)
    ids = torch.zeros(len(LENGTHS), L, dtype=torch.int64)
    for b, n in enumerate(LENGTHS):
        ids[b, 0] = 1
        ids[b, 1:n - 1] = torch.randint(3, 13 if b % 2 else V, (n - 2,), generator=g)
        ids[b, n - 1] = 2
    ids[2, 3:9] = ids[2, 10]                      # a run of one id
    mask = (torch.arange(L)[None, :] < torch.tensor(LENGTHS)[:, None]).long()
    return ids, mask


def _draw(model, proj, seed=7):
    """Every parameter drawn from one seed, bf16-representable: Linear weights N(0, fan_in^-1), tables N(0, 0.25),
    LayerNorm weights 1 + N(0, 0.01), biases N(0, 0.0025); the layers from fusion_layer on, which text mode never
    runs, are zeros (the fixture stays small)."""
    g = torch.Generator().manual_seed(seed)
    unused = tuple(f"encoder.layer.{i}." for i in range(CFG["fusion_layer"], CFG["num_hidden_layers"]))
    with torch.no_grad():
        for name, p in list(model.named_parameters()) + [("proj." + k, v) for k, v in proj.named_parameters()]:
            r = torch.randn(p.shape, generator=g)
            if name.startswith(unused):
                v = torch.zeros_like(r)
            elif name.endswith("bias"):
                v = 0.05 * r
            elif "LayerNorm" in name:
                v = 1.0 + 0.1 * r
            elif "embeddings" in name:
                v = 0.5 * r
            else:
                v = r * p.shape[1] ** -0.5
            p.copy_(v.to(torch.bfloat16).float())


def _bf16_bits(t):
    return t.detach().to(torch.bfloat16).view(torch.int16).numpy()


def load(path):
    """(cfg, fp32 state_dict of the BertModel, text_proj (weight, bias), the npz itself) of a fixture make() wrote."""
    z = np.load(path)
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {}
    for k in z.files:
        if k.startswith("w/"):
            sd[k[2:]] = torch.from_numpy(z[k]).view(torch.bfloat16).float()
        elif k.startswith("buf/"):
            sd[k[4:]] = torch.from_numpy(z[k])
    order = json.loads(bytes(z["keys"]).decode())
    proj = tuple(torch.from_numpy(z[k]).view(torch.bfloat16).float() for k in ("proj/weight", "proj/bias"))
    return cfg, {k: sd[k] for k in order}, proj, z


def make(path=ROOT / "tests" / "golden" / "bert_text.npz"):
    """The unmodified reference BertModel at CFG, fp32 on the CPU in eval mode, every weight drawn by _draw; the
    captions of caption_ids(); last_hidden_state, its [:, 0] row and that row through text_proj."""
    torch.manual_seed(0)
    model = build_reference().eval()
    proj = torch.nn.Linear(CFG["hidden_size"], PROJ)
    _draw(model, proj)
    ids, mask = caption_ids()
    with torch.no_grad():
        last = model(ids, attention_mask=mask, return_dict=True, mode="text").last_hidden_state
        pooled = last[:, 0]
        feat = proj(pooled)
    sd = model.state_dict()
    blob = {"cfg": np.frombuffer(json.dumps(dict(CFG, text_proj_dim=PROJ)).encode(), dtype=np.uint8),
            "keys": np.frombuffer(json.dumps(list(sd)).encode(), dtype=np.uint8),
            "ids": ids.numpy(), "mask": mask.numpy(), "last_hidden_state": last.numpy(), "pooled": pooled.numpy(),
            "text_proj": feat.numpy(), "proj/weight": _bf16_bits(proj.weight), "proj/bias": _bf16_bits(proj.bias)}
    for k, t in sd.items():
        blob[("w/" if t.is_floating_point() else "buf/") + k] = _bf16_bits(t) if t.is_floating_point() else t.numpy()
    np.savez_compressed(path, **blob)
    print(f"bert_text: last_hidden_state {tuple(last.shape)}, {len(blob)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    assert available(), "reference not mounted"
    make()
