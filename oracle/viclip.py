"""TEST / BASELINE INFRASTRUCTURE ONLY — the oracle of ViCLIP (InternVideo1/Pretrain/ViCLIP).

  stage()        copies the unmodified clip_vision.py, clip_text.py, simple_tokenizer.py with its
                 bpe_simple_vocab_16e6.txt.gz, models/utils.py (with the prompts.py it imports) and criterions.py into
                 the git-ignored oracle/_ref/reference/ (same layout as the reference tree; __graft_entry__.build()
                 runs it), so tools/viclip_table.py can time the reference modules on the GPU box
  import_viclip() imports clip_vision.py and clip_text.py unmodified, behind stand-ins for what this image lacks
  restate()      a CPU fp32 restatement of the two towers and the VTC loss in functional torch
  make()         writes tests/golden/viclip.npz by executing the unmodified reference modules:
                 python oracle/viclip.py

Nothing here reads the reference at import time; only tests/, tools/ and the build import this module.
"""
from __future__ import annotations

import importlib
import importlib.util
import json
import os
import re
import shutil
import sys
import types
import zlib
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
VC = "InternVideo1/Pretrain/ViCLIP"
CLIP = VC + "/models/backbones/clip"
FILES = (CLIP + "/clip_vision.py", CLIP + "/clip_text.py", CLIP + "/simple_tokenizer.py",
         CLIP + "/bpe_simple_vocab_16e6.txt.gz", VC + "/models/utils.py", VC + "/models/prompts.py",
         VC + "/models/criterions.py")
STAGED = Path(__file__).resolve().parent / "_ref" / "reference"

# narrow towers with head_dim 64, so the GPU kernels apply
VISION = dict(input_resolution=56, patch_size=14, width=128, layers=2, heads=2, output_dim=64, kernel_size=1,
              num_frames=4)
TEXT = dict(embed_dim=64, context_length=32, vocab_size=512, transformer_width=128, transformer_heads=2,
            transformer_layers=2, checkpoint_num=0)
B, T = 4, 4
MASK_P = 0.5
MASK_SEED = 1234
N_TOKENS = (VISION["input_resolution"] // VISION["patch_size"]) ** 2 * T + 1     # unmasked video: cls + T L patches
IDX = (0, 1, 1, 3)          # a duplicated idx: two captions of one video
# the recipe's temperature is 0.01; at 0.01 the logits carry 100x the bf16 rounding of the normalised embeddings, and
# the softmax gradients of a bf16 port scatter by several percent, so the fixture trains at 0.1
TEMP = 1 / 10.0


def _source_root():
    from oracle import ref_shim
    return Path(ref_shim.REF_ROOT)


def stage(verbose=True) -> bool:
    src = Path("/root/reference")
    try:
        mounted = (src / VC).is_dir()
    except OSError:
        mounted = False
    if not mounted:
        return (STAGED / FILES[0]).is_file()
    for rel in FILES:
        (STAGED / rel).parent.mkdir(parents=True, exist_ok=True)
        shutil.copyfile(src / rel, STAGED / rel)
    if verbose:
        print(f"viclip.stage: {len(FILES)} ViCLIP files -> {STAGED / VC}")
    return True


def available() -> bool:
    return (_source_root() / FILES[0]).is_file()


def _regex_stub():
    """`regex` is not installed: a stand-in whose compile maps the Unicode classes simple_tokenizer's pattern uses to
    `re` (CLIP_TEXT.__init__ builds a tokenizer; nothing is tokenized)."""
    m = types.ModuleType("regex")
    m.IGNORECASE = re.IGNORECASE
    m.compile = lambda p, flags=0: re.compile(p.replace(r"\p{L}", r"[^\W\d_]").replace(r"\p{N}", r"\d"), flags)
    m.findall = re.findall
    m.sub = re.sub
    return m


def import_viclip():
    """(clip_vision module, clip_text module) of the unmodified reference.  Stand-ins: timm (oracle/ref_shim.py), ftfy
    and regex.  clip_vision.py imports `models.utils` by its absolute name; ViCLIP's models/utils.py is loaded under a
    private package and bound to that name only while clip_vision.py executes, so it never meets the `models` package
    of InternVideo2 that other oracle code loads."""
    from oracle import ref_shim
    ref_shim.install_stubs()
    pkg = "_ivref_viclip"
    if pkg + ".clip_vision" in sys.modules:
        return sys.modules[pkg + ".clip_vision"], sys.modules[pkg + ".clip_text"]
    root = _source_root() / VC
    sys.modules.setdefault("ftfy", types.SimpleNamespace(fix_text=lambda s: s))
    sys.modules.setdefault("regex", _regex_stub())
    for name, path in ((pkg, root / "models" / "backbones" / "clip"), (pkg + "_models", root / "models")):
        m = types.ModuleType(name)
        m.__path__ = [str(path)]
        sys.modules[name] = m
    mutils = importlib.import_module(pkg + "_models.utils")
    saved = {k: sys.modules.get(k) for k in ("models", "models.utils")}
    shim = types.ModuleType("models")
    shim.__path__ = []
    shim.utils = mutils
    sys.modules["models"], sys.modules["models.utils"] = shim, mutils
    try:
        vision = importlib.import_module(pkg + ".clip_vision")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    text = importlib.import_module(pkg + ".clip_text")
    return vision, text


def criterions_source(which):
    """The source of ViCLIP's ("iv1") or InternVideo2's ("iv2") criterions.py."""
    rel = VC + "/models/criterions.py" if which == "iv1" else "InternVideo2/multi_modality/models/criterions.py"
    return (_source_root() / rel).read_text()


class FixedDropPath(nn.Module):
    """An injected DropPath draw: multiplies the [N, B, D] branch output by factor [N] (timm's shape on that layout)."""

    def __init__(self, factor):
        super().__init__()
        self.factor = factor

    def forward(self, x):
        return x * self.factor.reshape(-1, 1, 1).to(x.dtype)


def drop_path_factors(n, layers=VISION["layers"], keep=0.5, seed=77):
    """fp32 [2 * layers, n]: block 0 keeps every row (rate 0 there), later branches drop token positions with
    Bernoulli(keep) / keep, the cls position (0) of the first such branch always dropped."""
    g = torch.Generator().manual_seed(seed)
    f = torch.ones(2 * layers, n)
    for r in range(2, 2 * layers):
        f[r] = (torch.rand(n, generator=g) < keep).float() / keep
    f[2, 0] = 0.0
    return f


def weights(shape, freq):
    """Fixed loss weights of one output (a closed form, so the fixture need not store them)."""
    i = torch.arange(int(np.prod(shape)), dtype=torch.float64)
    return torch.cos(freq * i + 0.3).reshape(shape).float()


def caption_ids(V=TEXT["vocab_size"], L=TEXT["context_length"], seed=5):
    """SOT (V - 2), words, EOT (V - 1, the largest id of its row), zero padding; the EOT at a different position in each
    caption, the last slot included."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(B, L, dtype=torch.int64)
    for b, n in enumerate((3, 12, 30, 7)):
        ids[b, 0] = V - 2
        ids[b, 1:n + 1] = torch.randint(1, V - 2, (n,), generator=g)
        ids[b, n + 1] = V - 1
    return ids


def inputs(seed=3):
    g = torch.Generator().manual_seed(seed)
    r = VISION["input_resolution"]
    video = torch.randn(B, 3, T, r, r, generator=g).to(torch.bfloat16).float()
    image = torch.randn(B, 3, 1, r, r, generator=g).to(torch.bfloat16).float()
    return video, image


# ------------------------------------------------------------------------------- the restatement
def _block(x, sd, p, H, causal, f1=None, f2=None):
    """clip_vision.py:33-61 on [B, n, D]: x + dp1 * attn(ln_1(x)), x + dp2 * c_proj(QuickGELU(c_fc(ln_2(x)))).
    f1 / f2: DropPath factors per token position [n] or None."""
    Bn, n, D = x.shape
    d = D // H
    h = F.layer_norm(x, (D,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], 1e-5)
    q, k, v = (h @ sd[p + "attn.in_proj_weight"].t() + sd[p + "attn.in_proj_bias"]).reshape(Bn, n, 3, H, d) \
        .permute(2, 0, 3, 1, 4)
    s = (q * d ** -0.5) @ k.transpose(-1, -2)
    if causal:
        s = s + torch.full((n, n), float("-inf")).triu(1)
    a = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(Bn, n, D)
    a = a @ sd[p + "attn.out_proj.weight"].t() + sd[p + "attn.out_proj.bias"]
    x = x + (a if f1 is None else a * f1[None, :, None])
    h = F.layer_norm(x, (D,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], 1e-5)
    h = h @ sd[p + "mlp.c_fc.weight"].t() + sd[p + "mlp.c_fc.bias"]
    h = (h * torch.sigmoid(1.702 * h)) @ sd[p + "mlp.c_proj.weight"].t() + sd[p + "mlp.c_proj.bias"]
    return x + (h if f2 is None else h * f2[None, :, None])


def restate_vision(sd, x, kept=None, return_embed=False, factors=None, H=VISION["heads"], p=VISION["patch_size"]):
    """VisionTransformer.forward (clip_vision.py:137-177).  x [B, 3, T, H, W]; kept: int64 [B, k] kept positions of the
    `(n t)` token order (mask_tokens), None for all; factors: [2 * layers, n] DropPath factors."""
    Bn, _, Tn = x.shape[:3]
    e = F.conv3d(x, sd["conv1.weight"], stride=sd["conv1.weight"].shape[2:])      # :138
    D = e.shape[1]
    e = e.permute(0, 2, 3, 4, 1).reshape(Bn, Tn, -1, D)                          # [B, T, L, D]
    pe = sd["positional_embedding"]
    tpe = sd["temporal_positional_embedding"]
    e = e + pe[1:][None, None]                                                    # :142
    e = e + (tpe.mean(1)[:, None] if Tn == 1 else tpe[0][None, :, None])          # :149-154
    e = e.transpose(1, 2).reshape(Bn, -1, D)                                      # (n t) order, :155
    if kept is not None:
        e = torch.stack([e[b, kept[b]] for b in range(Bn)])                       # :157-158
    cls = (sd["class_embedding"] + pe[0]).expand(Bn, 1, D)
    h = torch.cat([cls, e], 1)                                                    # :160
    h = F.layer_norm(h, (D,), sd["ln_pre.weight"], sd["ln_pre.bias"], 1e-5)      # :162
    nl = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    for i in range(nl):
        f1, f2 = (None, None) if factors is None else (factors[2 * i], factors[2 * i + 1])
        h = _block(h, sd, f"transformer.resblocks.{i}.", H, False, f1, f2)
    h = F.layer_norm(h, (D,), sd["ln_post.weight"], sd["ln_post.bias"], 1e-5)    # :167
    return h if return_embed else h[:, 0] @ sd["proj"]                            # :169-174


def restate_text(sd, ids, H=TEXT["transformer_heads"], return_embed=False):
    """CLIP_TEXT.forward (clip_text.py:161-178): token embedding + position table, causal blocks, ln_final, the EOT row
    (ids.argmax) times text_projection; with return_embed every row times text_projection."""
    x = sd["token_embedding.weight"][ids] + sd["positional_embedding"]
    D = x.shape[-1]
    nl = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    for i in range(nl):
        x = _block(x, sd, f"transformer.resblocks.{i}.", H, True)
    x = F.layer_norm(x, (D,), sd["ln_final.weight"], sd["ln_final.bias"], 1e-5)
    if return_embed:
        return x @ sd["text_projection"]
    return x[torch.arange(x.shape[0]), ids.argmax(-1)] @ sd["text_projection"]


def restate_vtc(v, t, idx, temp):
    """VTC_VTM_Loss.vtc_loss on one rank (criterions.py:15-55, 64-102, 200-215): normalised rows, similarities / temp,
    targets the idx-equality mask with unit row sums, the mean of the two cross-entropies."""
    v, t = F.normalize(v, dim=-1), F.normalize(t, dim=-1)
    s = v @ t.t() / temp
    m = (idx[:, None] == idx[None, :]).float()
    m = m / m.sum(1, keepdim=True)
    return (-(F.log_softmax(s, 1) * m).sum(1).mean() - (F.log_softmax(s.t(), 1) * m).sum(1).mean()) / 2


def temp_grad_scale(v, t, idx, temp):
    """The scale of dL/dtemp for the VTC loss of restate_vtc: the sum of the magnitudes of its terms,
    (1 / temp) sum_ij |dL/ds_ij s_ij| over the logits s, in float64.  dL/dtemp is a cancelling sum of those terms (on
    the fixture about 1/50 of this scale), so an error of the embeddings moves it by that factor more, relative to
    itself, than it moves the logits; the GPU test measures its error against this scale."""
    v, t = F.normalize(v.double(), dim=-1), F.normalize(t.double(), dim=-1)
    s = (v @ t.t() / float(temp)).requires_grad_(True)
    m = (idx[:, None] == idx[None, :]).double()
    m = m / m.sum(1, keepdim=True)
    loss = (-(F.log_softmax(s, 1) * m).sum(1).mean() - (F.log_softmax(s.t(), 1) * m).sum(1).mean()) / 2
    (ds,) = torch.autograd.grad(loss, s)
    return float((ds * s.detach()).abs().sum() / float(temp))


def restate(sd, z):
    """Every stored output of the fixture from the state_dict (keys "vision_encoder." / "text_encoder." / "temp")."""
    vs = {k[len("vision_encoder."):]: v for k, v in sd.items() if k.startswith("vision_encoder.")}
    ts = {k[len("text_encoder."):]: v for k, v in sd.items() if k.startswith("text_encoder.")}
    video, image = inputs()
    kept = torch.from_numpy(z["kept"]).long()
    ids = caption_ids()
    out = {"vision_masked": restate_vision(vs, video, kept), "text": restate_text(ts, ids),
           "embed": restate_vision(vs, video, return_embed=True), "image": restate_vision(vs, image),
           "droppath": restate_vision(vs, video, factors=drop_path_factors(N_TOKENS)),
           "text_all": restate_text(ts, ids, return_embed=True)}
    out["loss_vtc"] = restate_vtc(out["vision_masked"], out["text"], torch.tensor(IDX), sd["temp"])
    return out


def total_loss(out):
    """The scalar whose gradients the fixture stores: the VTC loss plus fixed-weight sums of the other outputs (the
    text tower's every-token output among them, so its gradients are not the VTC softmax's alone)."""
    return (out["loss_vtc"] + (out["embed"] * weights(out["embed"].shape, 0.37)).sum()
            + (out["image"] * weights(out["image"].shape, 0.53)).sum()
            + (out["droppath"] * weights(out["droppath"].shape, 0.71)).sum()
            + (out["text_all"] * weights(out["text_all"].shape, 0.29)).sum())


# ------------------------------------------------------------------------------- the fixture
GRAD_SAMPLE = 1024         # gradient elements stored per parameter (all of a smaller one)


def draw_param(name, shape):
    """The fixture's value of one parameter, bf16-representable, from a generator seeded by its name alone (so the
    fixture stores names and shapes, not values): LayerNorm weights 1 + N(0, 0.1^2), biases N(0, 0.05^2), the text
    position table N(0, 0.01^2), the temporal table N(0, 0.05^2), the token table N(0, 1) (nn.Embedding's init), the
    projections N(0, 1 / rows), every other tensor N(0, 1 / fan_in)."""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    r = torch.randn(shape, generator=g)
    leaf = name.split(".")[-1]
    if ".ln" in name:
        v = 1 + 0.1 * r if leaf == "weight" else 0.05 * r
    elif leaf.endswith("bias"):
        v = 0.05 * r
    elif name == "text_encoder.positional_embedding":
        v = 0.01 * r
    elif leaf == "temporal_positional_embedding":
        v = 0.05 * r
    elif name == "text_encoder.token_embedding.weight":
        v = r
    elif leaf in ("proj", "text_projection"):
        v = r * shape[0] ** -0.5
    elif name == "temp":
        v = torch.full(shape, TEMP)
    else:
        v = r * int(np.prod(shape[1:] or (shape[-1],))) ** -0.5
    return v.to(torch.bfloat16).float()


def sample_index(numel):
    """The flat indices of a parameter whose gradient the fixture stores: all of them up to GRAD_SAMPLE, else
    GRAD_SAMPLE sorted indices drawn from a generator seeded by numel."""
    if numel <= GRAD_SAMPLE:
        return torch.arange(numel)
    g = torch.Generator().manual_seed(numel)
    return torch.randperm(numel, generator=g)[:GRAD_SAMPLE].sort().values


def sample(t):
    """The stored elements of a gradient (sample_index), as float32."""
    flat = t.detach().reshape(-1).float()
    return flat[sample_index(flat.numel()).to(flat.device)]


def build_reference():
    """The reference towers at VISION / TEXT with every parameter set by draw_param, and the temperature."""
    vision_mod, text_mod = import_viclip()
    vis = vision_mod.VisionTransformer(**VISION)
    txt = text_mod.CLIP_TEXT(**TEXT)
    with torch.no_grad():
        for prefix, m in (("vision_encoder.", vis), ("text_encoder.", txt)):
            for name, p in m.named_parameters():
                p.copy_(draw_param(prefix + name, tuple(p.shape)))
    temp = nn.Parameter(draw_param("temp", ()))
    return vis, txt, temp


def load(path=ROOT / "tests" / "golden" / "viclip.npz"):
    """(fp32 state_dict with "vision_encoder." / "text_encoder." / "temp" keys, drawn by draw_param from the names and
    shapes the fixture lists, the npz)."""
    z = np.load(path)
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {name: draw_param(name, tuple(shape)) for name, shape in cfg["params"]}
    return sd, z


def make(path=ROOT / "tests" / "golden" / "viclip.npz"):
    """Executes the unmodified reference towers on inputs() and caption_ids() and stores the outputs, the kept
    positions of the mask draw, and for every parameter its name, shape and sampled gradient (sample); the
    parameters themselves and the inputs are drawn again from their seeds where the fixture is read."""
    from oracle import ref_shim
    crit, _ = ref_shim.import_criterions()
    vis, txt, temp = build_reference()
    video, image = inputs()
    ids = caption_ids()
    vis.train()
    torch.manual_seed(MASK_SEED)
    masked = vis(video, masking_prob=MASK_P)                  # mask_tokens draws from the CPU generator
    torch.manual_seed(MASK_SEED)                              # the kept positions of that draw, for the port's check
    L = (VISION["input_resolution"] // VISION["patch_size"]) ** 2 * T
    Lm = int(MASK_P * L)
    ind = torch.argsort(torch.rand_like(torch.zeros(B, L)), dim=-1)[:, :Lm]
    keep = torch.ones(B, L, dtype=torch.bool)
    keep[torch.arange(B)[:, None], ind] = False
    kept = keep.nonzero()[:, 1].reshape(B, -1)
    text = txt(ids)
    loss_vtc = crit.VTC_VTM_Loss(False).vtc_loss(masked, text, torch.tensor(IDX), temp, all_gather=False)
    embed = vis(video, return_embed=True)
    image_out = vis(image)
    f = drop_path_factors(N_TOKENS)
    blocks = vis.transformer.resblocks
    saved = [(b.drop_path1, b.drop_path2) for b in blocks]
    for i, b in enumerate(blocks):
        b.drop_path1, b.drop_path2 = FixedDropPath(f[2 * i]), FixedDropPath(f[2 * i + 1])
    dp = vis(video)
    for b, (d1, d2) in zip(blocks, saved):
        b.drop_path1, b.drop_path2 = d1, d2
    text_all = txt(ids, return_embed=True)[0]
    out = {"loss_vtc": loss_vtc, "embed": embed, "image": image_out, "droppath": dp, "text_all": text_all}
    total_loss(out).backward()
    params = [("vision_encoder." + k, p) for k, p in vis.named_parameters()] + \
             [("text_encoder." + k, p) for k, p in txt.named_parameters()] + [("temp", temp)]
    cfg = dict(vision=VISION, text=TEXT, B=B, T=T, mask_p=MASK_P, mask_seed=MASK_SEED, idx=IDX,
               params=[[k, list(p.shape)] for k, p in params])
    blob = {"cfg": np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), "kept": kept.numpy().astype(np.int16),
            "vision_masked": masked.detach().numpy(), "text": text.detach().numpy(), "embed": embed.detach().numpy(),
            "image_out": image_out.detach().numpy(), "droppath": dp.detach().numpy(),
            "text_all": text_all.detach().numpy(), "loss_vtc": loss_vtc.detach().numpy()}
    for k, p in params:
        blob["g/" + k] = sample(p.grad).numpy()
    np.savez_compressed(path, **blob)
    print(f"viclip: loss_vtc {float(loss_vtc):.6f}, kept {tuple(kept.shape)}, {len(blob)} arrays, "
          f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    assert available(), "reference not mounted"
    make()
