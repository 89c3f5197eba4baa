"""TEST / BASELINE INFRASTRUCTURE ONLY — the oracle of InternVideo-MM (InternVideo1/Pretrain/Multi-Modalities-Pretraining).

  stage()      copies the unmodified clip_utils/model.py, clip_utils/utils/{clip_vit_only_global,attention,
               attention_module}.py and the two packages' __init__.py into the git-ignored oracle/_ref/reference/ (same
               layout as the reference tree; __graft_entry__.build() runs it), so tools/mm_table.py can time the
               reference modules on the GPU box
  import_mm()  imports model.py and the utils package unmodified, under a private stub parent package: the real
               clip_utils/__init__.py (clip.py: PIL, torchvision, tqdm) and InternVideo/__init__.py (decord,
               torchvision) are never executed; timm comes from oracle/ref_shim.py's stand-in
  restate()    a CPU fp32 restatement of both towers, the extractor and the zero-shot probabilities in functional torch
  make()       writes tests/golden/internvideo_mm.npz by executing the unmodified reference modules:
               python oracle/internvideo_mm.py

Nothing here reads the reference at import time; only tests/, tools/ and the build import this module.
"""
from __future__ import annotations

import importlib
import json
import os
import shutil
import sys
import types
import zlib
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
MM = "InternVideo1/Pretrain/Multi-Modalities-Pretraining/InternVideo/clip_utils"
FILES = (MM + "/__init__.py", MM + "/model.py", MM + "/utils/__init__.py", MM + "/utils/clip_vit_only_global.py",
         MM + "/utils/attention.py", MM + "/utils/attention_module.py")
STAGED = Path(__file__).resolve().parent / "_ref" / "reference"

# narrow towers with head_dim 64, so the GPU kernels apply: a 4 x 4 grid of 14-pixel patches, 4 frames, extractor taps
# after backbone layers 2 and 3
NARROW = "vit_only_global_narrow"
VISION = dict(input_resolution=56, patch_size=14, width=128, layers=4, heads=2, output_dim=64)
MODEL = dict(embed_dim=64, vision_width=128, context_length=16, vocab_size=512, transformer_width=128,
             transformer_heads=2, transformer_layers=2, n_layers=2, n_dim=128, n_head=2, t_size=4,
             mlp_dropout=[0.5, 0.5], backbone=NARROW, return_list=[2, 3])
B, T = 2, 4
EOT_AT = (3, 8, 15, 1)                      # the EOT of each caption: the last slot and a one-word caption included
MASKED = ((0, 2), (1, 5), (1, 6), (2, 9))   # (caption, position) rows replaced by text_mask_embedding
N_CAND = 3                                  # the demo's three captions: the first three


def _source_root():
    from oracle import ref_shim
    return Path(ref_shim.REF_ROOT)


def stage(verbose=True) -> bool:
    src = Path("/root/reference")
    try:
        mounted = (src / MM).is_dir()
    except OSError:
        mounted = False
    if not mounted:
        return (STAGED / FILES[1]).is_file()
    for rel in FILES:
        (STAGED / rel).parent.mkdir(parents=True, exist_ok=True)
        shutil.copyfile(src / rel, STAGED / rel)
    if verbose:
        print(f"internvideo_mm.stage: {len(FILES)} files -> {STAGED / MM}")
    return True


def available() -> bool:
    return (_source_root() / FILES[1]).is_file()


def import_mm():
    """(model module, utils package) of the unmodified reference, with the narrow backbone registered in the utils
    package's namespace (register_narrow), where VideoIntern looks backbones up by name."""
    from oracle import ref_shim
    ref_shim.install_stubs()
    pkg = "_ivref_mm_clip_utils"
    if pkg + ".model" not in sys.modules:
        m = types.ModuleType(pkg)
        m.__path__ = [str(_source_root() / MM)]
        sys.modules[pkg] = m
        importlib.import_module(pkg + ".utils")
        importlib.import_module(pkg + ".model")
    utils = sys.modules[pkg + ".utils"]
    register_narrow(utils, utils.clip_vit_only_global.VisionTransformer)
    return sys.modules[pkg + ".model"], utils


def register_narrow(namespace, vision_cls):
    """Registers the fixture's narrow backbone factory (VISION) as NARROW in a backbone namespace (the reference's
    utils package, or internvideo_mm.BACKBONES): the factories of the reference hard-code their widths.  VideoIntern
    does not pass n_layers on; like the reference's factories, the narrow one defaults it to its return_list's length."""
    def narrow(pretrained=False, n_layers=len(MODEL["return_list"]), **kw):
        return vision_cls(**VISION, n_layers=n_layers, **kw).eval()
    if isinstance(namespace, dict):
        namespace[NARROW] = narrow
    else:
        setattr(namespace, NARROW, narrow)


# ------------------------------------------------------------------------------- parameters and inputs
def draw_param(name, shape):
    """The fixture's value of one parameter, bf16-representable, from a generator seeded by its name alone: LayerNorm
    weights 1 + N(0, 0.1^2), biases N(0, 0.05^2), the dpe weights N(0, 0.2^2) (the reference zero-inits their bias, the
    extractor's out_proj and c_proj, balance and temporal_cls_token; drawn here, a fixture at init would pass an
    extractor that did nothing), balance N(0, 1), temporal_cls_token N(0, 0.5^2), the text position table and mask
    embedding N(0, 0.01^2) / N(0, 0.02^2), the token table N(0, 1), logit_scale log(1 / 0.07), the projections
    N(0, 1 / rows), every other tensor N(0, 1 / fan_in)."""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    r = torch.randn(shape, generator=g)
    leaf = name.split(".")[-1]
    if ".ln" in name or name.startswith("ln_") or name.startswith("visual_ln"):
        v = 1 + 0.1 * r if leaf == "weight" else 0.05 * r
    elif ".dpe." in name and leaf == "weight":
        v = 0.2 * r
    elif leaf.endswith("bias"):
        v = 0.05 * r
    elif leaf == "balance":
        v = r
    elif leaf == "temporal_cls_token":
        v = 0.5 * r
    elif name == "positional_embedding":
        v = 0.01 * r
    elif name == "text_mask_embedding":
        v = 0.02 * r
    elif name == "token_embedding.weight":
        v = r
    elif name == "logit_scale":
        v = torch.full(shape, float(np.log(1 / 0.07)))
    elif leaf in ("visual_proj", "text_projection"):
        v = r * shape[0] ** -0.5
    else:
        v = r * int(np.prod(shape[1:] or (shape[-1],))) ** -0.5
    return v.to(torch.bfloat16).float()


def caption_ids(V=MODEL["vocab_size"], L=MODEL["context_length"], seed=5):
    """SOT (V - 2), words, EOT (V - 1, the largest id of its row) at EOT_AT, zero padding."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(len(EOT_AT), L, dtype=torch.int64)
    for b, e in enumerate(EOT_AT):
        ids[b, 0] = V - 2
        ids[b, 1:e] = torch.randint(1, V - 2, (e - 1,), generator=g)
        ids[b, e] = V - 1
    return ids


def text_mask():
    m = torch.zeros(len(EOT_AT), MODEL["context_length"], dtype=torch.bool)
    for b, l in MASKED:
        m[b, l] = True
    return m


def inputs(seed=3):
    """(video [B, 3, T, 56, 56], one-frame clips [B, 3, 1, 56, 56]), bf16-representable."""
    g = torch.Generator().manual_seed(seed)
    r = VISION["input_resolution"]
    video = torch.randn(B, 3, T, r, r, generator=g).to(torch.bfloat16).float()
    image = torch.randn(B, 3, 1, r, r, generator=g).to(torch.bfloat16).float()
    return video, image


# ------------------------------------------------------------------------------- the restatement
def dpe_ln(x, w, b, lw, lb, N, T, Hg, Wg, eps=1e-5):
    """clip_vit_only_global.py:221-231 and Extractor :147: x [N*T*(1 + Hg*Wg), C] -> ln_3 of each patch token plus its
    depthwise 3x3x3 conv (zero padded), and ln_3 of each frame's cls token; any float dtype."""
    C = x.shape[1]
    L = 1 + Hg * Wg
    v = x.reshape(N, T, L, C)
    p = v[:, :, 1:].reshape(N, T, Hg, Wg, C).permute(0, 4, 1, 2, 3)
    conv = F.conv3d(p, w, b, padding=1, groups=C).permute(0, 2, 3, 4, 1).reshape(N, T, L - 1, C)
    y = torch.cat([v[:, :, :1], v[:, :, 1:] + conv], 2).reshape(-1, C)
    return F.layer_norm(y, (C,), lw, lb, eps)


def extractor(cls, keys, sd, p, H):
    """Extractor.forward (:124-149) with ln_3 already applied: cls [N, C], keys [N, n, C]."""
    N, C = cls.shape
    d = C // H
    w, b = sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"]
    q = F.layer_norm(cls, (C,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], 1e-5) @ w[:C].t() + b[:C]
    k = keys @ w[C:2 * C].t() + b[C:2 * C]
    v = keys @ w[2 * C:].t() + b[2 * C:]
    q = q.reshape(N, H, 1, d)
    k = k.reshape(N, -1, H, d).transpose(1, 2)
    v = v.reshape(N, -1, H, d).transpose(1, 2)
    a = (torch.softmax(q @ k.transpose(-1, -2) / d ** 0.5, -1) @ v).reshape(N, C)
    x = cls + a @ sd[p + "attn.out_proj.weight"].t() + sd[p + "attn.out_proj.bias"]
    h = F.layer_norm(x, (C,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], 1e-5)
    h = h @ sd[p + "mlp.c_fc.weight"].t() + sd[p + "mlp.c_fc.bias"]
    return x + (h * torch.sigmoid(1.702 * h)) @ sd[p + "mlp.c_proj.weight"].t() + sd[p + "mlp.c_proj.bias"]


def restate_video(sd, x, T_down, return_list=MODEL["return_list"], H=VISION["heads"]):
    """VideoIntern.encode_video (model.py:202-218, clip_vit_only_global.py:203-286): x [N, 3, T, H, W] ->
    (features [N, embed_dim], the stream [L, N, T_down, C])."""
    from oracle.viclip import _block
    vs = {k[len("visual."):]: v for k, v in sd.items() if k.startswith("visual.")}
    Nn, _, Tn = x.shape[:3]
    e = F.conv3d(x, vs["conv1.weight"], stride=vs["conv1.weight"].shape[2:])
    C, Hg, Wg = e.shape[1], e.shape[3], e.shape[4]
    e = e.permute(0, 2, 3, 4, 1).reshape(Nn * Tn, Hg * Wg, C)
    h = torch.cat([vs["class_embedding"].expand(Nn * Tn, 1, C), e], 1) + vs["positional_embedding"]
    h = F.layer_norm(h, (C,), vs["ln_pre.weight"], vs["ln_pre.bias"], 1e-5)       # [NT, L, C]
    N, L = Nn * Tn // T_down, h.shape[1]
    cls = vs["transformer.temporal_cls_token"].reshape(1, C).expand(N, C)
    nl = len({k.split(".")[2] for k in vs if k.startswith("transformer.resblocks.")})
    j = -1
    for i in range(nl):
        h = _block(h, vs, f"transformer.resblocks.{i}.", H, False)
        if i in return_list:
            j += 1
            p = f"transformer.dec.{j}."
            keys = dpe_ln(h.reshape(-1, C), vs[f"transformer.dpe.{j}.weight"], vs[f"transformer.dpe.{j}.bias"],
                          vs[p + "ln_3.weight"], vs[p + "ln_3.bias"], N, T_down, Hg, Wg)
            cls = extractor(cls, keys.reshape(N, T_down * L, C), vs, p, H)
    w = torch.sigmoid(vs["transformer.balance"])
    feats = (1 - w) * cls + w * h.reshape(N, T_down, L, C)[:, :, 0].mean(1)
    out = F.layer_norm(feats, (C,), sd["visual_ln_post.weight"], sd["visual_ln_post.bias"], 1e-5) @ sd["visual_proj"]
    return out, h.reshape(N, T_down, L, C).permute(2, 0, 1, 3)


def restate_text(sd, ids, mask=None, H=MODEL["transformer_heads"]):
    """VideoIntern.encode_text (model.py:220-245): -> (features [B, embed_dim], ln_final of every token)."""
    from oracle.viclip import _block
    x = sd["token_embedding.weight"][ids]
    if mask is not None:
        x = x.clone()
        x[mask] = sd["text_mask_embedding"].reshape(-1)
    x = x + sd["positional_embedding"]
    D = x.shape[-1]
    for i in range(MODEL["transformer_layers"]):
        x = _block(x, sd, f"transformer.resblocks.{i}.", H, True)
    x = F.layer_norm(x, (D,), sd["ln_final.weight"], sd["ln_final.bias"], 1e-5)
    return x[torch.arange(x.shape[0]), ids.argmax(-1)] @ sd["text_projection"], x


def zero_shot(v, t, logit_scale):
    """demo.py:12-19: softmax over the captions of the scaled cosine similarities."""
    v, t = F.normalize(v, dim=1), F.normalize(t, dim=1)
    return (v @ t.t() * logit_scale.exp()).softmax(dim=-1)


def restate(sd):
    """Every stored output of the fixture from the state_dict and the fixed inputs."""
    video, image = inputs()
    ids = caption_ids()
    out = {}
    out["video"], stream = restate_video(sd, video, T)
    out["image"], _ = restate_video(sd, image, 1)
    out["stream"] = stream
    out["text"], out["text_all"] = restate_text(sd, ids)
    out["text_masked"], _ = restate_text(sd, ids, text_mask())
    out["probs"] = zero_shot(out["video"], out["text"][:N_CAND], sd["logit_scale"])
    return out


# ------------------------------------------------------------------------------- the fixture
def build_reference():
    """The reference VideoIntern at MODEL, every parameter set by draw_param."""
    model_mod, _ = import_mm()
    m = model_mod.VideoIntern(**MODEL)
    with torch.no_grad():
        for name, p in m.named_parameters():
            p.copy_(draw_param(name, tuple(p.shape)))
    return m.eval()


def load(path=ROOT / "tests" / "golden" / "internvideo_mm.npz"):
    """(fp32 state_dict drawn by draw_param from the names and shapes the fixture lists, in its order; the npz)."""
    z = np.load(path)
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {name: draw_param(name, tuple(shape)) for name, shape in cfg["params"]}
    return sd, z


def make(path=ROOT / "tests" / "golden" / "internvideo_mm.npz"):
    """Executes the unmodified reference VideoIntern on inputs(), caption_ids() and text_mask() and stores the inputs,
    the outputs, and the name and shape of every parameter in state_dict order.  The parameter values are draw_param's
    of those names (1.6 M of them would make a 3 MB fixture), so load() rebuilds the state_dict bit for bit."""
    m = build_reference()
    video, image = inputs()
    ids = caption_ids()
    with torch.no_grad():
        v = m.encode_video(video)
        img = m.encode_video(image, mode="image")
        v_all, stream = m.encode_video(video, return_all_feats=True)
        txt, txt_all = m.encode_text(ids, return_all_feats=True)
        txt_masked = m.encode_text(ids, masked_indices=text_mask())
        probs = zero_shot(v, txt[:N_CAND], m.logit_scale)
    assert torch.equal(v, v_all)
    sd = m.state_dict()
    cfg = dict(model=MODEL, vision=VISION, B=B, T=T, eot_at=EOT_AT, masked=MASKED,
               params=[[k, list(t.shape)] for k, t in sd.items()])
    bits = lambda t: t.to(torch.bfloat16).view(torch.int16).numpy()
    blob = {"cfg": np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), "video_in": bits(video),
            "image_in": bits(image), "ids": ids.numpy(), "mask": text_mask().numpy(),
            "video": v.numpy(), "image": img.numpy(), "stream": stream.numpy(), "text": txt.numpy(),
            "text_all": txt_all.numpy(), "text_masked": txt_masked.numpy(), "probs": probs.numpy()}
    np.savez_compressed(path, **blob)
    print(f"internvideo_mm: probs {probs.numpy().round(4).tolist()}, {len(blob)} arrays, {os.path.getsize(path)} bytes")


def stored_inputs(z):
    f = lambda k: torch.from_numpy(z[k].copy()).view(torch.bfloat16).float()
    return f("video_in"), f("image_in")


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    assert available(), "reference not mounted"
    make()
