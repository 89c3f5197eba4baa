"""TEST / BASELINE INFRASTRUCTURE ONLY — the oracle of InternVideo-Next's video encoder (InternVideo-Next/models).

  stage()        copies the unmodified models/InternVideo_next.py, pos_embed.py and flash_attention_class.py into the
                 git-ignored oracle/_ref/reference/ (same layout as the reference tree; __graft_entry__.build() runs
                 it), so tools/next_table.py can time the reference module on the GPU box
  import_next()  imports InternVideo_next.py unmodified as a member of a private package (models/__init__.py, which
                 pulls in transformers and ModernBERT, is never executed), behind oracle/ref_shim.py's timm and FA2
                 stand-ins
  restate()      a restatement of the encoder in functional torch (fp32 on the CPU for the fixture; the GPU tests run it
                 on the device, in fp32 and under bf16 autocast)
  make()         writes tests/golden/internvideo_next.npz by executing the unmodified reference module:
                 python oracle/internvideo_next.py

Nothing here reads the reference at import time; only tests/, tools/ and the build import this module.
"""
from __future__ import annotations

import contextlib
import importlib
import io
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
NEXT = "InternVideo-Next/models"
FILES = (NEXT + "/InternVideo_next.py", NEXT + "/pos_embed.py", NEXT + "/flash_attention_class.py")
STAGED = Path(__file__).resolve().parent / "_ref" / "reference"

# a narrow encoder with head_dim 64 (the GPU kernels' head dims): 4 cls tokens + 4 frames of 4 x 4 patches, n = 68
CFG = dict(img_size=56, patch_size=14, num_frames=4, tubelet_size=1, embed_dim=128, num_heads=2, depth=2, mlp_ratio=4,
           attn_pool_num_heads=2, clip_embed_dim=64, qkv_bias=False, init_values=1e-5, qk_normalization=True,
           drop_path_rate=0.0, cls_token_num=4)
# the naive path of the reference: plain RMSNorm blocks and nn.GELU (erf) MLPs
NAIVE = dict(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False)
B = 2


def _source_root():
    from oracle import ref_shim
    return Path(ref_shim.REF_ROOT)


def stage(verbose=True) -> bool:
    src = Path("/root/reference")
    try:
        mounted = (src / NEXT).is_dir()
    except OSError:
        mounted = False
    if not mounted:
        return (STAGED / FILES[0]).is_file()
    for rel in FILES:
        (STAGED / rel).parent.mkdir(parents=True, exist_ok=True)
        shutil.copyfile(src / rel, STAGED / rel)
    if verbose:
        print(f"internvideo_next.stage: {len(FILES)} files -> {STAGED / NEXT}")
    return True


def available() -> bool:
    return (_source_root() / FILES[0]).is_file()


def import_next():
    """The unmodified InternVideo_next module.  Its relative imports (.pos_embed, .flash_attention_class) resolve inside
    the private package; timm and FA2's rms_norm / FusedMLP come from ref_shim's stand-ins."""
    from oracle import ref_shim
    ref_shim.install_stubs()
    pkg = "_ivref_next_models"
    if pkg not in sys.modules:
        m = types.ModuleType(pkg)
        m.__path__ = [str(_source_root() / NEXT)]
        sys.modules[pkg] = m
    return importlib.import_module(pkg + ".InternVideo_next")


def build(factory=None, **kw):
    """A reference encoder (the named factory, or InternVideo2(**kw)) on its naive path, its prints silenced."""
    mod = import_next()
    with contextlib.redirect_stdout(io.StringIO()):
        if factory is not None:
            return getattr(mod, factory)(**NAIVE, **kw)
        return mod.InternVideo2(**NAIVE, **kw)


# ------------------------------------------------------------------------------- the restatement
def _rms(x, w, eps=1e-6):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def block(h, sd, p, num_heads):
    """Block.forward (InternVideo_next.py:282-300, the unfused form) on h [B, n, D] with the tensors sd[p + ...]:
    h + ls1 * attn(norm1(h)), then + ls2 * mlp(norm2(.)), q/k RMSNorm over all heads, erf GELU."""
    Bn, n, D = h.shape
    d = D // num_heads
    a = _rms(h, sd[p + "norm1.weight"])
    qkv = a @ sd[p + "attn.qkv.weight"].t()
    if p + "attn.qkv.bias" in sd:
        qkv = qkv + sd[p + "attn.qkv.bias"]
    q, k, vv = qkv.split(D, -1)
    if p + "attn.q_norm.weight" in sd:
        q, k = _rms(q, sd[p + "attn.q_norm.weight"]), _rms(k, sd[p + "attn.k_norm.weight"])
    q, k, vv = (z.reshape(Bn, n, num_heads, d).transpose(1, 2) for z in (q, k, vv))
    s = torch.softmax((q * d ** -0.5) @ k.transpose(-1, -2), -1)
    a = (s @ vv).transpose(1, 2).reshape(Bn, n, D) @ sd[p + "attn.proj.weight"].t() + sd[p + "attn.proj.bias"]
    h = h + (a * sd[p + "ls1.gamma"] if p + "ls1.gamma" in sd else a)
    a = _rms(h, sd[p + "norm2.weight"]) @ sd[p + "mlp.fc1.weight"].t() + sd[p + "mlp.fc1.bias"]
    a = F.gelu(a) @ sd[p + "mlp.fc2.weight"].t() + sd[p + "mlp.fc2.bias"]
    return h + (a * sd[p + "ls2.gamma"] if p + "ls2.gamma" in sd else a)


def restate(sd, x, projected=False, num_heads=CFG["num_heads"], pool_heads=CFG["attn_pool_num_heads"],
            patch=CFG["patch_size"], tubelet=CFG["tubelet_size"], cls_token_num=CFG["cls_token_num"]):
    """InternVideo2.forward (InternVideo_next.py:496-538) in functional torch on sd's tensors (any dtype and device).
    x [B, C, T, H, W]."""
    Bn, C, T, H, W = x.shape
    P, t = patch, tubelet
    f, gh, gw = T // t, H // P, W // P
    # PatchEmbed (:332-342): norm_before over each patch's (t hp wp c) vector, the Conv3d, norm over D
    v = x.permute(0, 2, 3, 4, 1).reshape(Bn, f, t, gh, P, gw, P, C).permute(0, 1, 3, 5, 2, 4, 6, 7)
    v = _rms(v.reshape(Bn, f * gh * gw, t * P * P * C), sd["patch_embed.norm_before.weight"])
    v = v.reshape(Bn, f * gh * gw, t, P, P, C)
    w = sd["patch_embed.proj.weight"]                                       # [D, C, t, P, P]
    e = torch.einsum("bnzyxc,dczyx->bnd", v, w) + sd["patch_embed.proj.bias"]
    e = _rms(e, sd["patch_embed.norm.weight"])
    h = torch.cat([sd["cls_token"].expand(Bn, -1, -1), e], 1) + sd["pos_embed"]
    depth = len({k.split(".")[1] for k in sd if k.startswith("blocks.")})
    D = h.shape[-1]
    for i in range(depth):
        h = block(h, sd, f"blocks.{i}.", num_heads)
    if not projected:
        return h[:, cls_token_num:]
    # AttentionPoolingBlock (:84-117): one query, the mean token
    c = "clip_projector."
    ln = lambda z, nm: F.layer_norm(z, (D,), sd[c + nm + ".weight"], sd[c + nm + ".bias"], 1e-5)  # noqa: E731
    xq, xk, xv = ln(h.mean(1, keepdim=True), "norm1_q"), ln(h, "norm1_k"), ln(h, "norm1_v")
    ca = c + "cross_attn."
    q = xq @ sd[ca + "q.weight"].t() + sd[ca + "q_bias"]
    k = xk @ sd[ca + "k.weight"].t() + sd[ca + "k_bias"]
    vv = xv @ sd[ca + "v.weight"].t() + sd[ca + "v_bias"]
    dp = D // pool_heads
    q, k, vv = (z.reshape(Bn, -1, pool_heads, dp).transpose(1, 2) for z in (q, k, vv))
    s = torch.softmax((q * dp ** -0.5) @ k.transpose(-1, -2), -1)
    o = (s @ vv).transpose(1, 2).reshape(Bn, 1, D)
    return (o @ sd[ca + "proj.weight"].t() + sd[ca + "proj.bias"]).squeeze(1)


def weights(shape, freq):
    """Fixed loss weights of one output (a closed form, so the fixture need not store them)."""
    i = torch.arange(int(np.prod(shape)), dtype=torch.float64)
    return torch.cos(freq * i + 0.3).reshape(shape).float()


def total_loss(tokens, pooled):
    """The scalar whose gradients the fixture stores: fixed-weight sums of both outputs."""
    return (tokens.float() * weights(tokens.shape, 0.37).to(tokens.device)).sum() + \
        (pooled.float() * weights(pooled.shape, 0.53).to(pooled.device)).sum()


# ------------------------------------------------------------------------------- the fixture
GRAD_SAMPLE = 1024         # gradient elements stored per parameter (all of a smaller one)


def draw_param(name, shape):
    """The fixture's value of one parameter, bf16-representable, from a generator seeded by its name alone (so the
    fixture stores names and shapes, not values): norm weights 1 + N(0, 0.1^2), biases N(0, 0.05^2), LayerScale gammas
    0.1 (1 + N(0, 0.25^2)) (the recipe's 1e-5 would hide the blocks), cls tokens and the position table N(0, 0.25),
    every other tensor N(0, 1 / fan_in)."""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    r = torch.randn(shape, generator=g)
    leaf = name.split(".")[-1]
    if leaf == "gamma":
        v = 0.1 * (1 + 0.25 * r)
    elif "norm" in name and leaf == "weight":
        v = 1 + 0.1 * r
    elif leaf.endswith("bias"):
        v = 0.05 * r
    elif leaf in ("cls_token", "pos_embed"):
        v = 0.5 * r
    else:
        v = r * int(np.prod(shape[1:])) ** -0.5
    return v.to(torch.bfloat16).float()


def sample_index(numel):
    if numel <= GRAD_SAMPLE:
        return torch.arange(numel)
    g = torch.Generator().manual_seed(numel)
    return torch.randperm(numel, generator=g)[:GRAD_SAMPLE].sort().values


def sample(t):
    """The stored elements of a gradient (sample_index), as float32."""
    flat = t.detach().reshape(-1).float()
    return flat[sample_index(flat.numel()).to(flat.device)]


def video(seed=3):
    """The fixture's input: bf16-representable, with a per-patch scale that varies across the frame so that
    norm_before matters."""
    g = torch.Generator().manual_seed(seed)
    r = CFG["img_size"]
    x = torch.randn(B, 3, CFG["num_frames"], r, r, generator=g)
    x = x * (0.25 + torch.rand(B, 1, CFG["num_frames"], r // 14, 1, r // 14, 1, generator=g).expand(
        -1, -1, -1, -1, 14, -1, 14).reshape(B, 1, CFG["num_frames"], r, r))
    return x.to(torch.bfloat16).float()


def state_dict(names_shapes):
    return {name: draw_param(name, tuple(shape)) for name, shape in names_shapes}


def load(path=ROOT / "tests" / "golden" / "internvideo_next.npz"):
    """(fp32 state_dict drawn by draw_param from the names and shapes the fixture lists, the npz)."""
    z = np.load(path)
    cfg = json.loads(bytes(z["cfg"]).decode())
    return state_dict(cfg["params"]), z


def make(path=ROOT / "tests" / "golden" / "internvideo_next.npz"):
    """Executes the unmodified reference encoder on video() with every parameter set by draw_param, and stores both
    outputs and, for every parameter, its name, shape and sampled gradient of total_loss."""
    model = build(**CFG)
    with torch.no_grad():
        for name, p in model.named_parameters():
            p.copy_(draw_param(name, tuple(p.shape)))
    x = video()
    tokens = model(x)
    pooled = model(x, projected=True)
    total_loss(tokens, pooled).backward()
    params = list(model.named_parameters())
    cfg = dict(model=CFG, B=B, params=[[k, list(p.shape)] for k, p in params])
    blob = {"cfg": np.frombuffer(json.dumps(cfg).encode(), dtype=np.uint8), "tokens": tokens.detach().numpy(),
            "pooled": pooled.detach().numpy()}
    for k, p in params:
        blob["g/" + k] = sample(p.grad).numpy()
    np.savez_compressed(path, **blob)
    print(f"internvideo_next: tokens {tuple(tokens.shape)}, pooled {tuple(pooled.shape)}, {len(blob)} arrays, "
          f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    assert available(), "reference not mounted"
    make()
