"""TEST INFRASTRUCTURE ONLY — CPU restatement (the parity oracle) of the reference's hot path.

Plain functional torch (fp32 unless the caller passes fp64) over a `state_dict`-keyed dict of
tensors; no nn.Module, no CUDA, no dependency on /root/reference.  Every function cites the
reference lines it restates (paths relative to /root/reference).  The restatement is PINNED by
tests/test_oracle_cpu.py against (a) golden vectors produced by executing the unmodified reference
modules (oracle/make_golden.py -> tests/golden/*.npz) and (b) the live reference when it is mounted.
The reference itself ships no golden vectors or tests for this path (SURVEY.md §4, §8c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline/reference legs may import this.
The product (internvideo_b200/) never does.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

SM = "InternVideo2/single_modality/models/internvideo2_pretrain.py"


# ------------------------------------------------------------------------------------ elementary
def rmsnorm(x, weight, eps=1e-6):
    """RMSNorm.forward — {SM}:123-128 (fp32 statistics, weight applied after the cast back)."""
    dt = x.dtype
    h = x.to(torch.float32)
    var = h.pow(2).mean(-1, keepdim=True)
    h = h * torch.rsqrt(var + eps)
    return weight * h.to(dt)


def layernorm(x, weight, bias, eps=1e-5):
    """nn.LayerNorm(eps=1e-5) used by AttentionPoolingBlock / decoders — {SM}:525,532."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * weight + bias


def gelu(x, approximate="none"):
    """nn.GELU (erf) in Mlp {SM}:224,233; tanh form = FA2 FusedMLP (SURVEY §0 fact 2)."""
    if approximate == "tanh":
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


def linear(x, w, b=None):
    y = x @ w.t()
    return y if b is None else y + b


# ------------------------------------------------------------------------------------ patch embed
def patch_embed(x, w, b, tubelet=1, patch=14):
    """PatchEmbed.forward — {SM}:327-331: Conv3d(k=s=(tubelet,p,p)) then flatten(3).permute(0,2,3,1).

    Restated as an explicit im2col GEMM: tokens ordered (t, h, w); each token's K axis ordered
    (c, dt, dy, dx) exactly like the Conv3d weight [D, C, tubelet, p, p] flattened.
    Returns [B, T', L, D].
    """
    B, C, T, H, W = x.shape
    Tt, Hh, Ww = T // tubelet, H // patch, W // patch
    cols = x.reshape(B, C, Tt, tubelet, Hh, patch, Ww, patch)
    cols = cols.permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(B, Tt, Hh * Ww, C * tubelet * patch * patch)
    return cols @ w.reshape(w.shape[0], -1).t() + b


def visible_indices(mask):
    """Order-preserving compaction indices of `x[~mask]` — {SM}:659.  mask [B, N] bool, True = masked.

    Returns int64 [B, n] (n = number of visible tokens per clip, equal across the batch).
    """
    B, N = mask.shape
    vis = ~mask
    n = int(vis[0].sum())
    idx = torch.empty(B, n, dtype=torch.int64)
    for bi in range(B):
        nz = torch.nonzero(vis[bi], as_tuple=False).flatten()
        assert nz.numel() == n, "every clip must keep the same number of tokens (reshape at :659)"
        idx[bi] = nz
    return idx


def embed_tokens(p, x, mask, tubelet=1, patch=14):
    """{SM}:630-659 — patch embed, cls cat, + pos_embed, boolean compaction."""
    t = patch_embed(x, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], tubelet, patch)
    B, T, L, C = t.shape
    t = t.reshape(B, T * L, C)
    t = torch.cat([p["cls_token"].expand(B, -1, -1), t], dim=1) + p["pos_embed"]
    idx = visible_indices(mask)
    return torch.gather(t, 1, idx[:, :, None].expand(-1, -1, C)), idx


# ------------------------------------------------------------------------------------ block
def attention(p, pre, x, num_heads, qk_norm=True):
    """Attention._naive_attn — {SM}:173-191 (q/k RMSNorm over the flattened H*d, :178-181)."""
    B, N, C = x.shape
    d = C // num_heads
    qkv = linear(x, p[pre + "qkv.weight"], p.get(pre + "qkv.bias"))
    q, k, v = qkv.reshape(B, N, 3, C).unbind(2)
    if qk_norm:
        q = rmsnorm(q, p[pre + "q_norm.weight"])
        k = rmsnorm(k, p[pre + "k_norm.weight"])
    q = q.reshape(B, N, num_heads, d).transpose(1, 2)
    k = k.reshape(B, N, num_heads, d).transpose(1, 2)
    v = v.reshape(B, N, num_heads, d).transpose(1, 2)
    attn = ((q * d ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    o = (attn @ v).transpose(1, 2).reshape(B, N, C)
    return linear(o, p[pre + "proj.weight"], p[pre + "proj.bias"])


def mlp(p, pre, x, gelu_mode="none"):
    """Mlp.forward — {SM}:238-244."""
    h = gelu(linear(x, p[pre + "fc1.weight"], p[pre + "fc1.bias"]), gelu_mode)
    return linear(h, p[pre + "fc2.weight"], p[pre + "fc2.bias"])


def block(p, i, x, num_heads, gelu_mode="none", drop_path=None, qk_norm=True):
    """Block.forward naive branch — {SM}:290-291 (LayerScale fp32 :139-143).
    drop_path: None (eval / rate 0) or (f1, f2), per-sample factors [B] = Bernoulli(keep)/keep that timm's
    DropPath multiplies the attention / MLP branch with in training ({SM}:264,274).
    qk_norm: the block's qk_normalization (the q/k RMSNorms, {SM}:178-181); False skips them."""
    pre = f"blocks.{i}."
    a = attention(p, pre + "attn.", rmsnorm(x, p[pre + "norm1.weight"]), num_heads, qk_norm)
    if pre + "ls1.gamma" in p:
        a = a * p[pre + "ls1.gamma"]
    if drop_path is not None:
        a = a * drop_path[0][:, None, None]
    x = x + a
    m = mlp(p, pre + "mlp.", rmsnorm(x, p[pre + "norm2.weight"]), gelu_mode)
    if pre + "ls2.gamma" in p:
        m = m * p[pre + "ls2.gamma"]
    if drop_path is not None:
        m = m * drop_path[1][:, None, None]
    return x + m


# ------------------------------------------------------------------------------------ heads
def attention_pool(p, x, num_heads, pre="clip_projector."):
    """AttentionPoolingBlock — {SM}:107-114 over AttentiveBlock :98-104 and CrossAttention :50-80."""
    B, N, C = x.shape
    d = C // num_heads
    xq = layernorm(x.mean(1, keepdim=True), p[pre + "norm1_q.weight"], p[pre + "norm1_q.bias"])
    xk = layernorm(x, p[pre + "norm1_k.weight"], p[pre + "norm1_k.bias"])
    xv = layernorm(x, p[pre + "norm1_v.weight"], p[pre + "norm1_v.bias"])
    ca = pre + "cross_attn."
    q = linear(xq, p[ca + "q.weight"], p.get(ca + "q_bias")).reshape(B, 1, num_heads, d).transpose(1, 2)
    k = linear(xk, p[ca + "k.weight"], p.get(ca + "k_bias")).reshape(B, N, num_heads, d).transpose(1, 2)
    v = linear(xv, p[ca + "v.weight"], p.get(ca + "v_bias")).reshape(B, N, num_heads, d).transpose(1, 2)
    attn = ((q * d ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    o = (attn @ v).transpose(1, 2).reshape(B, 1, C)
    return linear(o, p[ca + "proj.weight"], p[ca + "proj.bias"]).squeeze(1)


def l2n(x):
    """x / x.norm(dim=-1, keepdim=True) — no eps ({SM}:359,397)."""
    return x / x.norm(dim=-1, keepdim=True)


def linear_decoder(p, pre, x):
    """Linear_Decoder.forward — {SM}:355-365."""
    return l2n(layernorm(linear(x, p[pre + "head.weight"], p[pre + "head.bias"]),
                         p[pre + "norm.weight"], p[pre + "norm.bias"]))


def mlp_decoder(p, pre, x):
    """MLP_Decoder.forward — {SM}:393-403 (Linear, GELU(erf), Linear, LayerNorm, L2)."""
    h = gelu(linear(x, p[pre + "head.0.weight"], p[pre + "head.0.bias"]))
    h = linear(h, p[pre + "head.2.weight"], p[pre + "head.2.bias"])
    return l2n(layernorm(h, p[pre + "norm.weight"], p[pre + "norm.bias"]))


# ------------------------------------------------------------------------------------ full forward
def forward_pretrain(p, cfg, x, mask, gelu_mode="none", return_hidden=False, drop_path=None):
    """PretrainInternVideo2.forward — {SM}:629-744 (joint pos-embed branch, naive blocks).

    cfg: dict(depth, num_heads, attn_pool_num_heads, patch_size, tubelet_size,
              clip_return_index [list], mae_return_index [list]).
    drop_path: optional [2*depth, B] per-sample DropPath factors (rows 2i / 2i+1 = block i's two branches).
    Returns (x_clip_align [K,B,n,Ct], x_align [B,Cf], x_mae_align [K',B,n-1,Cm]).
    """
    h, idx = embed_tokens(p, x, mask, cfg.get("tubelet_size", 1), cfg["patch_size"])
    B, n, C = h.shape
    x_clip, x_mae = [], []
    hidden = [h]
    for i in range(cfg["depth"]):
        h = block(p, i, h, cfg["num_heads"], gelu_mode,
                  None if drop_path is None else (drop_path[2 * i], drop_path[2 * i + 1]))
        hidden.append(h)
        if i in cfg["clip_return_index"]:
            x_clip.append(h)
        if i in cfg["mae_return_index"]:
            x_mae.append(h[:, 1:])
    pooled = attention_pool(p, h, cfg["attn_pool_num_heads"])
    # CLIP branch: + clip_pos_embed[~mask] (:712-714), per-layer Linear_Decoder (:716-719)
    cpe = torch.gather(p["clip_pos_embed"].expand(B, -1, -1), 1, idx[:, :, None].expand(-1, -1, C))
    x_clip_align = torch.stack([linear_decoder(p, f"clip_decoder.{k}.", xc + cpe)
                                for k, xc in enumerate(x_clip)])
    if "final_clip_decoder.head.weight" in p:
        x_align = linear_decoder(p, "final_clip_decoder.", pooled)
    else:
        x_align = pooled
    # MAE branch: mae_pos_embed[~mask[:,1:]] (:735-737); cls is always visible so idx[:,1:]-1
    midx = idx[:, 1:] - 1
    mpe = torch.gather(p["mae_pos_embed"].expand(B, -1, -1), 1, midx[:, :, None].expand(-1, -1, C))
    x_mae_align = torch.stack([mlp_decoder(p, f"mae_decoder.{k}.", xm + mpe)
                               for k, xm in enumerate(x_mae)])
    if return_hidden:
        return x_clip_align, x_align, x_mae_align, hidden, pooled
    return x_clip_align, x_align, x_mae_align


MMV = "InternVideo2/multi_modality/models/backbones/internvideo2/internvideo2_clip_vision.py"


def forward_clip_tower(p, cfg, x, use_image=False, pre=""):
    """InternVideo2.forward (unmasked CLIP / stage-2 tower) — {MMV}:497-548, joint position table.
    x [B,C,T,H,W]; cfg: dict(depth, num_heads, attn_pool_num_heads, patch_size, tubelet_size, num_frames).
    use_image: the temporal mean of the position table is used for single frames (:524-527).
    Returns the pooled [B, clip_embed_dim] features."""
    t = patch_embed(x, p[pre + "patch_embed.proj.weight"], p[pre + "patch_embed.proj.bias"],
                    cfg.get("tubelet_size", 1), cfg["patch_size"])
    B, T, L, C = t.shape
    t = torch.cat([p[pre + "cls_token"].expand(B, -1, -1), t.reshape(B, T * L, C)], dim=1)
    pe = p[pre + "pos_embed"]
    if use_image:
        Tm = cfg["num_frames"] // cfg.get("tubelet_size", 1)
        pe = torch.cat([pe[:, :1], pe[:, 1:].view(1, Tm, L, C).mean(dim=1)], dim=1)
    h = t + pe
    q = {k[len(pre):]: v for k, v in p.items() if k.startswith(pre)} if pre else p
    for i in range(cfg["depth"]):
        h = block(q, i, h, cfg["num_heads"], cfg.get("gelu_mode", "none"))
    return attention_pool(q, h, cfg["attn_pool_num_heads"])


def clip_small_embed(p, cfg, image, use_image=False):
    """InternVideo2_CLIP_small.encode_vision — InternVideo2/multi_modality/models/internvideo2_clip_small.py:125-142:
    [B,T,C,H,W] -> permute -> tower -> vision_align (LayerNorm, Linear :35-41)."""
    v = forward_clip_tower(p, cfg, image.permute(0, 2, 1, 3, 4), use_image, pre="vision_encoder.")
    v = layernorm(v, p["vision_align.0.weight"], p["vision_align.0.bias"])
    return linear(v, p["vision_align.1.weight"], p["vision_align.1.bias"])


# ------------------------------------------------------------------------------------ frozen teachers + mask
IVL = "InternVideo2/single_modality/models/internvl_clip_vision.py"
VMAE = "InternVideo2/single_modality/models/videomae.py"
ENG = "InternVideo2/single_modality/engines/engine_for_pretraining.py"


def internvl_clip_forward(p, cfg, image):
    """InternVL_CLIP.forward — {IVL}:414-465 (naive blocks, clip_norm_type 'l2', return_attn).
    image [B,C,T,H,W]; cfg: dict(depth, num_heads, attn_pool_num_heads, patch_size, return_index).
    Returns (z [K,B,1+T*HW,C], x [B,Cf], attn [B*T,HW])."""
    t = patch_embed(image, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], 1, cfg["patch_size"])
    B, T, L, C = t.shape
    h = torch.cat([p["cls_token"].expand(B * T, -1, -1), t.reshape(B * T, L, C)], dim=1) + p["pos_embed"]
    z = []
    for i in range(cfg["depth"]):
        h = block(p, i, h, cfg["num_heads"])
        if i in cfg["return_index"]:
            z.append(h)
    # AttentionPoolingBlock with return_attn ({IVL}:55-88,114-121): attention averaged over the heads
    pre, H = "clip_projector.", cfg["attn_pool_num_heads"]
    d = C // H
    xq = layernorm(h.mean(1, keepdim=True), p[pre + "norm1_q.weight"], p[pre + "norm1_q.bias"])
    xk = layernorm(h, p[pre + "norm1_k.weight"], p[pre + "norm1_k.bias"])
    xv = layernorm(h, p[pre + "norm1_v.weight"], p[pre + "norm1_v.bias"])
    ca = pre + "cross_attn."
    BT, N = h.shape[0], h.shape[1]
    q = linear(xq, p[ca + "q.weight"], p[ca + "q_bias"]).reshape(BT, 1, H, d).transpose(1, 2)
    k = linear(xk, p[ca + "k.weight"], p[ca + "k_bias"]).reshape(BT, N, H, d).transpose(1, 2)
    v = linear(xv, p[ca + "v.weight"], p[ca + "v_bias"]).reshape(BT, N, H, d).transpose(1, 2)
    a = ((q * d ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    x = linear((a @ v).transpose(1, 2).reshape(BT, 1, C), p[ca + "proj.weight"], p[ca + "proj.bias"]).squeeze(1)
    attn = a.mean(1)                                                     # [BT, 1, N]
    z = torch.stack(z)
    K = z.shape[0]
    cls, zz = z[:, :, :1, :], z[:, :, 1:, :]
    cls = cls.view(K, B, T, 1, C).mean(2)
    zz = torch.cat((cls, zz.reshape(K, B, T * L, C)), dim=2)
    zz = zz / zz.norm(dim=-1, keepdim=True)
    x = x.view(B, T, -1).mean(1)
    x = x / x.norm(dim=-1, keepdim=True)
    return zz, x, attn[:, 0, 1:]


def videomae_teacher_forward(p, cfg, x, pos_embed, head_axis_attention=True):
    """VideoMAE teacher VisionTransformer.forward — {VMAE}:283-313 over Block :104-132 / Attention :62-101.
    cfg: dict(depth, num_heads, patch_size, tubelet_size, return_index, eps).  head_axis_attention=True restates what
    the reference's flash_attn_func call computes on its [B,H,N,d] inputs (FA2 layout is [B,seqlen,nheads,d]): softmax
    over the H heads of each token, result reinterpreted by .reshape(B, N, -1) ({VMAE}:94-97)."""
    w = p["patch_embed.proj.weight"]
    t = patch_embed(x, w, p["patch_embed.proj.bias"], cfg["tubelet_size"], cfg["patch_size"])
    B = t.shape[0]
    C = t.shape[-1]
    h = t.reshape(B, -1, C) + pos_embed
    N, H = h.shape[1], cfg["num_heads"]
    d = C // H
    z = []
    for i in range(cfg["depth"]):
        pre = f"blocks.{i}."
        y = layernorm(h, p[pre + "norm1.weight"], p[pre + "norm1.bias"], cfg["eps"])
        bias = None
        if pre + "attn.q_bias" in p:
            bias = torch.cat((p[pre + "attn.q_bias"], torch.zeros_like(p[pre + "attn.v_bias"]), p[pre + "attn.v_bias"]))
        qkv = linear(y, p[pre + "attn.qkv.weight"], bias).reshape(B, N, 3, H, d).permute(2, 0, 3, 1, 4)   # [3,B,H,N,d]
        q, k, v = qkv[0], qkv[1], qkv[2]
        if head_axis_attention:     # FA2 semantics on [B, S=H, heads=N, d]
            sc = torch.einsum("bihd,bjhd->bhij", q * d ** -0.5, k)
            o = torch.einsum("bhij,bjhd->bihd", sc.softmax(-1), v).reshape(B, N, -1)
        else:
            sc = (q * d ** -0.5) @ k.transpose(-2, -1)
            o = (sc.softmax(-1) @ v).transpose(1, 2).reshape(B, N, -1)
        a = linear(o, p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"])
        h = h + (p[pre + "gamma_1"] * a if pre + "gamma_1" in p else a)
        y = layernorm(h, p[pre + "norm2.weight"], p[pre + "norm2.bias"], cfg["eps"])
        m = linear(gelu(linear(y, p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"])),
                   p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"])
        h = h + (p[pre + "gamma_2"] * m if pre + "gamma_2" in p else m)
        if i == cfg["depth"] - 1:
            h = layernorm(h, p["norm.weight"], p["norm.bias"], cfg["eps"])
        if i in cfg["return_index"]:
            z.append(h)
    out = torch.stack(z)
    return out / out.norm(dim=-1, keepdim=True)


MM2 = "InternVideo2/multi_modality/models/backbones/internvideo2/internvideo2.py"


def forward_stage2_tower(p, cfg, x, mask=None, use_image=False, x_vis_return_idx=-1, x_vis_only=False):
    """PretrainInternVideo2.forward of the stage-2 recipe — {MM2}:578-668 (joint position tables, naive blocks).
    cfg: dict(depth, num_heads, attn_pool_num_heads, patch_size, tubelet_size, num_frames, return_index [list]).
    mask None = every token visible (:613-616); use_image = temporal mean of the tables, or the image tables when the
    state dict holds `img_pos_embed` (:598-606, :658-667); the block loop stops after block depth + x_vis_return_idx (:631).
    Returns x_vis, or (x_vis, x_pool_vis, x_clip_align [K,B,n,Ct], x_align)."""
    t = patch_embed(x, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], cfg.get("tubelet_size", 1), cfg["patch_size"])
    B, T, L, C = t.shape
    t = torch.cat([p["cls_token"].expand(B, -1, -1), t.reshape(B, T * L, C)], dim=1)

    def table(which):
        pe = p[which + "pos_embed"]
        if not use_image:
            return pe
        if which + "img_pos_embed" in p:
            return p[which + "img_pos_embed"]
        Tm = cfg["num_frames"] // cfg.get("tubelet_size", 1)
        return torch.cat([pe[:, :1], pe[:, 1:].view(1, Tm, -1, C).mean(dim=1)], dim=1)

    h = t + table("")
    if mask is not None:
        idx = visible_indices(mask)
        h = torch.gather(h, 1, idx[:, :, None].expand(-1, -1, C))
    else:
        idx = torch.arange(h.shape[1])[None].expand(B, -1)
    x_clip = []
    for i in range(cfg["depth"]):
        h = block(p, i, h, cfg["num_heads"], cfg.get("gelu_mode", "none"))
        if i in cfg["return_index"]:
            x_clip.append(h)
        if i == cfg["depth"] + x_vis_return_idx:
            break
    if x_vis_only:
        return h
    pooled = attention_pool(p, h, cfg["attn_pool_num_heads"])
    x_align = linear_decoder(p, "final_clip_decoder.", pooled) if "final_clip_decoder.head.weight" in p else pooled
    cpe = torch.gather(table("clip_").expand(B, -1, -1), 1, idx[:, :, None].expand(-1, -1, C))
    x_clip_align = torch.stack([linear_decoder(p, f"clip_decoder.{k}.", xc + cpe) for k, xc in enumerate(x_clip)])
    return h, pooled, x_clip_align, x_align


IV1 = "InternVideo1/Pretrain/VideoMAE"


def sinusoid_table(n_position, d_hid):
    """get_sinusoid_encoding_table — {IV1}/modeling_finetune.py:224-242."""
    pos = torch.arange(n_position, dtype=torch.float64)[:, None]
    j = torch.arange(d_hid)[None, :]
    ang = pos / torch.pow(torch.tensor(10000.0, dtype=torch.float64), 2 * (j // 2) / d_hid)
    ang[:, 0::2] = torch.sin(ang[:, 0::2])
    ang[:, 1::2] = torch.cos(ang[:, 1::2])
    return ang.float()[None]


def _iv1_block(p, pre, h, num_heads, eps):
    """Block.forward — {IV1}/modeling_finetune.py:174-181 over Attention :101-129 (q_bias | 0 | v_bias)."""
    B, N, C = h.shape
    y = layernorm(h, p[pre + "norm1.weight"], p[pre + "norm1.bias"], eps)
    bias = None
    if pre + "attn.q_bias" in p:
        bias = torch.cat((p[pre + "attn.q_bias"], torch.zeros_like(p[pre + "attn.v_bias"]), p[pre + "attn.v_bias"]))
    qkv = linear(y, p[pre + "attn.qkv.weight"], bias).reshape(B, N, 3, num_heads, -1).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    d = q.shape[-1]
    o = (((q * d ** -0.5) @ k.transpose(-2, -1)).softmax(-1) @ v).transpose(1, 2).reshape(B, N, -1)
    a = linear(o, p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"])
    h = h + (p[pre + "gamma_1"] * a if pre + "gamma_1" in p else a)
    y = layernorm(h, p[pre + "norm2.weight"], p[pre + "norm2.bias"], eps)
    m = linear(gelu(linear(y, p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"])), p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"])
    return h + (p[pre + "gamma_2"] * m if pre + "gamma_2" in p else m)


def forward_iv1_videomae(p, cfg, x, mask, return_encoder=False):
    """PretrainVisionTransformer.forward — {IV1}/modeling_pretrain.py:366-387 (encoder :124-143, decoder :253-266).
    cfg: dict(encoder_depth, encoder_num_heads, decoder_depth, decoder_num_heads, patch_size, tubelet_size, eps).
    x [B,3,T,H,W], mask [B,N] bool (True = masked).  Returns the pixel predictions of the masked tubelets
    [B, N_mask, 3*tubelet*p*p] (x[mask] order)."""
    eps = cfg.get("eps", 1e-6)
    w = p["encoder.patch_embed.proj.weight"]
    t = patch_embed(x, w, p["encoder.patch_embed.proj.bias"], cfg["tubelet_size"], cfg["patch_size"])
    B, C = t.shape[0], t.shape[-1]
    t = t.reshape(B, -1, C)
    N = t.shape[1]
    t = t + sinusoid_table(N, C)
    vis = torch.stack([torch.nonzero(~mask[b]).flatten() for b in range(B)])
    msk = torch.stack([torch.nonzero(mask[b]).flatten() for b in range(B)])
    h = torch.gather(t, 1, vis[:, :, None].expand(-1, -1, C))
    for i in range(cfg["encoder_depth"]):
        h = _iv1_block(p, f"encoder.blocks.{i}.", h, cfg["encoder_num_heads"], eps)
    h = layernorm(h, p["encoder.norm.weight"], p["encoder.norm.bias"], eps)
    if return_encoder:
        return h
    h = linear(h, p["encoder_to_decoder.weight"])
    Cd = h.shape[-1]
    pos = sinusoid_table(N, Cd).expand(B, -1, -1)
    pos_vis = torch.gather(pos, 1, vis[:, :, None].expand(-1, -1, Cd))
    pos_msk = torch.gather(pos, 1, msk[:, :, None].expand(-1, -1, Cd))
    full = torch.cat([h + pos_vis, p["mask_token"] + pos_msk], dim=1)
    for i in range(cfg["decoder_depth"]):
        full = _iv1_block(p, f"decoder.blocks.{i}.", full, cfg["decoder_num_heads"], eps)
    y = layernorm(full[:, -msk.shape[1]:], p["decoder.norm.weight"], p["decoder.norm.bias"], eps)
    return linear(y, p["decoder.head.weight"], p["decoder.head.bias"])


def attention_guided_mask(attn, B, mask_ratio, importance):
    """{ENG}:105-116 with the multinomial draw (`importance`, a permutation per frame) given."""
    BT, N = attn.shape
    n_vis = N - int(N * mask_ratio)
    m = torch.ones((BT, N))
    pos1 = torch.arange(BT).view(-1, 1).repeat(1, n_vis)
    m[pos1, importance[:, :n_vis]] = 0
    m = torch.cat((torch.zeros(B, 1), m.view(B, -1)), dim=1)
    return m.to(torch.bool)


def align_loss(out, tgt):
    """(2 - 2 * (out * tgt).sum(-1)).mean() — InternVideo2/single_modality/engines/engine_for_pretraining.py:131-136."""
    return (2 - 2 * (out * tgt).sum(dim=-1)).mean()


# ------------------------------------------------------------------------------------ contrastive
MM = "InternVideo2/multi_modality/models/criterions.py"


def get_sim(v, t, temp=1.0):
    """get_sim 2-D branch — {MM}:31-32,51-53 (F.normalize eps=1e-12)."""
    v = v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    t = t / t.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    s = v @ t.t() / temp
    return s, s.t()


def get_mask(idx, dtype=torch.float32, normalize=True):
    """VTC_VTM_Loss.get_mask — {MM}:200-216: (idx == idx^T), rows normalised to sum 1."""
    idx = idx.view(-1, 1)
    m = torch.eq(idx, idx.t()).to(dtype)
    if normalize:
        m = m / m.sum(1, keepdim=True)
    return m


def vtc_loss(v_all, t_all, idx_all, temp):
    """VTC_VTM_Loss.vtc_loss after the gather — {MM}:93-102."""
    s_v2t, s_t2v = get_sim(v_all, t_all, temp)
    tg = get_mask(idx_all, s_v2t.dtype)
    l1 = -(F.log_softmax(s_v2t, dim=1) * tg).sum(1).mean()
    l2 = -(F.log_softmax(s_t2v, dim=1) * tg).sum(1).mean()
    return (l1 + l2) / 2


def allgather_rows(local_list):
    """AllGather.forward — InternVideo2/multi_modality/models/utils.py:197-202: cat over ranks in rank order."""
    return torch.cat(list(local_list), dim=0)


def allgather_backward(grad_output, rank, batch):
    """AllGather.backward — models/utils.py:205-209: LOCAL slice only, no collective."""
    return grad_output[batch * rank: batch * (rank + 1)]


# ------------------------------------------------------------------------------------ IV1 pixel target
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def pixel_targets(images, mask, patch=16, tubelet=2, normalize=True):
    """Target construction of the IV1 VideoMAE pixel head —
    InternVideo1/Pretrain/VideoMAE/engine_for_pretraining.py:66-98.

    images [B,3,T,H,W] (ImageNet-normalised), mask [B,N] bool True=masked.
    Returns labels [B, N_mask, tubelet*patch*patch*3].
    """
    mean = torch.tensor(IMAGENET_MEAN, dtype=images.dtype)[None, :, None, None, None]
    std = torch.tensor(IMAGENET_STD, dtype=images.dtype)[None, :, None, None, None]
    un = images * std + mean
    B, C, T, H, W = un.shape
    t, h, w = T // tubelet, H // patch, W // patch
    sq = un.reshape(B, C, t, tubelet, h, patch, w, patch).permute(0, 2, 4, 6, 3, 5, 7, 1)
    sq = sq.reshape(B, t * h * w, tubelet * patch * patch, C)        # b (t h w) (p0 p1 p2) c
    if normalize:
        mu = sq.mean(dim=-2, keepdim=True)
        var = sq.var(dim=-2, unbiased=True, keepdim=True)
        sq = (sq - mu) / (var.sqrt() + 1e-6)
    patchv = sq.reshape(B, t * h * w, -1)                            # b n (p c)
    Cc = patchv.shape[-1]
    return patchv[mask].reshape(B, -1, Cc)


def mse_loss(pred, target):
    """nn.MSELoss() — engine_for_pretraining.py:43,106."""
    return ((pred - target) ** 2).mean()


for _f in (rmsnorm, layernorm, gelu, patch_embed, visible_indices, embed_tokens, attention, mlp,
           block, attention_pool, l2n, linear_decoder, mlp_decoder, forward_pretrain):
    if _f.__doc__:
        _f.__doc__ = _f.__doc__.replace("{SM}", SM)
forward_clip_tower.__doc__ = forward_clip_tower.__doc__.replace("{MMV}", MMV)
for _f in (internvl_clip_forward, videomae_teacher_forward, attention_guided_mask):
    _f.__doc__ = _f.__doc__.replace("{IVL}", IVL).replace("{VMAE}", VMAE).replace("{ENG}", ENG)
for _f in (get_sim, get_mask, vtc_loss):
    _f.__doc__ = _f.__doc__.replace("{MM}", MM)
