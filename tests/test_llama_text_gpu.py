"""InternVideo2-CLIP's LLaMA text tower on the GPU: the SwiGLU GEMM epilogue and the RoPE kernel element by element
against float64, the tiny tower against tests/golden/llama_text.npz (outputs of the unmodified reference), one full-size
layer and the full 7B tower against the fp32 restatement (oracle/llama_text.py), and the InternVideo2_CLIP wrapper's
loss and trainable gradients against an fp32 restatement of the whole model.  No test reads the reference tree."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from gemm_ref import gemm_ref
from internvideo_b200 import lowlevel as ll
from internvideo_b200.llama_modules import LLAMA_7B, LLaMA, rope_tables
from oracle import llama_text as ol
from oracle import restate as rs

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
bf = torch.bfloat16

# every kernel form the bf16 entry point runs IVB_EPI_SWIGLU on: the cooperative kernel at each tile_n, the ping-pong
# kernel, and the library's own choice
FORMS = [("coop128", ll.FLAG_1CTA, 128), ("coop176", ll.FLAG_1CTA, 176), ("coop192", ll.FLAG_1CTA, 192),
         ("coop256", ll.FLAG_1CTA, 256), ("pingpong", ll.FLAG_PINGPONG, 0), ("auto", 0, 0)]


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(bf)


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm())


def _swiglu_ref(x, w):
    """float64 silu(x gate^T) * (x up^T) and its bound: the fp32 accumulation bounds of both products (gemm_ref, as the
    other epilogue tests use them) carried through silu(g) u, plus 2^-8 of |silu(g)| |u| for the fp32 evaluation and
    the one bf16 rounding."""
    I = w.shape[0] // 2
    (v, e), = gemm_ref(x, w, epi=ll.EPI_F32)
    g, u, eg, eu = v[:, :I], v[:, I:], e[:, :I], e[:, I:]
    s = torch.sigmoid(g)
    f = g * s
    df = s * (1 + g * (1 - s))
    ref = f * u
    return ref, df.abs() * u.abs() * eg + f.abs() * eu + 2.0 ** -8 * (f * u).abs()


@pytest.mark.parametrize("M,K,I", [(8192, 4096, 11008), (1000, 4096, 344), (1000, 256, 8)],
                         ids=["7b", "tail344", "tail8"])
def test_swiglu_against_fp64(cuda_lib, M, K, I):
    x = _mk((M, K), 1)
    w = _mk((2 * I, K), 2, K ** -0.5 * 2)
    ref, bound = _swiglu_ref(x, w)
    for name, flags, tile_n in FORMS:
        out = ll.gemm(x, w, epi=ll.EPI_SWIGLU, flags=flags, tile_n=tile_n)
        assert out.shape == (M, I)
        err = ((out.double() - ref).abs() / (bound + 1e-300)).max().item()
        assert err <= 1.0, (name, err)
        again = ll.gemm(x, w, epi=ll.EPI_SWIGLU, flags=flags, tile_n=tile_n)
        assert torch.equal(out.view(torch.int16), again.view(torch.int16)), name
    torch.cuda.synchronize()


def test_swiglu_writes_into_a_view(cuda_lib):
    """out0 a column slot of a wider buffer (pitch > I): only its columns are written."""
    M, K, I = 300, 512, 344
    x, w = _mk((M, K), 3), _mk((2 * I, K), 4, 0.05)
    buf = torch.full((M, I + 40), 7.0, device="cuda", dtype=bf)
    ll.gemm(x, w, epi=ll.EPI_SWIGLU, out0=buf[:, 16:16 + I])
    ref = ll.gemm(x, w, epi=ll.EPI_SWIGLU)
    assert torch.equal(buf[:, 16:16 + I], ref)
    assert bool((buf[:, :16] == 7).all()) and bool((buf[:, 16 + I:] == 7).all())


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("L", [1, 32, 77])
def test_rope_against_fp64(cuda_lib, d, L):
    B, H = 3, 4
    qkv = _mk((B * L, 3 * H * d + 8), 5 + L + d)[:, :3 * H * d]
    before = qkv.clone()
    cos, sin = rope_tables(L, d, 10000.0, "cuda")
    ll._rope_qk(qkv[:, :H * d], qkv[:, H * d:2 * H * d], B, L, H, d, cos, sin)
    c, s = cos.double().repeat(B, 1)[:, None, :], sin.double().repeat(B, 1)[:, None, :]
    for slot in (0, 1):
        x = before[:, slot * H * d:(slot + 1) * H * d].double().reshape(B * L, H, d)
        x1, x2 = x[..., :d // 2], x[..., d // 2:]
        ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
        bound = 2.0 ** -8 * torch.cat([x1.abs() + x2.abs()] * 2, -1)
        got = qkv[:, slot * H * d:(slot + 1) * H * d].double().reshape(B * L, H, d)
        assert bool(((got - ref).abs() <= bound).all()), (slot, float((got - ref).abs().max()))
    assert torch.equal(qkv[:, 2 * H * d:], before[:, 2 * H * d:])       # v untouched


def _tiny(cfg, sd, clip_embed_dim):
    model = LLaMA(use_flash_attn=True, transformer_width=cfg["hidden_size"], use_lora=False,
                  clip_embed_dim=clip_embed_dim, config={k: v for k, v in cfg.items() if k != "clip_embed_dim"})
    model.load_state_dict(sd, strict=True)
    return model.bfloat16().cuda().requires_grad_(False).eval()


def test_tiny_tower_against_reference_golden(cuda_lib):
    cfg, sd, z = ol.load(GOLD / "llama_text.npz")
    model = _tiny(cfg, sd, cfg["clip_embed_dim"])
    ids = torch.from_numpy(z["ids"]).cuda()
    out = model(ids)
    ref = torch.from_numpy(z["out"])
    for b in range(ids.shape[0]):
        assert _rel(out[b].float().cpu(), ref[b]) < 1e-2, b
    # a CUDA-graph replay gives the plain call's bits
    static = ids.clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout = model(static)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gout.view(torch.int16), out.view(torch.int16))
    # a caption whose nonzero ids are not a prefix, and one with none, get NaN rows; the others keep their bits
    bad = ids.clone()
    bad[1, 2] = 0
    bad[3] = 0
    o2 = model(bad)
    assert bool(o2[1].isnan().all()) and bool(o2[3].isnan().all())
    assert torch.equal(o2[0].view(torch.int16), out[0].view(torch.int16))
    assert torch.equal(o2[2].view(torch.int16), out[2].view(torch.int16))


def _random_state(model, seed, device="cuda"):
    """fp32 parameters drawn on the device: N(0, 1/fan_in) weights, a N(0, 1) token table, RMSNorm weights 1 + N(0,
    0.1^2)."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for k, v in model.state_dict().items():
        r = torch.randn(tuple(v.shape), generator=g, device=device)
        if k.endswith("norm.weight"):
            r = 1 + 0.1 * r
        elif k.endswith("embed_tokens.weight"):
            pass
        else:
            r = r * (v.shape[0] if k == "text_projection" else v.shape[1]) ** -0.5
        sd[k] = r.to(bf)
    return sd


def _ids(B, L, V, seed, lengths):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(3, V, (B, L), generator=g, device="cuda")
    ids[:, 0] = 1
    keep = torch.arange(L, device="cuda")[None, :] < torch.tensor(lengths, device="cuda")[:, None]
    return ids * keep


def _against_restatement(cfg, B, L, seed):
    """(port's error, the restatement's own error when run in bf16), each relative to the fp32 restatement, on random
    device-built weights of `cfg`."""
    with torch.device("meta"):
        model = LLaMA(transformer_width=cfg["hidden_size"], use_lora=False, clip_embed_dim=768, config=cfg).bfloat16()
    model = model.to_empty(device="cuda").requires_grad_(False)
    model.load_state_dict(_random_state(model, seed), strict=True)
    lengths = [L - (7 * b) % L for b in range(B)]
    ids = _ids(B, L, cfg["vocab_size"], seed + 1, lengths)
    out = model(ids).float()
    sd = model.state_dict()          # after the forward: gate and up are views of the joined buffer
    full = dict(ol.CFG, **cfg)
    with torch.no_grad():
        ref32 = ol.restate(sd, ids, full, dtype=torch.float32)
        ref16 = ol.restate(sd, ids, full, dtype=bf).float()
    return _rel(out, ref32), _rel(ref16, ref32)


def test_full_size_layer_against_fp32(cuda_lib):
    """One LLaMA-7B layer (D 4096, I 11008, 32 heads of 128) at 256 x 32 tokens."""
    cfg = dict(LLAMA_7B, num_hidden_layers=1, vocab_size=4096)
    err, err16 = _against_restatement(cfg, 256, 32, 11)
    assert err < 1e-2 and err <= 3 * err16, (err, err16)


def test_full_7b_tower_against_fp32(cuda_lib):
    """The whole 32-layer tower at 8 x 32: within 3x the error of the restatement itself run in bf16."""
    err, err16 = _against_restatement(dict(LLAMA_7B), 8, 32, 12)
    assert err <= 3 * err16, (err, err16)
    torch.cuda.empty_cache()


def test_clip_wrapper_loss_and_trainable_gradients(cuda_lib):
    """InternVideo2_CLIP with the tiny vision tower of tests/golden/clip_small.npz (frozen, projector open) and the tiny
    LLaMA (frozen, text_projection open): loss_vtc and the projector and text_projection gradients against an fp32
    restatement (oracle/restate.py's tower and loss, oracle/llama_text.py's text tower); nothing else gets a gradient."""
    from internvideo_b200.clip_modules import InternVideo2_CLIP
    z = np.load(GOLD / "clip_small.npz")
    vcfg = json.loads(bytes(z["cfg"]).decode())
    ve = dict(in_chans=3, qkv_bias=False, head_drop_path_rate=0.0, use_flash_attn=False, use_fused_rmsnorm=False,
              use_fused_mlp=False, fused_mlp_heuristic=1, tubelet_size=1, sep_pos_embed=False, use_checkpoint=False,
              checkpoint_num=0, **{k: v for k, v in vcfg.items() if k != "align_dim"})
    config = dict(model=dict(vision_encoder=ve, temp=0.07, temp_min=0.01, freeze_vision=True,
                             open_vision_clip_projector=True, freeze_text=True, open_text_projection=True))
    tcfg, tsd, tz = ol.load(GOLD / "llama_text.npz")
    E = vcfg["clip_embed_dim"]
    tsd["text_projection"] = ol.draw_param("text_projection", (tcfg["hidden_size"], E))
    text = LLaMA(transformer_width=tcfg["hidden_size"], use_lora=False, clip_embed_dim=E,
                 config={k: v for k, v in tcfg.items() if k != "clip_embed_dim"})
    model = InternVideo2_CLIP(config, text_encoder=text)
    vsd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/vision_encoder.")}
    missing, unexpected = model.load_state_dict(dict(vsd, temp=torch.tensor(0.07),
                                                     **{"text_encoder." + k: v for k, v in tsd.items()}), strict=False)
    assert not unexpected and not missing, (missing, unexpected)
    model = model.bfloat16().cuda().train()
    image = torch.from_numpy(z["image"]).cuda().to(bf)
    idx = torch.from_numpy(z["idx"]).cuda()
    ids = torch.from_numpy(tz["ids"]).cuda()
    out = model(image, ids, idx)
    out["loss_vtc"].backward()

    p = {k: v.detach().float().clone() for k, v in model.state_dict().items()}
    train = [k for k in p if k.startswith("vision_encoder.clip_projector.") or k == "text_encoder.text_projection"]
    for k in train:
        p[k].requires_grad_(True)
    v = rs.forward_clip_tower(p, dict(vcfg, tubelet_size=1), image.float().permute(0, 2, 1, 3, 4),
                              pre="vision_encoder.")
    t = ol.restate({k[len("text_encoder."):]: w for k, w in p.items() if k.startswith("text_encoder.")}, ids, tcfg)
    loss = rs.vtc_loss(v, t, idx, p["temp"])
    loss.backward()
    assert abs(float(out["loss_vtc"]) - float(loss)) < 1e-2 * max(1.0, abs(float(loss)))
    named = dict(model.named_parameters())
    gmax = max(float(p[k].grad.norm()) for k in train)
    bad = {}
    for k in train:
        if float(p[k].grad.norm()) < 1e-5 * gmax:     # the key biases: softmax ignores a shift shared by every key
            assert float(named[k].grad.float().norm()) < 1e-3 * gmax, k
        elif _rel(named[k].grad.float(), p[k].grad) > 3e-2:
            bad[k] = _rel(named[k].grad.float(), p[k].grad)
    assert not bad, bad
    for k, prm in named.items():
        if k not in train and k != "temp":
            assert prm.grad is None, k
