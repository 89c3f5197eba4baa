"""The MobileCLIP text tower on the H100: causal attention forward and backward tile by tile against float64, the token
embedding and its fixed-order gradients, the tower against tests/golden/text_tower.npz (outputs of the unmodified
reference TextTransformer; <= 1e-2 relative for outputs, <= 3e-2 for parameter gradients, as elsewhere), and a
video-text step of InternVideo2_CLIP_small with the tower, eager and replayed from a CUDA graph."""
import math
from pathlib import Path

import numpy as np
import pytest
import torch

from attn_ref import tile_errors, worst
from oracle import text_tower

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
GOLD = Path(__file__).parent / "golden" / "text_tower.npz"

# tile error of O / dQ / dK / dV and max |lse2 error|: the non-causal kernels' limits (tests/test_attn_gpu.py)
LIMITS = {"o": 1.2e-2, "lse": 1.0e-5, "dq": 1.3e-2, "dk": 1.3e-2, "dv": 9.5e-3}


def _randn(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


def _causal_ref(q, k, v, dout, B, n, H, d, scale):
    """float64 causal attention per clip: O, lse2 [B, H, n] and the analytic dQ, dK, dV (the -inf upper triangle
    gives P = 0 above the diagonal, so dS = P * (dP - rowsum(P * dP)) is 0 there too)."""
    heads = lambda x, b: x[b * n:(b + 1) * n].double().reshape(n, H, d).transpose(0, 1)  # noqa: E731
    flat = lambda x: x.transpose(0, 1).reshape(n, H * d)  # noqa: E731
    out = torch.empty((B * n, H * d), dtype=torch.float64, device=q.device)
    lse2 = torch.empty((B, H, n), dtype=torch.float64, device=q.device)
    grads = [torch.empty_like(out) for _ in range(3)]
    mask = torch.full((n, n), float("-inf"), dtype=torch.float64, device=q.device).triu(1)
    for b in range(B):
        qb, kb, vb, gb = (heads(t, b) for t in (q, k, v, dout))
        s = qb @ kb.transpose(-2, -1) * scale + mask
        lse = torch.logsumexp(s, -1, keepdim=True)
        p = torch.exp(s - lse)
        out[b * n:(b + 1) * n] = flat(p @ vb)
        lse2[b] = lse.squeeze(-1) / math.log(2.0)
        dp = gb @ vb.transpose(-2, -1)
        ds = p * (dp - (p * dp).sum(-1, keepdim=True))
        for g, t in zip(grads, (scale * ds @ kb, scale * ds.transpose(-2, -1) @ qb, p.transpose(-2, -1) @ gb)):
            g[b * n:(b + 1) * n] = flat(t)
    return out, lse2, grads


def _tiles(kind, got, ref, B, n, H, d):
    e, (b, h, band) = worst(tile_errors(got, ref, B, n, H, d))
    assert e <= LIMITS[kind], f"{kind}: {e:.3e} > {LIMITS[kind]:.1e} at clip {b}, head {h}, rows from {64 * band}"


# (n, d, H): the text tower's 77 tokens; one whole 128-row block; 200 = two blocks, the second with one live warpgroup
# and a ragged key tile (d = 88: a zero-filled head tail); 417 = four blocks and a tail; 1025 = nine blocks, 17 key
# tiles, head dim 128
CASES = [(77, 64, 8), (128, 64, 8), (200, 88, 16), (417, 64, 4), (1025, 128, 2)]


@pytest.mark.parametrize("n,d,H", CASES)
def test_causal_attention_matches_fp64(cuda_lib, n, d, H):
    B, D = 2, H * d
    scale = d ** -0.5
    qkv = _randn(B * n, 3 * D, seed=n + d).to(bf16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    dout = _randn(B * n, D, seed=n + 7).to(bf16)
    out, lse = cuda_lib.attn_fwd(q, k, v, B, n, H, d, scale, causal=True)
    o_ref, lse_ref, g_ref = _causal_ref(q, k, v, dout, B, n, H, d, scale)
    _tiles("o", out, o_ref, B, n, H, d)
    e_lse, where = worst((lse.double() - lse_ref).abs())
    assert e_lse <= LIMITS["lse"], (e_lse, where)
    g = torch.full((B * n, 3 * D), float("nan"), device="cuda", dtype=bf16)     # a skipped element stays NaN
    cuda_lib.attn_bwd(q, k, v, out, dout, lse, B, n, H, d, scale, g[:, :D], g[:, D:2 * D], g[:, 2 * D:], causal=True)
    for name, got, ref in zip(("dq", "dk", "dv"), (g[:, :D], g[:, D:2 * D], g[:, 2 * D:]), g_ref):
        assert bool(torch.isfinite(got).all()), name
        _tiles(name, got, ref, B, n, H, d)


def test_causal_attention_refuses_droppath_rowscale(cuda_lib):
    from internvideo_b200 import _lib
    q = torch.zeros(2 * 77, 128, device="cuda", dtype=bf16)
    rs = torch.ones(2 * 77, device="cuda")
    with pytest.raises(_lib.IvbError, match="causal"):
        cuda_lib.attn_fwd(q, q, q, 2, 77, 2, 64, 0.125, rowscale=rs, causal=True)


# ------------------------------------------------------------------------------------------- token embedding
def _ids(B, L, V, seed):
    """Captions with many repeats: zero padding and words from a small vocabulary, EOT (V - 1) at varying positions."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 40, (B, L), generator=g)
    for b in range(B):
        e = 1 + b * 7 % (L - 1)
        ids[b, e] = V - 1
        ids[b, e + 1:] = 0
    return ids.cuda()


def test_token_embedding_forward_backward(cuda_lib):
    """Forward: E[id] + P exactly (an fp32 sum of two bf16 values).  Backward at the cfg-3 per-GPU shape (128
    captions x 77 tokens, vocabulary 49408, width 512) against float64 sums, and bit for bit the same on a second
    run."""
    B, L, V, D = 128, 77, 49408, 512
    ids = _ids(B, L, V, seed=3)
    E = _randn(V, D, seed=1).to(bf16)
    P = _randn(L, D, seed=2).to(bf16)
    out, err = cuda_lib._token_embed_fwd(ids, E, P)
    assert int(err) == 0
    ref = (E.float()[ids] + P.float()).reshape(B * L, D)
    assert torch.equal(out, ref)
    g = _randn(B * L, D, seed=4)
    dE, dP = cuda_lib._token_embed_bwd(ids, g, V)
    dE_ref = torch.zeros(V, D, dtype=torch.float64, device="cuda").index_add_(0, ids.reshape(-1), g.double())
    dP_ref = g.double().reshape(B, L, D).sum(0)
    torch.testing.assert_close(dE.double(), dE_ref, atol=2e-3, rtol=1e-5)
    torch.testing.assert_close(dP.double(), dP_ref, atol=2e-3, rtol=1e-5)
    dE2, dP2 = cuda_lib._token_embed_bwd(ids, g, V)
    assert torch.equal(dE, dE2) and torch.equal(dP, dP2)


def test_token_embedding_flags_bad_ids(cuda_lib):
    ids = torch.tensor([[1, 2, 1000], [3, -1, 4]], device="cuda")
    E = _randn(1000, 64, seed=1).to(bf16)
    P = _randn(3, 64, seed=2).to(bf16)
    out, err = cuda_lib._token_embed_fwd(ids, E, P)
    assert int(err) in (3, 5)                                    # 1 + a row holding a bad id
    assert torch.equal(out[2], E[0].float() + P[2].float())      # read as id 0


# ------------------------------------------------------------------------------------------- the tower
def _rel(a, b):
    a = a.detach().float().cpu(); b = b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _tower():
    from internvideo_b200.text_modules import TextTransformer
    cfg, sd, z = text_tower.load(GOLD)
    tower = TextTransformer(cfg, cfg["projection_dim"])
    tower.load_state_dict(sd, strict=True)
    return z, tower.bfloat16().cuda()


def test_text_tower_matches_reference_golden(cuda_lib):
    z, tower = _tower()
    ids = torch.from_numpy(z["ids"]).cuda()
    pooled = tower(ids)
    every = tower(ids[:text_tower.ALL_TOKENS_ROWS], return_all_tokens=True)
    assert _rel(pooled, torch.from_numpy(z["pooled"])) < 1e-2
    assert _rel(every, torch.from_numpy(z["all_tokens"])) < 1e-2
    wp, wa = (w.cuda() for w in text_tower.loss_weights(pooled.shape, every.shape))
    ((pooled.float() * wp).sum() + (every.float() * wa).sum()).backward()
    bad = {k: _rel(p.grad, torch.from_numpy(z["g/" + k])) for k, p in tower.named_parameters()}
    bad = {k: r for k, r in bad.items() if r > 3e-2}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])


def test_text_tower_no_grad_path(cuda_lib):
    """A tower whose parameters need no gradient runs its blocks without saving anything and gives the outputs of the
    differentiated path; key_padding_mask is ignored under causal masking, as in the reference."""
    z, tower = _tower()
    ids = torch.from_numpy(z["ids"]).cuda()
    trained = tower(ids)
    tower.requires_grad_(False)
    frozen = tower(ids, key_padding_mask=ids == 0)
    assert frozen.grad_fn is None
    assert _rel(frozen, trained) < 1e-3


def test_text_tower_bad_id_poisons_output(cuda_lib):
    z, tower = _tower()
    ids = torch.from_numpy(z["ids"]).cuda()
    ids[0, 1] = tower.vocab_size
    with torch.no_grad():
        assert bool(torch.isnan(tower(ids)).all())


def test_clip_small_with_text_tower_step_replays_in_a_cuda_graph(cuda_lib):
    """A video-text step of InternVideo2_CLIP_small with the text tower passed as text_encoder= (vision tower, text
    tower, alignment head and VTC loss, forward and backward) captured in engine.GraphedStep replays with the eager
    step's loss, and the trainable text tower receives gradients.  The loss sums rows with atomics, so its last bits
    may differ between any two runs: 8 fp32 ulps are allowed."""
    from internvideo_b200.clip_modules import InternVideo2_CLIP_small
    from internvideo_b200.engine import GraphedStep
    _, tower = _tower()
    ve = dict(embed_dim=64, depth=2, num_heads=2, mlp_ratio=4, num_frames=4, tubelet_size=1, img_size=28, patch_size=14,
              attn_pool_num_heads=2, clip_embed_dim=16, align_dim=tower.projection_dim, drop_path_rate=0.0,
              use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False)
    torch.manual_seed(0)
    model = InternVideo2_CLIP_small(dict(model=dict(vision_encoder=ve, temp=0.07, temp_min=0.01, freeze_vision=False,
                                                    freeze_text=False)), text_encoder=tower)
    model = model.bfloat16().cuda().train()
    B = 8
    image = _randn(B, 4, 3, 28, 28, seed=5).to(bf16)
    text = torch.from_numpy(np.load(GOLD)["ids"]).cuda()
    idx = torch.arange(B, device="cuda")

    def step(image, text, idx):
        model.zero_grad(set_to_none=False)
        loss = model(image, text, idx)["loss_vtc"]
        loss.backward()
        return loss

    step(image, text, idx)
    loss_eager = float(step(image, text, idx))
    g = model.text_encoder.transformer[0].pre_norm_mha[1].qkv_proj.weight.grad
    assert g is not None and float(g.float().norm()) > 0
    graphed = GraphedStep(step, [image.clone(), text.clone(), idx.clone()], warmup=1)
    loss_graph = float(graphed(image, text, idx)[0])
    torch.cuda.synchronize()
    print(f"CLIP step with the text tower: eager loss {loss_eager!r}, graph replay {loss_graph!r}")
    assert loss_eager == loss_eager and abs(loss_graph - loss_eager) <= 8 * 2.0 ** -23 * abs(loss_eager)
