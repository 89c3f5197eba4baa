"""The MobileCLIP text tower on the H100: the causal attention's refusal of a DropPath plan (its comparison with the
masked float64 reference is the causal form of tests/test_attn_gpu.py), the token embedding and its fixed-order
gradients, the tower against tests/golden/text_tower.npz (outputs of the unmodified reference TextTransformer;
<= 1e-2 relative for outputs, <= 3e-2 for parameter gradients, as elsewhere), and a video-text step of
InternVideo2_CLIP_small with the tower, eager and replayed from a CUDA graph."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import text_tower

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
GOLD = Path(__file__).parent / "golden" / "text_tower.npz"


def _randn(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


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
