"""FP8 for the LayerNorm towers on the H100 (gpu): InternVideo1's VideoMAE blocks and the MobileCLIP text tower's causal
blocks trained under modules.set_fp8, the text tower and the stage-2 BERT text layers under modules.set_fp8_inference.

- Block level, at real widths: a VideoMAEBlock (D = 768, 12 heads, q/v bias, gamma) and a causal TransformerEncoder
  (D = 512, 8 heads, full qkv bias, no gamma), each in every set_fp8 mode, against the bf16 block and against a float64
  restatement (output, dx and every parameter gradient, relative Frobenius error); the checkpointed block gives the
  plain block's bits, and switching off gives the bf16 bits back.
- Model level: iv1_videomae.npz and text_tower.npz (outputs of the unmodified references) in per-token FP8; a few
  training steps on one batch drop the loss like bf16; the gradient sink gives autograd's gradient; the IV1 step captured
  in a CUDA graph replays with the eager loss.
- Inference: bert_text.npz and the text tower under set_fp8_inference against bf16; BERT's padded rows behave as in
  bf16; switching off restores the bf16 bits; a weight changed in place is re-quantised.

Bounds.  u = 2^-4 is the unit roundoff of E4M3 (2^-3 of E5M2).  A GEMM whose operands are each rounded with relative
error at most u_a and u_b is off by at most u_a + u_b per product, and so is its relative Frobenius error: the block's
output 2u(E4M3) = 0.125, dx and the parameter gradients 4u = 0.25 (E4M3 gradients x E4M3 weights, and weight gradients
reading the FP8 forward's activations), per-tensor FP8's gradients 2(u(E5M2) + u(E4M3)) = 0.375: the bounds
tests/test_fp8_modes_gpu.py derives for the RMSNorm block.  They catch a wrong scale, format or operand, which is off by
factors, not by percent.  The FP8 weight gradients are held to 0.15, as there.  Against float64 the same bounds hold
(the bf16 block itself is within 1e-2 of float64, checked here too).
"""
import json
from functools import partial
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from internvideo_b200 import _lib
from internvideo_b200 import modules as M

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
bf16 = torch.bfloat16
MODES = {"tensor": dict(scaling="tensor"), "token": dict(scaling="token"),
         "token_wgrad": dict(scaling="token", wgrad=True)}
U_E4M3, U_E5M2 = 2.0 ** -4, 2.0 ** -3
OUT_BOUND = 2 * U_E4M3
GRAD_BOUND = {"tensor": 2 * (U_E5M2 + U_E4M3), "token": 4 * U_E4M3, "token_wgrad": 4 * U_E4M3}
WGRAD_BOUND = 0.15


def _rel(a, b):
    a = a.detach().double(); b = b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------ the blocks
# (block, the Linear / LayerNorm / bias names of its parameters, B, n, causal)
def _videomae_block():
    return M.VideoMAEBlock(768, 12, 4.0, qkv_bias=True, init_values=0.1, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def _text_block():
    from internvideo_b200.text_modules import TransformerEncoder
    return TransformerEncoder(512, 2048, 8)


BLOCKS = {"videomae": (_videomae_block, 4, 157, False), "text_causal": (_text_block, 16, 77, True)}


def _names(blk):
    """BlockParams field -> parameter name (None: absent)."""
    if isinstance(blk, M.VideoMAEBlock):
        return dict(n1w="norm1.weight", n1b="norm1.bias", qkvw="attn.qkv.weight", projw="attn.proj.weight",
                    projb="attn.proj.bias", g1="gamma_1", n2w="norm2.weight", n2b="norm2.bias", fc1w="mlp.fc1.weight",
                    fc1b="mlp.fc1.bias", fc2w="mlp.fc2.weight", fc2b="mlp.fc2.bias", g2="gamma_2")
    return dict(n1w="pre_norm_mha.0.weight", n1b="pre_norm_mha.0.bias", qkvw="pre_norm_mha.1.qkv_proj.weight",
                qkvb="pre_norm_mha.1.qkv_proj.bias", projw="pre_norm_mha.1.out_proj.weight",
                projb="pre_norm_mha.1.out_proj.bias", n2w="pre_norm_ffn.0.weight", n2b="pre_norm_ffn.0.bias",
                fc1w="pre_norm_ffn.1.weight", fc1b="pre_norm_ffn.1.bias", fc2w="pre_norm_ffn.4.weight",
                fc2b="pre_norm_ffn.4.bias")


def _make(kind, mode=None, with_cp=False):
    """The block with every parameter drawn from one seed (Linear weights N(0, 1/fan_in), biases N(0, 0.05^2), norm
    weights 1 + N(0, 0.1^2), gamma 0.5 + N(0, 0.1^2)), bf16 on the device, in set_fp8 mode `mode` (None: bf16)."""
    make = BLOCKS[kind][0]
    blk = make()
    blk.with_cp = with_cp
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for name, p in blk.named_parameters():
            r = torch.randn(p.shape, generator=g)
            if p.dim() == 2:
                p.copy_(r * p.shape[1] ** -0.5)
            elif "gamma" in name:
                p.copy_(0.5 + 0.1 * r)
            elif name.endswith("weight"):                 # the LayerNorm weights
                p.copy_(1 + 0.1 * r)
            else:                                         # every bias, q_bias and v_bias
                p.copy_(0.05 * r)
    blk = blk.bfloat16().cuda()
    if mode is not None:
        assert M.set_fp8(blk, True, **MODES[mode]) == 1
    return blk


def _inputs(kind, D):
    _, B, n, _ = BLOCKS[kind]
    g = torch.Generator(device="cuda").manual_seed(5)
    return torch.randn(B * n, D, device="cuda", generator=g), torch.randn(B * n, D, device="cuda", generator=g)


def _forward(blk, x, kind):
    _, B, n, causal = BLOCKS[kind]
    if isinstance(blk, M.VideoMAEBlock):
        return blk.forward_stream(x, B, n)
    return blk.forward_stream(x, B, n, causal)


def _run(blk, kind):
    x, dy = _inputs(kind, blk.norm1.weight.shape[0] if isinstance(blk, M.VideoMAEBlock) else blk.embed_dim)
    for p in blk.parameters():
        p.grad = None
    xs = x.clone().requires_grad_(True)
    y = _forward(blk, xs, kind)
    y.backward(dy)
    return y.detach(), xs.grad, {k: p.grad.clone() for k, p in blk.named_parameters()}


def _ref64(blk, kind):
    """(y, dx, gradients) of the block restated in float64 with torch ops (LayerNorm, the qkv bias, softmax attention
    with the causal mask, erf GELU, gamma)."""
    _, B, n, causal = BLOCKS[kind]
    P = {k: p.detach().double().requires_grad_(True) for k, p in blk.named_parameters()}
    t = {f: P[nm] for f, nm in _names(blk).items()}
    if isinstance(blk, M.VideoMAEBlock):
        H, scale, eps1, eps2 = blk.attn.num_heads, blk.attn.scale, blk.norm1.eps, blk.norm2.eps
        qb, vb = P["attn.q_bias"], P["attn.v_bias"]
        t["qkvb"] = torch.cat([qb, torch.zeros_like(qb), vb])
    else:
        a = blk.pre_norm_mha[1]
        H, scale, eps1, eps2 = a.num_heads, a.scaling, blk.pre_norm_mha[0].eps, blk.pre_norm_ffn[0].eps
    x, dy = _inputs(kind, t["n1w"].shape[0])
    x = x.double().requires_grad_(True)
    D = x.shape[1]
    d = D // H
    h = F.layer_norm(x, (D,), t["n1w"], t["n1b"], eps1)
    qkv = h @ t["qkvw"].t() + t["qkvb"]
    q, k, v = (qkv[:, i * D:(i + 1) * D].reshape(B, n, H, d).transpose(1, 2) for i in range(3))
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(n, n, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B * n, D)
    o = a @ t["projw"].t() + t["projb"]
    x1 = x + (o * t["g1"] if "g1" in t else o)
    h2 = F.layer_norm(x1, (D,), t["n2w"], t["n2b"], eps2)
    f = F.gelu(h2 @ t["fc1w"].t() + t["fc1b"]) @ t["fc2w"].t() + t["fc2b"]
    y = x1 + (f * t["g2"] if "g2" in t else f)
    y.backward(dy.double())
    return y.detach(), x.grad, {k: p.grad for k, p in P.items()}


@pytest.fixture(scope="module", params=sorted(BLOCKS))
def kind(request):
    return request.param


@pytest.fixture(scope="module")
def bf16_and_ref(kind):
    blk = _make(kind)
    return _run(blk, kind), _ref64(blk, kind)


def _errors(got, ref, kind):
    x, dy = _inputs(kind, got[0].shape[1])
    (y1, dx1, g1), (y0, dx0, g0) = got, ref
    r = {"y": _rel(y1 - x, y0 - x.to(y0.dtype)), "dx": _rel(dx1 - dy, dx0 - dy.to(dx0.dtype))}
    r.update({k: _rel(g1[k], g0[k]) for k in g0})
    return r


def test_bf16_block_matches_float64(cuda_lib, kind, bf16_and_ref):
    """The yardstick: the bf16 block against the float64 restatement."""
    r = _errors(*bf16_and_ref, kind)
    print(f"{kind} bf16 vs float64:", {k: round(v, 4) for k, v in r.items()})
    bad = {k: v for k, v in r.items() if v > 1e-2}
    assert not bad, bad


@pytest.mark.parametrize("mode", sorted(MODES))
def test_block_against_bf16_and_float64(cuda_lib, kind, bf16_and_ref, mode):
    got = _run(_make(kind, mode), kind)
    for against, ref in (("bf16", bf16_and_ref[0]), ("float64", bf16_and_ref[1])):
        r = _errors(got, ref, kind)
        print(f"{kind} {mode} FP8 vs {against}:", {k: round(v, 4) for k, v in r.items()})
        assert r["y"] <= OUT_BOUND, r
        bad = {k: v for k, v in r.items() if k != "y" and v > GRAD_BOUND[mode]}
        assert not bad, bad
        assert r["y"] > 0 and not torch.equal(got[0], bf16_and_ref[0][0])     # not the bf16 bits: the FP8 path ran
    if mode == "token_wgrad":
        yt, dxt, gt = _run(_make(kind, "token"), kind)
        assert torch.equal(got[0], yt) and torch.equal(got[1], dxt)
        names = _names(BLOCKS[kind][0]())
        weights = {names[f] for f in ("qkvw", "projw", "fc1w", "fc2w")}
        for k in gt:
            if k not in weights:
                assert torch.equal(got[2][k], gt[k]), k
        for k in weights:
            r = _rel(got[2][k], bf16_and_ref[0][2][k])
            assert 0 < r <= WGRAD_BOUND and not torch.equal(got[2][k], gt[k]), (k, r)


@pytest.mark.parametrize("mode", sorted(MODES))
def test_checkpointed_block_is_bit_identical_and_off_gives_bf16_bits(cuda_lib, kind, bf16_and_ref, mode):
    y1, dx1, g1 = _run(_make(kind, mode, with_cp=True), kind)
    blk = _make(kind, mode)
    y0, dx0, g0 = _run(blk, kind)
    assert torch.equal(y1, y0) and torch.equal(dx1, dx0)
    for k in g0:
        assert torch.equal(g1[k], g0[k]), k
    assert M.set_fp8(blk, False) == 1
    y2, dx2, g2 = _run(blk, kind)
    yb, dxb, gb = bf16_and_ref[0]
    assert torch.equal(y2, yb) and torch.equal(dx2, dxb)
    for k in gb:
        assert torch.equal(g2[k], gb[k]), k


# ------------------------------------------------------------------------------------------------ InternVideo1
def _iv1(mode=None):
    from internvideo_b200.videomae_v1 import PretrainVisionTransformer
    z = np.load(GOLD / "iv1_videomae.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    model = PretrainVisionTransformer(norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), **cfg)
    model.load_state_dict({k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}, strict=True)
    model = model.bfloat16().cuda().train()
    if mode is not None:
        assert M.set_fp8(model, True, **MODES[mode]) == cfg["encoder_depth"] + cfg["decoder_depth"]
    images = torch.from_numpy(z["images"]).cuda().to(bf16)
    mask = torch.from_numpy(z["mask"]).cuda()
    return z, model, images, mask


@pytest.mark.parametrize("mode", ["token", "token_wgrad"])
def test_iv1_videomae_golden_in_fp8(cuda_lib, mode):
    """The loss within 2u(E4M3) relative of the reference's, every gradient within the gradient bound."""
    from internvideo_b200 import videomae_v1 as v1
    z, model, images, mask = _iv1(mode)
    loss = v1.pretrain_loss(model, images, mask, normalize_target=True)
    ref = float(z["loss"])
    print(f"IV1 {mode}: loss {float(loss):.5f}, reference {ref:.5f}")
    assert abs(float(loss) - ref) <= OUT_BOUND * abs(ref)
    loss.backward()
    gr = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("g/")}
    gmax = max(float(g.norm()) for g in gr.values())
    r = {k: _rel(p.grad.float().cpu(), gr[k]) for k, p in model.named_parameters() if float(gr[k].norm()) >= 1e-5 * gmax}
    print(f"IV1 {mode} gradients, worst:", sorted(r.items(), key=lambda kv: -kv[1])[:4])
    bad = {k: v for k, v in r.items() if v > GRAD_BOUND[mode]}
    assert not bad, bad


@pytest.mark.parametrize("mode", ["token", "token_wgrad"])
def test_text_tower_golden_in_fp8(cuda_lib, mode):
    from internvideo_b200.text_modules import TextTransformer
    from oracle import text_tower
    cfg, sd, z = text_tower.load(GOLD / "text_tower.npz")
    tower = TextTransformer(cfg, cfg["projection_dim"])
    tower.load_state_dict(sd, strict=True)
    tower = tower.bfloat16().cuda()
    assert M.set_fp8(tower, True, **MODES[mode]) == cfg["n_transformer_layers"]
    ids = torch.from_numpy(z["ids"]).cuda()
    pooled = tower(ids)
    every = tower(ids[:text_tower.ALL_TOKENS_ROWS], return_all_tokens=True)
    rp, ra = _rel(pooled, torch.from_numpy(z["pooled"]).cuda()), _rel(every, torch.from_numpy(z["all_tokens"]).cuda())
    wp, wa = (w.cuda() for w in text_tower.loss_weights(pooled.shape, every.shape))
    ((pooled.float() * wp).sum() + (every.float() * wa).sum()).backward()
    r = {k: _rel(p.grad, torch.from_numpy(z["g/" + k]).cuda()) for k, p in tower.named_parameters()}
    print(f"text tower {mode}: pooled {rp:.4f}, all tokens {ra:.4f}; gradients, worst:",
          sorted(r.items(), key=lambda kv: -kv[1])[:4])
    assert 0 < rp <= OUT_BOUND and 0 < ra <= OUT_BOUND
    bad = {k: v for k, v in r.items() if v > GRAD_BOUND[mode]}
    assert not bad, bad


def _iv1_losses(mode, steps=40):
    from internvideo_b200 import videomae_v1 as v1
    from internvideo_b200.engine import PretrainEngine
    _, model, images, mask = _iv1(mode)
    eng = PretrainEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.05, clip_grad=0.0)
    losses = []
    for _ in range(steps):
        eng.zero_grad()
        loss = v1.pretrain_loss(model, images, mask)
        loss.backward()
        eng.step()
        losses.append(float(loss))
    return losses


def _text_losses(mode, steps=40):
    """Training steps of the text_tower.npz tower towards a fixed random target of its pooled output (MSE)."""
    from internvideo_b200.engine import PretrainEngine
    from internvideo_b200.text_modules import TextTransformer
    from oracle import text_tower
    cfg, sd, z = text_tower.load(GOLD / "text_tower.npz")
    tower = TextTransformer(cfg, cfg["projection_dim"])
    tower.load_state_dict(sd, strict=True)
    tower = tower.bfloat16().cuda().train()
    if mode is not None:
        M.set_fp8(tower, True, **MODES[mode])
    ids = torch.from_numpy(z["ids"]).cuda()
    target = torch.randn(ids.shape[0], cfg["projection_dim"], device="cuda",
                         generator=torch.Generator(device="cuda").manual_seed(2))
    eng = PretrainEngine(tower, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.0, clip_grad=0.0)
    losses = []
    for _ in range(steps):
        eng.zero_grad()
        loss = (tower(ids).float() - target).square().mean()
        loss.backward()
        eng.step()
        losses.append(float(loss))
    return losses


@pytest.mark.parametrize("tower", ["iv1", "text"])
@pytest.mark.parametrize("mode", ["token", "token_wgrad"])
def test_loss_drops_like_bf16(cuda_lib, tower, mode):
    """40 steps on one fixed batch drop the FP8 loss at least 90 % as far as the bf16 loss (tests/test_fp8_modes_gpu.py's
    criterion for the student)."""
    run = _iv1_losses if tower == "iv1" else _text_losses
    bf, f8 = run(None), run(mode)
    print(f"{tower}: loss bf16 {bf[0]:.4f} -> {bf[-1]:.4f}, {mode} FP8 {f8[0]:.4f} -> {f8[-1]:.4f}")
    assert all(np.isfinite(f8)) and bf[0] - bf[-1] > 0
    assert f8[0] - f8[-1] >= 0.9 * (bf[0] - bf[-1]), (f8[0] - f8[-1], bf[0] - bf[-1])


@pytest.mark.parametrize("mode", ["token", "token_wgrad"])
def test_gradient_sink_matches_autograd(cuda_lib, mode):
    """The engine's direct gradients (wgrad GEMMs accumulating into the flat gradient) against autograd's, to the bound
    the bf16 and RMSNorm FP8 sink tests use."""
    from internvideo_b200 import videomae_v1 as v1
    from internvideo_b200.engine import PretrainEngine
    flats = []
    for direct in (False, True):
        _, model, images, mask = _iv1(mode)
        eng = PretrainEngine(model, lr=1e-3, clip_grad=0.0, direct_grads=direct)
        eng.zero_grad()
        v1.pretrain_loss(model, images, mask).backward()
        flats.append(eng.flat_grad.float().clone())
    rel = float((flats[1] - flats[0]).norm() / flats[0].norm())
    assert float(flats[0].norm()) > 0 and rel < 2e-3, rel


def test_iv1_fp8_step_replays_in_a_cuda_graph(cuda_lib):
    """The per-token FP8 IV1 step (forward, backward, AdamW) captured in engine.GraphedStep replays with the eager step's
    loss; both arms start from the same model and take one warm-up step.  8 fp32 ulps are allowed, as for the student's
    step."""
    from internvideo_b200 import videomae_v1 as v1
    from internvideo_b200.engine import GraphedStep, PretrainEngine
    arms = []
    for _ in range(2):
        _, model, images, mask = _iv1("token")
        eng = PretrainEngine(model, lr=1e-3, clip_grad=0.0)
        n_masked = int(mask[0].sum())                      # given, so the captured step reads nothing to the host

        def step(v, model=model, eng=eng, mask=mask, n_masked=n_masked):
            eng.zero_grad()
            loss = v1.pretrain_loss(model, v, mask, n_masked=n_masked)
            loss.backward()
            eng.step()
            return loss
        arms.append((step, images))
    step, images = arms[0]
    step(images)
    loss_eager = float(step(images))
    step, images = arms[1]
    graphed = GraphedStep(step, [images.clone()], warmup=1)
    loss_graph = float(graphed(images)[0])
    torch.cuda.synchronize()
    print(f"IV1 FP8 step: eager loss {loss_eager!r}, graph replay {loss_graph!r}")
    assert loss_eager == loss_eager and abs(loss_graph - loss_eager) <= 8 * 2.0 ** -23 * abs(loss_eager)


# ------------------------------------------------------------------------------------------------ inference
def _bert():
    from internvideo_b200.bert_modules import BertModel
    from oracle import bert_text
    cfg, sd, _, z = bert_text.load(GOLD / "bert_text.npz")
    model = BertModel(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.bfloat16().cuda().eval().requires_grad_(False)
    ids, mask = (torch.from_numpy(z[k]).cuda() for k in ("ids", "mask"))
    return model, ids, mask, z


def _last(model, ids, mask):
    return model(ids, attention_mask=mask, mode="text").last_hidden_state


def test_bert_fp8_inference_against_bf16(cuda_lib):
    """last_hidden_state, each caption's valid rows and the pooled rows within 2u(E4M3) of bf16 (and of the reference);
    switching off gives the bf16 bits back."""
    from oracle import bert_text
    model, ids, mask, z = _bert()
    base = _last(model, ids, mask)
    assert M.set_fp8_inference(model) == model.config.fusion_layer
    f8 = _last(model, ids, mask)
    r = {"last": _rel(f8, base), "pooled": _rel(f8[:, 0], base[:, 0]),
         "reference": _rel(f8, torch.from_numpy(z["last_hidden_state"]).cuda())}
    r.update({f"caption {b}": _rel(f8[b, :n], base[b, :n]) for b, n in enumerate(bert_text.LENGTHS)})
    print("BERT FP8 inference vs bf16:", {k: round(v, 4) for k, v in r.items()})
    assert all(0 < v <= OUT_BOUND for v in r.values()), r
    assert M.set_fp8_inference(model, False) == model.config.fusion_layer
    assert torch.equal(_last(model, ids, mask), base)


def test_bert_fp8_padded_rows_behave_as_in_bf16(cuda_lib):
    """Per-token scales keep every row to itself, as bf16 does: other ids in the padding leave the valid rows'
    bits; the padded rows are computed (finite, within the bound of bf16's); a bad mask makes only its captions NaN."""
    from oracle import bert_text
    model, ids, mask, _ = _bert()
    base = _last(model, ids, mask)
    M.set_fp8_inference(model)
    f8 = _last(model, ids, mask)
    ids2 = torch.where(mask.bool(), ids, torch.full_like(ids, 7))
    f8b = _last(model, ids2, mask)
    for b, n in enumerate(bert_text.LENGTHS):
        assert torch.equal(f8b[b, :n], f8[b, :n]), b
        if n < ids.shape[1]:
            assert bool(torch.isfinite(f8[b, n:].float()).all()) and _rel(f8[b, n:], base[b, n:]) <= OUT_BOUND, b
    bad = mask.clone()
    bad[1, 5] = 0
    bad[2] = 0
    out = _last(model, ids, bad)
    assert bool(torch.isnan(out[1:3]).all())
    assert torch.equal(out[0], f8[0]) and torch.equal(out[3], f8[3])


def test_bert_weight_changed_in_place_is_requantised(cuda_lib):
    model, ids, mask, _ = _bert()
    M.set_fp8_inference(model)
    before = _last(model, ids, mask)
    with torch.no_grad():
        model.encoder.layer[0].intermediate.dense.weight.mul_(0.5)
    after = _last(model, ids, mask)
    M.set_fp8_inference(model, False)
    M.set_fp8_inference(model)                             # a fresh quantisation of every weight
    assert not torch.equal(after, before) and torch.equal(_last(model, ids, mask), after)


def test_text_tower_fp8_inference(cuda_lib):
    """The frozen text tower under set_fp8_inference: within 2u(E4M3) of bf16, causal attention kept in bf16 with
    attention=True too, a forward that needs a gradient refused, and switching off gives the bf16 bits back."""
    from internvideo_b200.text_modules import TextTransformer
    from oracle import text_tower
    cfg, sd, z = text_tower.load(GOLD / "text_tower.npz")
    tower = TextTransformer(cfg, cfg["projection_dim"])
    tower.load_state_dict(sd, strict=True)
    tower = tower.bfloat16().cuda()
    ids = torch.from_numpy(z["ids"]).cuda()
    with torch.no_grad():
        base = tower(ids)
    assert M.set_fp8_inference(tower) == cfg["n_transformer_layers"]
    with pytest.raises(_lib.IvbError, match="has no gradient"):
        tower(ids)                                         # the parameters still require grad: a training forward
    tower.requires_grad_(False)
    f8 = tower(ids)
    assert 0 < _rel(f8, base) <= OUT_BOUND, _rel(f8, base)
    M.set_fp8_inference(tower, False)
    M.set_fp8_inference(tower, True, attention=True)
    assert torch.equal(tower(ids), f8)                     # causal: no FP8 attention
    M.set_fp8_inference(tower, False)
    assert torch.equal(tower(ids), base)
