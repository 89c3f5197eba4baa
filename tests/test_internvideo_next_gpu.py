"""InternVideo-Next's encoder on the H100 (gpu):
  - the pre-norm im2col at the real shape (B = 2, 16 x 224^2, K = 588) element by element against float64: the row's
    r within K 2^-24 + 2^-21 relative of the float64 rsqrt (an fp32 sum of K positive squares, then the approximate
    rsqrt), and every output within two bf16 roundings (the normalised pixel's and the product's, each at most 2^-8
    relative: 2^-7 + 2^-15 together) of w[pi(k)] a_k r at the kernel's r; padding columns exactly zero;
  - the norm_before weight gradient against a float64 sum of dcols * bf16(a r) over the rows, within 128 2^-24 of the
    sum of the terms' magnitudes (the kernel's fp32 sums chain at most 16 rows per warp, 8 warps and one slot per 128
    rows: fewer than 128 additions for the 64 slots here), and the same bits on a second run;
  - the tiny encoder against tests/golden/internvideo_next.npz, the unmodified reference's fp32 outputs and sampled
    gradients: both outputs within 1e-2 and every parameter gradient within 3e-2 relative (Frobenius), except the
    pooling projector's k bias and norm1_k bias: each shifts every key by the same vector, so every score of the one
    query by the same amount, which the softmax cancels; their gradients are zero up to rounding in both, and are held
    below 1e-2 of the gradient of the weight beside them (ZERO_GRADS); checkpointed blocks give the same bits as plain
    ones;
  - one large block at n = 4 100 (B = 1, 16 heads of 64) forward and backward against an fp32 torch statement of the
    block on the same bf16 inputs (output 1e-2, input and parameter gradients 3e-2 relative);
  - the large encoder at 16 x 224^2 against the fp32 restatement (oracle/internvideo_next.restate) on the same bf16
    weights and input: its error no larger than NEXT_FACTOR times the restatement's own error under bf16 autocast;
  - FP8 inference (set_fp8_inference) within OUT_BOUND of the bf16 output, the bound tests/test_fp8_layernorm_gpu.py
    holds the other towers to.
"""
from pathlib import Path

import pytest
import torch

from internvideo_b200 import internvideo_next as nx
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import modules as M
from oracle import internvideo_next as on

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden" / "internvideo_next.npz"
bf = torch.bfloat16
U_E4M3 = 2.0 ** -4
OUT_BOUND = 2 * U_E4M3
ZERO_GRADS = {"clip_projector.cross_attn.k_bias": "clip_projector.cross_attn.k.weight",
              "clip_projector.norm1_k.bias": "clip_projector.norm1_k.weight"}
NEXT_FACTOR = 3.0      # the port against fp32, over the restatement's own bf16-autocast error against fp32


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm())


def _video(B, T, S, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 3, T, S, S, device="cuda", generator=g)
    scale = 0.25 + torch.rand(B, 1, T, S // 14, 1, S // 14, 1, device="cuda", generator=g)
    return (x * scale.expand(-1, -1, -1, -1, 14, -1, 14).reshape(B, 1, T, S, S)).to(bf)


def _patches(video, P=14):
    """[B*T*L, C*P*P] float64 rows in the im2col's (c, dy, dx) column order (tubelet 1)."""
    B, C, T, H, W = video.shape
    v = video.double().reshape(B, C, T, H // P, P, W // P, P).permute(0, 2, 3, 5, 1, 4, 6)
    return v.reshape(B * T * (H // P) * (W // P), C * P * P)


def _pi(w, C=3, P=14):
    """norm_before's (dy dx c) weight in the im2col's (c, dy, dx) column order."""
    return w.reshape(P, P, C).permute(2, 0, 1).reshape(-1)


def _prenorm_operands(B=2, T=16, S=224, seed=0):
    video = _video(B, T, S, seed)
    N = T * (S // 14) ** 2
    idx = torch.arange(0, N + 1, device="cuda", dtype=torch.int32).repeat(B, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    w = (1 + 0.3 * torch.randn(588, device="cuda", generator=g)).to(bf)
    return video, idx, N, w


def test_im2col_prenorm_vs_fp64():
    video, idx, N, w = _prenorm_operands()
    cols, r = ll._im2col_prenorm(video, idx, 1, N, 1, 14, 592, w, eps=1e-6)
    torch.cuda.synchronize()
    a = _patches(video)
    r64 = torch.rsqrt(a.pow(2).mean(1) + 1e-6)
    assert float(((r.double() - r64).abs() / r64).max()) <= 588 * 2.0 ** -24 + 2.0 ** -21
    exact = _pi(w).double()[None, :] * a * r.double()[:, None]
    err = (cols[:, :588].double() - exact).abs()
    assert bool((err <= (2.0 ** -7 + 2.0 ** -15) * exact.abs()).all()), float((err / exact.abs()).max())
    assert torch.count_nonzero(cols[:, 588:]) == 0


def test_prenorm_wgrad_vs_fp64_and_deterministic():
    video, idx, N, w = _prenorm_operands(seed=5)
    cols, r = ll._im2col_prenorm(video, idx, 1, N, 1, 14, 592, w)
    g = torch.Generator(device="cuda").manual_seed(9)
    dcols = torch.randn(cols.shape, device="cuda", generator=g).to(bf)
    dw = ll._prenorm_wgrad(video, idx, 1, N, 1, 14, 592, r, dcols)
    dw2 = ll._prenorm_wgrad(video, idx, 1, N, 1, 14, 592, r, dcols)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2)
    xh = (_patches(video).float() * r[:, None]).to(bf).double()       # the kernel's bf16(a r)
    terms = dcols[:, :588].double() * xh
    ref, mag = terms.sum(0), terms.abs().sum(0)
    got = _pi(dw).double()
    assert bool(((got - ref).abs() <= 128 * 2.0 ** -24 * mag).all())


def _fixture_model(**kw):
    sd, z = on.load(GOLD)
    m = nx.InternVideo2(**on.NAIVE, **dict(on.CFG, **kw))
    m.load_state_dict(sd, strict=True)
    return m.to(bf).cuda(), z


def _run(m, x):
    tokens = m(x)
    pooled = m(x, projected=True)
    on.total_loss(tokens, pooled).backward()
    torch.cuda.synchronize()
    return tokens, pooled, {k: p.grad.clone() for k, p in m.named_parameters()}


def test_tiny_encoder_vs_fixture():
    m, z = _fixture_model()
    x = on.video().to(bf).cuda()
    tokens, pooled, grads = _run(m, x)
    assert tokens.shape == (2, 64, 128) and tokens.dtype == bf and pooled.shape == (2, 64)
    assert _rel(tokens, torch.from_numpy(z["tokens"])) <= 1e-2
    assert _rel(pooled, torch.from_numpy(z["pooled"])) <= 1e-2
    rel = {k: _rel(on.sample(g), torch.from_numpy(z["g/" + k])) for k, g in grads.items() if k not in ZERO_GRADS}
    print("tiny encoder: worst gradient", max((v, k) for k, v in rel.items()))
    assert not [k for k, v in rel.items() if v > 3e-2], sorted(rel.items(), key=lambda kv: -kv[1])[:5]
    for k, beside in ZERO_GRADS.items():
        assert float(grads[k].float().norm()) <= 1e-2 * float(grads[beside].float().norm()), k
    mc, _ = _fixture_model(use_checkpoint=True, checkpoint_num=2)
    assert all(b.with_cp for b in mc.blocks)
    t2, p2, g2 = _run(mc, x)
    assert torch.equal(t2, tokens) and torch.equal(p2, pooled)
    for k in grads:
        assert torch.equal(g2[k], grads[k]), k


def _drawn(model, prefix=""):
    """Sets every parameter from oracle/internvideo_next.draw_param (bf16), returns the fp32 state_dict of those values
    on the device."""
    sd = {}
    with torch.no_grad():
        for k, p in model.named_parameters():
            v = on.draw_param(prefix + k, tuple(p.shape))
            p.copy_(v)
            sd[k] = v.cuda()
    return sd


def test_large_block_n4100():
    D, H, n = 1024, 16, 4100
    torch.manual_seed(0)
    blk = M.Block(D, H, 4, qkv_bias=False, init_values=1e-5, qk_normalization=True, use_fused_mlp=False)
    sd = _drawn(blk, "blocks.0.")
    blk = blk.to(bf).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n, D, device="cuda", generator=g).to(bf).float().requires_grad_(True)
    wout = on.weights((n, D), 0.41).cuda()
    out = blk.forward_stream(x, 1, n)
    (out * wout).sum().backward()
    torch.cuda.synchronize()
    ref_sd = {"blocks.0." + k: v.requires_grad_(True) for k, v in sd.items()}
    xr = x.detach().clone().requires_grad_(True)
    ref = on.block(xr[None], ref_sd, "blocks.0.", H)[0]
    (ref * wout).sum().backward()
    assert _rel(out, ref) <= 1e-2
    assert _rel(x.grad, xr.grad) <= 3e-2
    for k, p in blk.named_parameters():
        assert _rel(p.grad, ref_sd["blocks.0." + k].grad) <= 3e-2, k


def test_large_encoder_vs_restatement():
    torch.manual_seed(0)
    m = nx.internvideo_next_large_patch14_224(**on.NAIVE, drop_path_rate=0.0)
    sd = _drawn(m)
    m = m.to(bf).cuda().eval()
    x = _video(1, 16, 224, seed=11)
    kw = dict(num_heads=16, pool_heads=16)
    with torch.no_grad():
        got = (m(x), m(x, projected=True))
        ref = [on.restate(sd, x.float(), projected=p, **kw) for p in (False, True)]
        with torch.autocast("cuda", dtype=bf):
            auto = [on.restate(sd, x.float(), projected=p, **kw) for p in (False, True)]
    for name, g_, r_, a_ in zip(("tokens", "pooled"), got, ref, auto):
        e_port, e_auto = _rel(g_, r_), _rel(a_, r_)
        print(f"large encoder {name}: port {e_port:.3e}, bf16 autocast {e_auto:.3e}, ratio {e_port / e_auto:.2f}")
        assert e_port <= NEXT_FACTOR * e_auto, (name, e_port, e_auto)


def test_fp8_inference():
    m, _ = _fixture_model()
    m.eval()
    x = on.video().to(bf).cuda()
    with torch.no_grad():
        ref = (m(x), m(x, projected=True))
        assert M.set_fp8_inference(m) == on.CFG["depth"]
        got = (m(x), m(x, projected=True))
        M.set_fp8_inference(m, False)
    for g_, r_ in zip(got, ref):
        assert _rel(g_, r_) <= OUT_BOUND
