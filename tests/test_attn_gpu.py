"""wgmma attention forward/backward vs fp32 softmax attention on the same bf16 inputs (gpu)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def ref_attn(q, k, v, B, n, H, d, scale):
    qf = q.float().reshape(B, n, H, d).transpose(1, 2)
    kf = k.float().reshape(B, n, H, d).transpose(1, 2)
    vf = v.float().reshape(B, n, H, d).transpose(1, 2)
    s = (qf * scale) @ kf.transpose(-2, -1)
    p = s.softmax(-1)
    o = (p @ vf).transpose(1, 2).reshape(B * n, H * d)
    lse2 = torch.logsumexp(s, -1) * math.log2(math.e)
    return o, lse2


CASES = [(2, 417, 16, 88), (1, 64, 2, 64), (2, 209, 6, 64), (1, 1025, 4, 64), (1, 833, 5, 128),
         (3, 13, 2, 64), (1, 128, 1, 88), (1, 1568, 2, 88), (1, 129, 3, 128),
         # grids larger than one wave, ragged last query / key tiles, 1, 2, 4 and 9 key tiles per block
         (5, 417, 16, 88), (40, 64, 4, 64), (6, 300, 25, 64), (2, 1025, 16, 64), (20, 144, 8, 128), (3, 257, 40, 32)]


@pytest.mark.parametrize("B,n,H,d", CASES)
def test_attn_fwd(cuda_lib, B, n, H, d):
    ll = cuda_lib
    torch.manual_seed(B * 1000 + n)
    D = H * d
    qkv = (torch.randn(B * n, 3 * D, device="cuda") * 1.5).to(torch.bfloat16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    scale = d ** -0.5
    out, lse = ll.attn_fwd(q, k, v, B, n, H, d, scale)
    torch.cuda.synchronize()
    o_ref, lse_ref = ref_attn(q, k, v, B, n, H, d, scale)
    assert _rel(out, o_ref) < 8e-3, _rel(out, o_ref)
    assert (lse - lse_ref).abs().max().item() < 2e-2


def test_attn_fwd_rescale_path(cuda_lib):
    """Scores that grow along the key axis force the lazy O-rescale branch."""
    ll = cuda_lib
    B, n, H, d = 1, 300, 2, 64
    D = H * d
    torch.manual_seed(1)
    q = torch.randn(B * n, D, device="cuda")
    k = torch.randn(B * n, D, device="cuda")
    ramp = torch.linspace(0, 6, n, device="cuda")[:, None]
    k = k + ramp * q.mean(0, keepdim=True).sign() * 0.5
    q = (q.abs() * q.mean(0, keepdim=True).sign()).to(torch.bfloat16)
    k = k.to(torch.bfloat16)
    v = torch.randn(B * n, D, device="cuda").to(torch.bfloat16)
    out, lse = ll.attn_fwd(q, k, v, B, n, H, d, 0.5)
    o_ref, lse_ref = ref_attn(q, k, v, B, n, H, d, 0.5)
    assert _rel(out, o_ref) < 8e-3
    assert (lse - lse_ref).abs().max().item() < 5e-2


@pytest.mark.parametrize("B,n,H,d", [(2, 417, 16, 88), (1, 64, 2, 64), (2, 209, 6, 64), (1, 1025, 2, 64),
                                     (1, 833, 3, 128), (3, 13, 2, 64), (1, 200, 1, 88),
                                     # more (clip, head, 128-row) work items than SMs: the persistent kernel's
                                     # cross-item path (next item's operands prefetched, rings and barrier phases
                                     # continuing across items) with an odd, an even and a single tile per item
                                     (5, 417, 16, 88), (6, 256, 25, 64), (40, 64, 4, 64)])
def test_attn_bwd(cuda_lib, B, n, H, d):
    ll = cuda_lib
    torch.manual_seed(B * 77 + n)
    D = H * d
    qkv = (torch.randn(B * n, 3 * D, device="cuda")).to(torch.bfloat16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    scale = d ** -0.5
    out, lse = ll.attn_fwd(q, k, v, B, n, H, d, scale)
    dout = torch.randn(B * n, D, device="cuda").to(torch.bfloat16)
    dqkv = torch.zeros(B * n, 3 * D, device="cuda", dtype=torch.bfloat16)
    ll.attn_bwd(q, k, v, out, dout, lse, B, n, H, d, scale, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])
    torch.cuda.synchronize()
    qr = q.float().requires_grad_(True); kr = k.float().requires_grad_(True); vr = v.float().requires_grad_(True)
    o_ref, _ = ref_attn(qr, kr, vr, B, n, H, d, scale)
    o_ref.backward(dout.float())
    assert _rel(dqkv[:, 2 * D:], vr.grad) < 1e-2, ("dv", _rel(dqkv[:, 2 * D:], vr.grad))
    assert _rel(dqkv[:, :D], qr.grad) < 1.5e-2, ("dq", _rel(dqkv[:, :D], qr.grad))
    assert _rel(dqkv[:, D:2 * D], kr.grad) < 1.5e-2, ("dk", _rel(dqkv[:, D:2 * D], kr.grad))


@pytest.mark.parametrize("B,n,H,d", [(2, 417, 16, 88), (3, 13, 2, 64), (1, 1025, 4, 64)])
def test_pool_attention_single_query(cuda_lib, B, n, H, d):
    """AttentionPoolingBlock core: one query per clip (internvideo2_pretrain.py:61-76)."""
    ll = cuda_lib
    torch.manual_seed(n)
    D = H * d
    q = torch.randn(B, D, device="cuda").to(torch.bfloat16)
    k = torch.randn(B * n, D, device="cuda").to(torch.bfloat16)
    v = torch.randn(B * n, D, device="cuda").to(torch.bfloat16)
    scale = d ** -0.5
    out, probs = ll.pool_attn_fwd(q, k, v, B, n, H, d, scale)
    qr = q.float().requires_grad_(True); kr = k.float().requires_grad_(True); vr = v.float().requires_grad_(True)
    s = torch.einsum("bhd,bkhd->bhk", qr.view(B, H, d) * scale, kr.view(B, n, H, d))
    p = s.softmax(-1)
    o = torch.einsum("bhk,bkhd->bhd", p, vr.view(B, n, H, d)).reshape(B, D)
    assert _rel(out, o) < 8e-3
    assert (probs - p).abs().max().item() < 1e-3
    do = torch.randn(B, D, device="cuda").to(torch.bfloat16)
    o.backward(do.float())
    dq, dk, dv = ll.pool_attn_bwd(q, k, v, probs, do, B, n, H, d, scale)
    assert _rel(dq, qr.grad) < 1e-2 and _rel(dk, kr.grad) < 1e-2 and _rel(dv, vr.grad) < 1e-2


def test_flash_attention_module_seam(cuda_lib):
    """The reference's attention seam: FlashAttention()(qkv[B,S,3,H,d]) -> (out[B,S,H,d], None), forward and backward
    (flash_attention_class.py:27-50), plus the refusals for what the pre-training path never passes."""
    from internvideo_b200.patch import FlashAttention
    torch.manual_seed(4)
    B, S, H, d = 2, 209, 6, 64
    qkv = torch.randn(B, S, 3, H, d, device="cuda").to(torch.bfloat16).requires_grad_(True)
    fa = FlashAttention(attention_dropout=0.0)
    out, none = fa(qkv)
    assert none is None and tuple(out.shape) == (B, S, H, d)
    dout = torch.randn_like(out)
    out.backward(dout)
    ref_in = qkv.detach().float().requires_grad_(True)
    flat = ref_in.reshape(B * S, 3 * H * d)
    D = H * d
    o_ref, _ = ref_attn(flat[:, :D], flat[:, D:2 * D], flat[:, 2 * D:], B, S, H, d, d ** -0.5)
    o_ref.backward(dout.float().reshape(B * S, D))
    assert _rel(out.reshape(B * S, D), o_ref) < 8e-3
    assert _rel(qkv.grad, ref_in.grad) < 1.5e-2
    with pytest.raises(NotImplementedError):
        fa(qkv, key_padding_mask=torch.ones(B, S, dtype=torch.bool, device="cuda"))
    with pytest.raises(NotImplementedError):
        fa(qkv, causal=True)
