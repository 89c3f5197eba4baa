"""The float64 attention reference and the per-tile error metric of tests/attn_ref.py, checked on the CPU: the
reference against autograd of a naive float64 attention, and the metric against an error that a global norm dilutes."""
import math

import pytest
import torch

from attn_ref import attn_ref_bwd, attn_ref_fwd, tile_errors, worst


def _naive(q, k, v, B, n, H, d, scale, causal=False, kv_len=None):
    """Attention written out with a [B, 1, n, n] additive mask: -inf above the diagonal (causal) and on the keys
    >= kv_len[b]."""
    qh, kh, vh = (t.reshape(B, n, H, d).transpose(1, 2) for t in (q, k, v))
    s = (qh @ kh.transpose(-2, -1)) * scale
    mask = torch.zeros(B, 1, n, n, dtype=s.dtype)
    if causal:
        mask += torch.full((n, n), float("-inf"), dtype=s.dtype).triu(1)
    for b, keys in enumerate(kv_len or ()):
        mask[b, ..., keys:] = float("-inf")
    s = s + mask
    o = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B * n, H * d)
    return o, torch.logsumexp(s, -1) / math.log(2)


def _operands(B, n, H, d):
    g = torch.Generator().manual_seed(n)
    q, k, v, dout = (torch.randn(B * n, H * d, generator=g, dtype=torch.float64) for _ in range(4))
    # strided views, as the kernels receive them
    qkv = torch.cat((q, k, v), 1)
    return qkv[:, :H * d], qkv[:, H * d:2 * H * d], qkv[:, 2 * H * d:], dout


@pytest.mark.parametrize("B,n,H,d,causal", [
    pytest.param(*shape, causal, id="-".join(map(str, shape)) + ("-causal" if causal else ""))
    for shape in [(1, 1, 1, 16), (2, 37, 3, 24), (3, 70, 2, 88)] for causal in (False, True)])
def test_reference_matches_autograd(B, n, H, d, causal):
    q, k, v, dout = _operands(B, n, H, d)
    scale = 0.7 * d ** -0.5
    o, lse2 = attn_ref_fwd(q, k, v, B, n, H, d, scale, causal=causal)
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    o_n, lse2_n = _naive(*leaves, B, n, H, d, scale, causal=causal)
    o_n.backward(dout)
    torch.testing.assert_close(o, o_n.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(lse2, lse2_n.detach(), rtol=1e-12, atol=1e-12)
    for got, leaf in zip(attn_ref_bwd(q, k, v, dout, B, n, H, d, scale, causal=causal), leaves):
        torch.testing.assert_close(got, leaf.grad, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("B,n,H,d", [(1, 1, 1, 16), (3, 37, 3, 24), (4, 70, 2, 88)])
def test_key_length_reference_matches_naive(B, n, H, d):
    """kv_len in {1, n} and one length in between; a clip with kv_len = 1 copies V row 0 into every row."""
    q, k, v, _ = _operands(B, n, H, d)
    kv = [(1, n, max(1, n // 2))[b % 3] for b in range(B)]
    o, lse2 = attn_ref_fwd(q, k, v, B, n, H, d, 0.6, kv_len=torch.tensor(kv, dtype=torch.int32))
    o_n, lse2_n = _naive(q, k, v, B, n, H, d, 0.6, kv_len=kv)
    torch.testing.assert_close(o, o_n, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(lse2, lse2_n, rtol=1e-12, atol=1e-12)
    assert torch.equal(o[:n], v[:1].expand(n, -1))
    full, full_lse = attn_ref_fwd(q, k, v, B, n, H, d, 0.6)
    for b in (b for b in range(B) if kv[b] == n):
        assert torch.equal(o[b * n:(b + 1) * n], full[b * n:(b + 1) * n]) and torch.equal(lse2[b], full_lse[b])


def test_tile_errors_flag_one_band_the_global_norm_dilutes():
    B, n, H, d = 5, 417, 16, 88
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(B * n, H * d, generator=g, dtype=torch.float64)
    got = ref.clone()
    b, h, band = 3, 11, 6                  # rows 384..416: the ragged last band of 33 rows
    rows = slice(b * n + 64 * band, b * n + min(n, 64 * band + 64))
    got[rows, h * d:(h + 1) * d] *= 1.05
    errs = tile_errors(got, ref, B, n, H, d)
    assert errs.shape == (B, H, 7)
    e, where = worst(errs)
    assert where == (b, h, band)
    assert 0.04 < e < 0.06, e
    assert int((errs > 0).sum()) == 1
    glob = float((got - ref).norm() / ref.norm())
    assert glob < 5e-3, glob               # what a single relative norm over the tensor sees


def test_tile_errors_normalise_by_the_whole_head():
    """A band whose reference is all zero reads its error relative to the head's rms, not as infinity."""
    B, n, H, d = 1, 128, 2, 16
    ref = torch.ones(B * n, H * d, dtype=torch.float64)
    ref[:64, :d] = 0.0
    got = ref.clone()
    got[:64, :d] = 0.01
    errs = tile_errors(got, ref, B, n, H, d)
    assert torch.isfinite(errs).all()
    assert abs(float(errs[0, 0, 0]) - 0.01 * math.sqrt(2)) < 1e-12   # the head's rms is sqrt(1/2)
