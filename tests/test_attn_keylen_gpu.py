"""The key-length attention forward (ivb_attn_fwd_keylen) on the H100, tile by tile against float64 attention whose
keys >= kv_len[b] are masked: the padded keys hold large finite values (+-1e4), so an unmasked one would dominate
its row.  With every kv_len = n it gives ivb_attn_fwd's bits; it is bitwise repeatable; an entry outside [1, n] makes
that clip's rows NaN and leaves the other clips' bits alone."""
import math

import pytest
import torch

from attn_ref import tile_errors, worst
from internvideo_b200 import _lib

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# tile error of O and max |lse2 error|: the non-causal forward's limits (tests/test_attn_gpu.py)
LIMITS = {"o": 1.2e-2, "lse": 1.0e-5}

# (B, n, H, d): 64 captions of 40 tokens of BERT-large's 16 heads of 64 (one key tile); the text tower's 77 tokens (two
# key tiles); 417 tokens with head dim 88 (seven key tiles, a zero-filled head tail); 193 tokens with head dim 40
CASES = [(64, 40, 16, 64), (4, 77, 8, 64), (2, 417, 16, 88), (3, 193, 4, 40)]


def _randn(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


def _lengths(B, n, shift):
    """kv_len [B] cycling through 1, 63, 64, 65 and n (those <= n), starting at the shift-th."""
    vals = [v for v in (1, 63, 64, 65, n) if v <= n]
    return torch.tensor([vals[(b + shift) % len(vals)] for b in range(B)], device="cuda", dtype=torch.int32), len(vals)


def _operands(B, n, H, d, kv, seed):
    """q, k, v: views of one [B*n, 3*H*d] bf16 buffer; the padded keys of k and v are +-1e4."""
    D = H * d
    qkv = _randn(B * n, 3 * D, seed=seed).to(bf16)
    big = torch.where(_randn(n, 2 * D, seed=seed + 1) > 0, 1e4, -1e4).to(bf16)
    for b, kb in enumerate(kv.tolist()):
        qkv[b * n + kb:(b + 1) * n, D:] = big[kb:]
    return qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]


def _masked_ref(q, k, v, B, n, H, d, scale, kv):
    """float64 softmax(scale q k^T) v per clip with keys >= kv[b] at -inf.  Returns (O [B*n, H*d], lse2 [B, H, n])."""
    heads = lambda x, b: x[b * n:(b + 1) * n].double().reshape(n, H, d).transpose(0, 1)  # noqa: E731
    out = torch.empty((B * n, H * d), dtype=torch.float64, device="cuda")
    lse2 = torch.empty((B, H, n), dtype=torch.float64, device="cuda")
    for b, kb in enumerate(kv.tolist()):
        s = heads(q, b) @ heads(k, b).transpose(-2, -1) * scale
        s[..., kb:] = float("-inf")
        lse = torch.logsumexp(s, -1, keepdim=True)
        out[b * n:(b + 1) * n] = (torch.exp(s - lse) @ heads(v, b)).transpose(0, 1).reshape(n, H * d)
        lse2[b] = lse.squeeze(-1) / math.log(2.0)
    return out, lse2


@pytest.mark.parametrize("B,n,H,d", CASES)
def test_keylen_attention_matches_fp64(cuda_lib, B, n, H, d):
    scale = d ** -0.5
    shifts = _lengths(B, n, 0)[1]
    for shift in range(shifts):          # every length in every clip position the shape has
        kv, _ = _lengths(B, n, shift)
        q, k, v = _operands(B, n, H, d, kv, seed=17 * shift + n)
        out, lse = cuda_lib.attn_fwd(q, k, v, B, n, H, d, scale, kv_len=kv)
        o_ref, lse_ref = _masked_ref(q, k, v, B, n, H, d, scale, kv)
        e, (b, h, band) = worst(tile_errors(out, o_ref, B, n, H, d))
        assert e <= LIMITS["o"], f"o: {e:.3e} at clip {b} (kv_len {int(kv[b])}), head {h}, rows from {64 * band}"
        e_lse, where = worst((lse.double() - lse_ref).abs())
        assert e_lse <= LIMITS["lse"], (e_lse, where)
        again, lse2 = cuda_lib.attn_fwd(q, k, v, B, n, H, d, scale, kv_len=kv)
        assert torch.equal(out, again) and torch.equal(lse, lse2)


@pytest.mark.parametrize("B,n,H,d", CASES)
def test_full_lengths_give_the_unmasked_bits(cuda_lib, B, n, H, d):
    q, k, v = _operands(B, n, H, d, torch.full((B,), n, dtype=torch.int32), seed=5)
    full = torch.full((B,), n, device="cuda", dtype=torch.int32)
    out, lse = cuda_lib.attn_fwd(q, k, v, B, n, H, d, d ** -0.5, kv_len=full)
    ref, ref_lse = cuda_lib.attn_fwd(q, k, v, B, n, H, d, d ** -0.5)
    assert torch.equal(out, ref) and torch.equal(lse, ref_lse)


def test_out_of_range_lengths_poison_only_their_clip(cuda_lib):
    B, n, H, d = 5, 77, 8, 64
    q, k, v = _operands(B, n, H, d, torch.full((B,), n, dtype=torch.int32), seed=9)
    kv = torch.tensor([n, 0, n + 1, -3, 30], device="cuda", dtype=torch.int32)
    out, lse = cuda_lib.attn_fwd(q, k, v, B, n, H, d, 0.125, kv_len=kv)
    ref, ref_lse = cuda_lib.attn_fwd(q, k, v, B, n, H, d, 0.125, kv_len=torch.tensor([n] * 4 + [30], device="cuda",
                                                                                       dtype=torch.int32))
    rows = out.reshape(B, n, H * d)
    assert bool(torch.isnan(rows[1:4]).all()) and bool(torch.isnan(lse[1:4]).all())
    for b in (0, 4):
        assert torch.equal(rows[b], ref.reshape(B, n, H * d)[b]) and torch.equal(lse[b], ref_lse[b])


def test_binding_refuses_bad_key_lengths(cuda_lib):
    q = torch.zeros(2 * 40, 128, device="cuda", dtype=bf16)
    kv = torch.full((2,), 40, device="cuda", dtype=torch.int32)
    with pytest.raises(_lib.IvbError, match="causal"):
        cuda_lib.attn_fwd(q, q, q, 2, 40, 2, 64, 0.125, causal=True, kv_len=kv)
    with pytest.raises(_lib.IvbError, match="kv_len must be a contiguous"):
        cuda_lib.attn_fwd(q, q, q, 2, 40, 2, 64, 0.125, kv_len=kv[:1])
    with pytest.raises(_lib.IvbError, match="kv_len: expected dtype"):
        cuda_lib.attn_fwd(q, q, q, 2, 40, 2, 64, 0.125, kv_len=kv.long())
