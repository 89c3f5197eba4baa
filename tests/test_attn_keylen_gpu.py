"""The key-length attention forward (ivb_attn_fwd_keylen) on the H100: with every kv_len = n it gives ivb_attn_fwd's
bits at every head dim; an entry outside [1, n] makes that clip's rows NaN and leaves the other clips' bits alone; the
binding refuses what the kernel does not take.  Its comparison with the masked float64 reference, its exact masking
and its bitwise repeatability are the key-length form of tests/test_attn_gpu.py."""
import pytest
import torch

from internvideo_b200 import _lib

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# (B, n, H, d): 64 captions of 40 tokens of BERT-large's 16 heads of 64 (one key tile); the text tower's 77 tokens (two
# key tiles); 417 tokens with head dim 88 (seven key tiles, a zero-filled head tail); 193 tokens with head dim 40; and
# every head dim the ABI accepts at 190 tokens (a ragged key tile, a second block with one live warpgroup)
CASES = [(64, 40, 16, 64), (4, 77, 8, 64), (2, 417, 16, 88), (3, 193, 4, 40)]
HEAD_DIM_CASES = [(2, 190, 3, d) for d in range(16, 129, 8)]


def _randn(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


def _operands(B, n, H, d, kv, seed):
    """q, k, v: views of one [B*n, 3*H*d] bf16 buffer; the padded keys of k and v are +-1e4."""
    D = H * d
    qkv = _randn(B * n, 3 * D, seed=seed).to(bf16)
    big = torch.where(_randn(n, 2 * D, seed=seed + 1) > 0, 1e4, -1e4).to(bf16)
    for b, kb in enumerate(kv.tolist()):
        qkv[b * n + kb:(b + 1) * n, D:] = big[kb:]
    return qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]


@pytest.mark.parametrize("B,n,H,d", CASES + HEAD_DIM_CASES)
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
