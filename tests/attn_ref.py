"""float64 reference of token-axis multi-head attention and the per-tile error metric the attention tests use.

Layout is the one the kernels take: q, k, v, out and dout are 2-D [B*n, H*d] views (any row pitch) whose rows are
the tokens of B clips of n tokens and whose columns are H heads of d.  lse2 is [B, H, n], the log2-domain logsumexp
of the scaled scores.  Everything runs in float64 on the inputs' device, one clip at a time, so n = 2049 fits.

Masks are the kernels' masks: causal drops key > query; kv_len [B] keeps keys [0, kv_len[b]) of clip b for every
query.  A masked score is -inf, so its P and dS are exactly 0.
"""
from __future__ import annotations

import math

import torch

LOG2E = math.log2(math.e)


def _heads(x, b, n, H, d):
    """Clip b of a [B*n, H*d] view as float64 [H, n, d]."""
    return x[b * n:(b + 1) * n].double().reshape(n, H, d).transpose(0, 1)


def _masked(n, causal, keys, device):
    """[n, n] bool, True where the key (column) is masked for the query (row); None when nothing is."""
    if not causal and keys >= n:
        return None
    i = torch.arange(n, device=device)
    return (i[None, :] > i[:, None]) & bool(causal) | (i[None, :] >= keys)


def _probs(qb, kb, scale, mask):
    s = (qb @ kb.transpose(-2, -1)) * scale                       # [H, n, n]
    if mask is not None:
        s = s.masked_fill(mask, float("-inf"))
    lse = torch.logsumexp(s, -1, keepdim=True)
    return torch.exp(s - lse), lse.squeeze(-1)


def _key_lengths(kv_len, B, n):
    return [n] * B if kv_len is None else [int(x) for x in (kv_len.tolist() if torch.is_tensor(kv_len) else kv_len)]


def attn_ref_fwd(q, k, v, B, n, H, d, scale, causal=False, kv_len=None):
    """O = softmax(scale * q k^T + mask) v per (clip, head).  kv_len: None or B ints in [1, n] (a list or an int
    tensor).  Returns (O float64 [B*n, H*d], lse2 float64 [B, H, n])."""
    out = torch.empty((B * n, H * d), dtype=torch.float64, device=q.device)
    lse2 = torch.empty((B, H, n), dtype=torch.float64, device=q.device)
    for b, keys in enumerate(_key_lengths(kv_len, B, n)):
        p, lse = _probs(_heads(q, b, n, H, d), _heads(k, b, n, H, d), scale, _masked(n, causal, keys, q.device))
        out[b * n:(b + 1) * n] = (p @ _heads(v, b, n, H, d)).transpose(0, 1).reshape(n, H * d)
        lse2[b] = lse * LOG2E
    return out, lse2


def attn_ref_bwd(q, k, v, dout, B, n, H, d, scale, causal=False):
    """Analytic gradients of attn_ref_fwd's O for the incoming gradient dout:
    dV = P^T dO,  dP = dO V^T,  dS = P * (dP - rowsum(dO * O)),  dQ = scale * dS K,  dK = scale * dS^T Q.
    Returns float64 (dq, dk, dv), each [B*n, H*d]."""
    grads = [torch.empty((B * n, H * d), dtype=torch.float64, device=q.device) for _ in range(3)]
    mask = _masked(n, causal, n, q.device)
    for b in range(B):
        qb, kb, vb, gb = (_heads(t, b, n, H, d) for t in (q, k, v, dout))
        p, _ = _probs(qb, kb, scale, mask)
        dp = gb @ vb.transpose(-2, -1)
        ds = p * (dp - (p * dp).sum(-1, keepdim=True))            # rowsum(dO * O) = rowsum(P * dP)
        for g, t in zip(grads, (scale * ds @ kb, scale * ds.transpose(-2, -1) @ qb, p.transpose(-2, -1) @ gb)):
            g[b * n:(b + 1) * n] = t.transpose(0, 1).reshape(n, H * d)
    return tuple(grads)


def tile_errors(got, ref, B, n, H, d, rows=64):
    """Relative error of every (clip, head, `rows`-row band) of a [B*n, H*d] result: the rms of the band's error
    divided by the rms of that (clip, head)'s whole reference.  Normalising by the whole head, not the band, keeps a
    band whose reference is near zero from reading as a huge relative error.  Returns float64 [B, H, ceil(n/rows)]."""
    err = (got.detach().double() - ref.double()).reshape(B, n, H, d)
    nb = (n + rows - 1) // rows
    pad = nb * rows - n
    e2 = torch.nn.functional.pad(err.square(), (0, 0, 0, 0, 0, pad)).reshape(B, nb, rows, H, d).sum((2, 4))
    cnt = torch.full((nb,), float(rows), dtype=torch.float64, device=err.device)
    cnt[-1] = rows - pad
    band_rms = (e2 / (cnt[None, :, None] * d)).sqrt().transpose(1, 2)              # [B, H, nb]
    ref_rms = ref.double().reshape(B, n, H, d).square().mean((1, 3)).sqrt()        # [B, H]
    return band_rms / (ref_rms[..., None] + 1e-30)


def worst(errs):
    """(largest value, its index as a tuple) of an error tensor, e.g. (err, (b, h, band)) of tile_errors."""
    flat = int(errs.argmax())
    idx = []
    for s in reversed(errs.shape):
        idx.append(flat % s)
        flat //= s
    return float(errs.max()), tuple(reversed(idx))
