"""References of the token front end (ivb_embed.cu) and of the VideoMAE pixel targets (ivb_loss.cu), exact where the
kernel is exact.

  - visible_indices: the index list of each clip in mask order, with the kernel's handling of a ragged mask (the flag
    names a clip whose count is wrong, and a short clip's unwritten tail points at token 1);
  - im2col: a bf16 gather of the Conv3d patches, zero past K;
  - gather_add: one fp32 add of the source row and the table row, rounded to the output type (nearest even);
  - scatter_add: fp32 adds onto the table gradient, clip after clip.  The rows of one clip name distinct table rows, so
    every table element receives its terms in clip order, one rounding each: the result is bit-exact;
  - pixel_targets: float64 of the labels, with a per-element error bound derived from the kernel's arithmetic (below).

Everything takes and returns CPU or CUDA tensors alike; the references run on the device of their inputs.
"""
from __future__ import annotations

import math

import torch

U24 = 2.0 ** -24        # fp32 unit roundoff
EVAL = 8.0              # fast-math divide, sqrt and reciprocal, in units of U24 (as tests/row_ref.py)


# ---------------------------------------------------------------- token front end
def visible_indices(mask, n_keep):
    """mask bool [B, N] (True = masked).  Returns (idx int32 [B, n_keep], flags): idx[b] lists the unmasked positions
    in order; a clip with fewer than n_keep of them has the rest of its row set to 1 (0 when N == 1), one with more
    keeps its first n_keep.  flags: the values the kernel's error flag may hold, {0} for an even mask, else
    {1 + b for every clip b whose count is not n_keep}."""
    B, N = mask.shape
    idx = torch.empty((B, n_keep), dtype=torch.int32)
    bad = set()
    safe = 1 if N > 1 else 0
    for b in range(B):
        pos = torch.nonzero(~mask[b].cpu(), as_tuple=False).flatten().to(torch.int32)
        if pos.numel() != n_keep:
            bad.add(1 + b)
        k = min(pos.numel(), n_keep)
        idx[b, :k] = pos[:k]
        idx[b, k:] = safe
    return idx.to(mask.device), (bad or {0})


def patches(video, tubelet, patch):
    """Every patch of video [B, C, T, H, W] as a row [B, T/t * H/p * W/p, C*t*p*p], rows ordered (frame, py, px) and each
    row ordered (c, dt, dy, dx) like the Conv3d weight."""
    B, C, T, H, W = video.shape
    t, h, w = T // tubelet, H // patch, W // patch
    x = video[:, :, :t * tubelet, :h * patch, :w * patch].reshape(B, C, t, tubelet, h, patch, w, patch)
    return x.permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(B, t * h * w, C * tubelet * patch * patch)


def im2col(video, idx, j0, rows_per_clip, tubelet, patch, kpad):
    """ivb_im2col_visible: row (b, j) is the patch of token idx[b, j0 + j] (token t >= 1 is patch t - 1), zero-padded to
    kpad.  Same dtype as video.  [B * rows_per_clip, kpad]."""
    p = patches(video, tubelet, patch)
    B, _, K = p.shape
    tok = idx[:, j0:j0 + rows_per_clip].long() - 1
    rows = torch.gather(p, 1, tok[:, :, None].expand(-1, -1, K).to(p.device))
    out = torch.zeros((B, rows_per_clip, kpad), dtype=video.dtype, device=video.device)
    out[:, :, :K] = rows
    return out.reshape(B * rows_per_clip, kpad)


def gather_add(src, table, idx, idx_off, B, rows, out_dtype):
    """ivb_gather_add: out[b, j] = src[b, j] + table[idx[b, j] + idx_off] (idx None: j).  src fp32 [B, rows, D] (expand
    a [1, rows, D] row for the cls broadcast) or None, table bf16 [N, D] or None.  The sum is one fp32 add (the float64
    sum of an fp32 and a bf16 value is exact), rounded to out_dtype; a missing src starts from +0 as the kernel does,
    a missing table adds nothing.  Returns out_dtype [B, rows, D]."""
    ref = src if src is not None else table
    D, dev = ref.shape[-1], ref.device
    v = src.double() if src is not None else torch.zeros((B, rows, D), dtype=torch.float64, device=dev)
    if table is not None:
        ti = idx.long().to(dev) if idx is not None else torch.arange(rows, device=dev)[None].expand(B, -1)
        v = v + table.double()[ti + idx_off]
    return v.float().to(out_dtype)


def scatter_add(g, idx, idx_off, table_grad):
    """ivb_scatter_add: table_grad[idx[b, j] + idx_off] += g[b, j] (idx None: j) in fp32, clip 0 first.  g fp32 or bf16
    [B, rows, D]; table_grad fp32 [N, D] is not modified.  Returns the new fp32 table gradient."""
    out = table_grad.clone()
    B, rows, _ = g.shape
    for b in range(B):
        ti = (idx[b].long() if idx is not None else torch.arange(rows, device=g.device)) + idx_off
        out.index_add_(0, ti.to(out.device), g[b].float().to(out.device))
    return out


# ---------------------------------------------------------------- pixel targets
def pixel_groups(video, midx, n_mask, tubelet, patch, mean3, std3):
    """The un-normalised pixels x * std + mean (float64, the fp32 constants taken as they are) of every masked patch and
    channel: [B * n_mask, C, t*p*p], pixels ordered (dt, dy, dx).  Also returns the bf16 values themselves."""
    B, C = video.shape[:2]
    p = patches(video, tubelet, patch)                                         # [B, L, C*npix]
    tok = midx.reshape(B, n_mask).long().to(p.device)
    x = torch.gather(p, 1, tok[:, :, None].expand(-1, -1, p.shape[-1])).double().reshape(B * n_mask, C, -1)
    u = x * std3.double().to(x.device)[None, :, None] + mean3.double().to(x.device)[None, :, None]
    return u, x


def _labels(u, rows, n, C):
    """'b n (p c)': [G, C, npix] -> [G, npix * C]."""
    return u.transpose(1, 2).reshape(rows, n * C)


def pixel_targets(video, midx, n_mask, tubelet, patch, normalize, mean3, std3):
    """Reference of ivb_pixel_targets with its arguments.  Returns (ref, scale), float64 [B * n_mask, t*p*p*C].

    normalize off: ref = x * std + mean and scale 0; the kernel rounds it once (fmaf).
    normalize on: per patch and channel, ref = c_i / (sqrt(sum c^2 / (n - 1)) + 1e-6), c_i = d_i - mean(d), with
    d_i = u_i - u_0 taken relative to the patch's first pixel as the kernel does, so a flat patch is exactly 0.
    `scale` bounds what the fp32 kernel may differ from ref, propagated through its steps (n = t*p*p pixels, each lane
    adding ceil(n / 32) terms in order, then five shuffle levels: m = ceil(n / 32) + 5 additions deep):
      u_i     one fmaf: error U24 |u_i|, the same bits for equal inputs, so d_i errs by U24 (|u_i| + |u_0|) only where
              x_i != x_0, plus U24 |d_i| for the subtraction
      mean    the sum of the d_i: their errors, plus m U24 sum |d_i|; the divide: EVAL U24 |mean|
      c_i     the errors of d_i and of the mean, plus U24 |c_i|
      var     sum of 2 |c_i| dc_i + dc_i^2, plus (m + 1) U24 sum c_i^2 for the squares and their sum; the divide EVAL U24
      sigma   |sqrt(a) - sqrt(b)| <= min(sqrt|a - b|, |a - b| / sqrt(b)), plus EVAL U24 sigma; + 1e-6 adds U24
      label   dc_i / den + |c_i| dden / den^2 (den at its lower bound), plus (EVAL + 1) U24 |label| for 1/den and the
              multiply."""
    C = video.shape[1]
    n = tubelet * patch * patch
    u, x = pixel_groups(video, midx, n_mask, tubelet, patch, mean3, std3)
    rows = u.shape[0]
    if not normalize:
        return _labels(u, rows, n, C), torch.zeros((rows, n * C), dtype=torch.float64, device=u.device)
    m = math.ceil(n / 32) + 5
    d = u - u[..., :1]
    mean = d.mean(-1, keepdim=True)
    c = d - mean
    var = (c * c).sum(-1, keepdim=True) / (n - 1)
    sig = var.sqrt()
    den = sig + 1e-6
    ref = c / den
    dd = (x != x[..., :1]).double() * U24 * (u.abs() + u[..., :1].abs()) + U24 * d.abs()
    dmean = (dd.sum(-1, keepdim=True) + m * U24 * (d.abs() + dd).sum(-1, keepdim=True)) / n + EVAL * U24 * mean.abs()
    dc = dd + dmean + U24 * (c.abs() + dd + dmean)
    q = ((c.abs() + dc) ** 2).sum(-1, keepdim=True)
    dvar = ((2 * c.abs() * dc + dc * dc).sum(-1, keepdim=True) + (m + 1) * U24 * q) / (n - 1) + EVAL * U24 * var
    dsig = torch.minimum(dvar.sqrt(), dvar / sig.clamp_min(1e-300)) + EVAL * U24 * sig
    dden = dsig + U24 * den
    den_lo = (den - dden).clamp_min(1e-6 * (1 - 4 * U24))
    scale = dc / den_lo + c.abs() * dden / (den * den_lo) + (EVAL + 1) * U24 * ref.abs()
    return _labels(ref, rows, n, C), _labels(scale, rows, n, C)
