"""tests/embed_ref.py against the oracle's restatement (oracle/restate.py) in float64 on small shapes (CPU), and the
pixel-target error bound against an fp32 emulation of the kernel's summation order: the pivoted sums stay inside it,
raw sums of a near-flat patch do not, and a flat patch's reference and bound are exactly 0."""
import numpy as np
import pytest
import torch

import embed_ref as er
from gemm_ref import elem_errors
from oracle import restate

dt = torch.float64
MEAN3 = torch.tensor(restate.IMAGENET_MEAN, dtype=torch.float32)
STD3 = torch.tensor(restate.IMAGENET_STD, dtype=torch.float32)


def _mask(B, N, keep, seed):
    g = torch.Generator().manual_seed(seed)
    m = torch.ones(B, N, dtype=torch.bool)
    for b in range(B):
        m[b, torch.randperm(N, generator=g)[:keep]] = False
    return m


@pytest.mark.parametrize("B,N,keep", [(3, 5, 2), (4, 33, 7), (2, 197, 40), (2, 197, 197), (2, 197, 1)])
def test_visible_indices_matches_restate(B, N, keep):
    m = _mask(B, N, keep, N)
    idx, flags = er.visible_indices(m, keep)
    assert flags == {0}
    assert torch.equal(idx.long(), restate.visible_indices(m))


def test_visible_indices_ragged():
    m = _mask(3, 33, 7, 1)
    m[0, torch.nonzero(m[0])[0]] = False             # clip 0 keeps 8
    m[2, torch.nonzero(~m[2])[-1]] = True            # clip 2 keeps 6
    idx, flags = er.visible_indices(m, 7)
    assert flags == {1, 3}
    assert torch.equal(idx[0].long(), torch.nonzero(~m[0]).flatten()[:7])
    assert torch.equal(idx[1].long(), torch.nonzero(~m[1]).flatten())
    assert torch.equal(idx[2, :6].long(), torch.nonzero(~m[2]).flatten()) and int(idx[2, 6]) == 1
    one = torch.zeros(2, 1, dtype=torch.bool)
    one[1, 0] = True
    idx, flags = er.visible_indices(one, 1)
    assert flags == {2} and idx.tolist() == [[0], [0]]


@pytest.mark.parametrize("tub,P,C,T,H,W", [(1, 14, 3, 2, 28, 42), (2, 16, 1, 4, 32, 32), (2, 14, 3, 2, 28, 28)])
def test_im2col_is_the_conv3d_patch(tub, P, C, T, H, W):
    """im2col rows times the flattened Conv3d weight give restate.patch_embed at the tokens idx names, and the padding
    is zero."""
    B, D = 2, 5
    g = torch.Generator().manual_seed(P)
    x = torch.randn(B, C, T, H, W, generator=g, dtype=dt)
    w = torch.randn(D, C, tub, P, P, generator=g, dtype=dt)
    L = (T // tub) * (H // P) * (W // P)
    m = torch.cat([torch.zeros(B, 1, dtype=torch.bool), _mask(B, L, 3, L)], 1)
    idx, _ = er.visible_indices(m, 4)
    K = C * tub * P * P
    cols = er.im2col(x, idx, 1, 3, tub, P, K + 8).reshape(B, 3, K + 8)
    assert torch.equal(cols[..., K:], torch.zeros(B, 3, 8, dtype=dt))
    full = restate.patch_embed(x, w, torch.zeros(D, dtype=dt), tub, P).reshape(B, L, D)
    want = torch.gather(full, 1, (idx[:, 1:].long() - 1)[:, :, None].expand(-1, -1, D))
    assert torch.allclose(cols[..., :K] @ w.reshape(D, K).t(), want, rtol=1e-12, atol=1e-12)
    conv = torch.nn.functional.conv3d(x, w, stride=(tub, P, P)).flatten(2).transpose(1, 2)
    assert torch.allclose(full, conv, rtol=1e-12, atol=1e-12)


def test_gather_add_and_scatter_add():
    g = torch.Generator().manual_seed(0)
    B, rows, D, N = 3, 5, 16, 9
    src = torch.randn(B, rows, D, generator=g)
    table = torch.randn(N, D, generator=g).to(torch.bfloat16)
    idx = torch.stack([torch.randperm(N, generator=g)[:rows] for _ in range(B)]).to(torch.int32)
    for off in (0, -1):
        ii = idx.clamp_min(-off)
        got = er.gather_add(src, table, ii, off, B, rows, torch.float32)
        assert torch.equal(got, src + table.float()[ii.long() + off])
        assert torch.equal(er.gather_add(src, table, ii, off, B, rows, torch.bfloat16), got.to(torch.bfloat16))
    assert torch.equal(er.gather_add(None, table, None, 0, B, rows, torch.float32),
                       table.float()[:rows].expand(B, -1, -1))
    neg = -torch.zeros(B, rows, D)
    assert torch.equal(er.gather_add(neg, None, None, 0, B, rows, torch.float32).view(torch.int32),
                       neg.view(torch.int32))                                       # src alone keeps -0
    t0 = torch.randn(N, D, generator=g)
    got = er.scatter_add(src, idx, 0, t0)
    want = t0.double().index_add(0, idx.long().flatten(), src.double().reshape(-1, D))
    assert torch.allclose(got.double(), want, rtol=1e-6, atol=1e-6)
    assert torch.equal(er.scatter_add(src, None, 2, t0)[2:2 + rows], ((t0[2:2 + rows] + src[0]) + src[1]) + src[2])


def _video(B, C, T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, T, H, W, generator=g).to(torch.bfloat16)


@pytest.mark.parametrize("tub,P", [(2, 16), (1, 16), (2, 14)])
@pytest.mark.parametrize("normalize", [True, False])
def test_pixel_targets_match_restate(tub, P, normalize):
    B, T, HW = 2, 2 * tub, 2 * P
    x = _video(B, 3, T, HW, HW, P + tub)
    L = 2 * 4
    m = _mask(B, L, 3, tub)                      # True = masked
    midx = torch.stack([torch.nonzero(m[b]).flatten() for b in range(B)]).to(torch.int32)
    m64, s64 = torch.tensor(restate.IMAGENET_MEAN, dtype=dt), torch.tensor(restate.IMAGENET_STD, dtype=dt)
    ref, scale = er.pixel_targets(x, midx.flatten(), 5, tub, P, normalize, m64, s64)
    want = restate.pixel_targets(x.double(), m, P, tub, normalize).reshape(B * 5, -1)
    assert torch.allclose(ref, want, rtol=1e-9, atol=1e-9), float((ref - want).abs().max())
    assert torch.isfinite(scale).all() and (scale >= 0).all()
    assert (scale > 0).all() == normalize


# ---------------------------------------------------------------- the kernel's arithmetic, emulated in fp32
def _warp_sum(terms):
    """terms float32 [G, n]: lane l adds terms l, l + 32, ... in order, then the xor butterfly (ivb_ptx.cuh warp_sum).
    Returns [G] (every lane holds the same value)."""
    G, n = terms.shape
    lanes = np.zeros((G, 32), dtype=np.float32)
    for i in range(0, n, 32):
        k = min(32, n - i)
        lanes[:, :k] = lanes[:, :k] + terms[:, i:i + k]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    return lanes[:, 0]


def _kernel_fp32(u, pivoted):
    """pixel_target_kernel's normalisation of fp32 pixels u [G, n] (pivoted: the sums relative to pixel 0)."""
    f = np.float32
    n = u.shape[1]
    base = u[:, :1] if pivoted else np.zeros_like(u[:, :1])
    d = (u - base).astype(f)
    mean = (_warp_sum(d) / f(n)).astype(f)[:, None]
    c = (d - mean).astype(f)
    var = (_warp_sum((c * c).astype(f)) / f(n - 1)).astype(f)[:, None]
    inv = (f(1) / (np.sqrt(var).astype(f) + f(1e-6))).astype(f)
    return (c * inv).astype(f)


def _groups(tub, P, kind, seed):
    """[G, n] bf16 pixel groups (one patch-channel each) and the fp32 pixels the kernel forms from them (channel 0)."""
    n = tub * P * P
    g = torch.Generator().manual_seed(seed)
    if kind == "flat":
        x = torch.randn(64, 1, generator=g).expand(64, n).contiguous()
    elif kind == "one_off":
        x = torch.randn(64, 1, generator=g).to(torch.bfloat16).expand(64, n).contiguous()
        x.view(torch.int16)[torch.arange(64), torch.randint(0, n, (64,), generator=g)] += 1      # one bf16 step
    else:
        x = torch.randn(64, n, generator=g)
    x = x.to(torch.bfloat16)
    u32 = (x.double() * float(STD3[0]) + float(MEAN3[0])).float().numpy()       # one fmaf rounding
    return x, u32


def _ref_groups(x, tub, P):
    """embed_ref.pixel_targets of the groups x [G, n] (channel 0, one frame layout per group)."""
    G, n = x.shape
    video = x.reshape(G, 1, tub, P, P)
    midx = torch.zeros(G, dtype=torch.int32)
    ref, scale = er.pixel_targets(video, midx, 1, tub, P, True, MEAN3[:1], STD3[:1])
    return ref.numpy(), scale.numpy()


@pytest.mark.parametrize("tub,P", [(2, 16), (1, 16), (2, 14)])
@pytest.mark.parametrize("kind", ["random", "one_off", "flat"])
def test_pixel_bound_holds_for_the_kernel_order(tub, P, kind):
    x, u32 = _groups(tub, P, kind, 3 * P + tub)
    ref, scale = _ref_groups(x, tub, P)
    got = _kernel_fp32(u32, pivoted=True)
    err = elem_errors(torch.from_numpy(got), torch.from_numpy(ref), torch.from_numpy(scale))
    assert float(err.max()) <= 1.0, float(err.max())
    if kind == "flat":
        assert (ref == 0).all() and (scale == 0).all() and (got == 0).all()


@pytest.mark.parametrize("tub,P", [(2, 16), (1, 16)])
def test_pixel_bound_rejects_raw_sums(tub, P):
    """Summing the raw pixels (no pivot) leaves a rounding residue in the mean: flat patches get labels far from 0 and
    near-flat ones leave the bound."""
    for kind in ("flat", "one_off"):
        x, u32 = _groups(tub, P, kind, 3 * P + tub)
        ref, scale = _ref_groups(x, tub, P)
        got = _kernel_fp32(u32, pivoted=False)
        err = elem_errors(torch.from_numpy(got), torch.from_numpy(ref), torch.from_numpy(scale))
        assert float(err.max()) > 10.0, (kind, float(err.max()))
