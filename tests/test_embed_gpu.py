"""The token front end (ivb_embed.cu) and the VideoMAE pixel targets (ivb_loss.cu), element by element against
tests/embed_ref.py, on every call form the towers make.

visible_indices, im2col_visible, gather_add and scatter_add are exact: their outputs must equal the reference bit for
bit.  EmbedFn's GEMM outputs and the pixel labels are checked as the largest per-element error over its tolerance
(gemm_ref.elem_errors: half an ulp of the output format plus the reference's fp32 scale), so 1 is the edge of what a
correct kernel can produce.

Every output the kernels write is a view into a wider buffer filled with NaN (int32 outputs: -7): nothing outside the
view may change, and a second call must give the same bits.

Each limit in LIMITS is at most twice the worst value measured over this file on an H100 80GB HBM3 (SXM, 700 W power
limit); the measured value is beside it.  The file (132 tests) runs in under 20 s there.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import embed_ref as er
from gemm_ref import U24, elem_errors

pytestmark = pytest.mark.gpu

bf16, f32, i32 = torch.bfloat16, torch.float32, torch.int32
MEAN3 = (0.485, 0.456, 0.406)
STD3 = (0.229, 0.224, 0.225)

# limit, and beside it the worst value measured over this file (H100 80GB HBM3 SXM, 700 W power limit)
LIMITS = {
    "x0": 1.1,          # EmbedFn forward, fp32 residual stream                        measured 0.567
    "dw": 1.9,          # EmbedFn patch-embed weight gradient, bf16                    measured 0.99995
    "db": 1.9,          # EmbedFn patch-embed bias gradient, bf16                      measured 0.998
    "dcls": 1.9,        # EmbedFn cls-token gradient, bf16                             measured 0.99935
    "raw": 2.0,         # un-normalised pixel targets, fp32: one ulp                   measured 1 (half an ulp)
    "label": 0.17,      # normalised pixel targets, fp32                               measured 0.0846
}


# ---------------------------------------------------------------- buffers and checks
class Frame:
    """Sentinel-filled buffers around the outputs of one call.  arm() snapshots them; check() asserts that every
    element outside the views the call writes kept its bits."""

    def __init__(self):
        self.items = []

    def buf(self, shape, dtype):
        """A sentinel-filled buffer of `shape` (NaN, or -7 for integers); out() registers the view a call writes."""
        return torch.full(shape, math.nan if dtype.is_floating_point else -7, device="cuda", dtype=dtype)

    def out(self, buf, view):
        self.items.append((buf, view))
        return view

    def arm(self):
        torch.cuda.synchronize()
        self.snaps = [b.clone() for b, _ in self.items]

    def check(self, what):
        torch.cuda.synchronize()
        for (buf, v), snap in zip(self.items, self.snaps):
            keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
            keep.as_strided(v.shape, v.stride(), v.storage_offset() - buf.storage_offset()).fill_(False)
            ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[buf.element_size()]
            changed = keep & (buf.view(ib) != snap.view(ib))
            assert not changed.any(), f"{what}: {int(changed.sum())} elements outside the output changed, first at " \
                                      f"{tuple(int(i) for i in changed.nonzero()[0])} of a {tuple(buf.shape)} buffer"


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _exact(what, got, ref):
    got, ref = got.reshape(ref.shape), ref.to(got.device)
    diff = _bits(got) != _bits(ref.to(got.dtype))
    if diff.any():
        pos = tuple(int(i) for i in diff.nonzero()[0])
        raise AssertionError(f"{what}: {int(diff.sum())} of {diff.numel()} elements differ, first at {pos}: got "
                             f"{got[pos].item()!r}, ref {ref[pos].item()!r}")


def _twice(what, call, outs):
    """Runs `call` a second time and asserts that every output in `outs` kept its bits."""
    first = [o.clone() for o in outs]
    call()
    torch.cuda.synchronize()
    for a, b in zip(first, outs):
        _exact(f"{what}, second run", b, a)


def _check(what, fam, got, ref, scale):
    got = got.reshape(ref.shape)
    bad = ~torch.isfinite(got)
    assert not bad.any(), f"{what}: {int(bad.sum())} non-finite {fam} elements, first at {tuple(bad.nonzero()[0])}"
    errs = elem_errors(got, ref.to(got.device), scale.to(got.device))
    flat = int(errs.argmax())
    e = float(errs.reshape(-1)[flat])
    pos = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ref.shape))
    assert e <= LIMITS[fam], (f"{what}: {fam} error {e:.3g} x tol > {LIMITS[fam]} at {pos}: got {float(got[pos]):.9g}, "
                              f"ref {float(ref[pos]):.9g}, scale {float(scale[pos]):.3g}")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ---------------------------------------------------------------- visible_indices
def _keep_mask(B, N, keep, seed, cls=True):
    """bool [B, N] (True = masked), `keep` random positions unmasked per clip; position 0 kept too when cls."""
    g = torch.Generator().manual_seed(seed)
    m = torch.ones(B, N, dtype=torch.bool)
    lo = 1 if cls else 0
    for b in range(B):
        m[b, lo + torch.randperm(N - lo, generator=g)[:keep]] = False
    if cls:
        m[:, 0] = False
    return m


def _visible(ll, mask, n_keep):
    """ivb_visible_indices into a framed idx; returns (idx [B, n_keep], err) after checking the frame and a rerun."""
    B, N = mask.shape
    fr = Frame()
    buf = fr.buf((B * n_keep + 16,), i32)
    idx = fr.out(buf, buf[8:8 + B * n_keep])
    err = torch.zeros(1, device="cuda", dtype=i32)
    m = mask.cuda().contiguous().view(torch.uint8)
    fr.arm()

    def call():
        ll._call("visible_indices", m, B, N, n_keep, idx, err)
    call()
    fr.check("visible_indices")
    _twice("visible_indices", call, [idx])
    return idx.view(B, n_keep), err


@pytest.mark.parametrize("N", [5, 33, 1 + 196, 1 + 8 * 256, 1 + 1568])
@pytest.mark.parametrize("form", ["student", "iv1_visible", "iv1_masked", "one", "all"])
def test_visible_indices_bit_exact(cuda_lib, N, form):
    ll = cuda_lib
    B, P = 4, N - 1
    if form == "student":                                   # 20 % of the patches kept, behind the cls slot
        mask = _keep_mask(B, N, max(1, P // 5), N)
    elif form == "one":
        mask = _keep_mask(B, N, 1, N)
    elif form == "all":
        mask = torch.zeros(B, N, dtype=torch.bool)
    else:                                                   # IV1: 90 % of the patches masked, listed both ways
        from internvideo_b200 import videomae_v1
        pm = _keep_mask(B, P, max(1, P // 10), N, cls=False)
        keep_masked = form == "iv1_masked"
        idx, err, k = videomae_v1.kept_indices(pm.cuda(), keep_masked=keep_masked)
        mask = torch.cat([torch.zeros(B, 1, dtype=torch.bool), ~pm if keep_masked else pm], 1)
        ref, flags = er.visible_indices(mask, k + 1)
        assert flags == {0} and int(err.item()) == 0
        _exact(f"kept_indices N={N} {form}", idx, ref)
    n = int((~mask[0]).sum())
    ref, flags = er.visible_indices(mask, n)
    idx, err = _visible(ll, mask, n)
    assert flags == {0} and int(err.item()) == 0
    _exact(f"visible_indices N={N} {form}", idx, ref)


@pytest.mark.parametrize("N", [5, 33, 1 + 196, 1 + 1568])
def test_visible_indices_ragged(cuda_lib, N):
    """One clip keeps one token too many and another one too few: the flag names one of them, the short clip's tail
    points at token 1 and the long clip lists its first n_keep tokens."""
    ll = cuda_lib
    B = 3
    keep = max(2, (N - 1) // 5)
    mask = _keep_mask(B, N, keep, N)
    mask[0, torch.nonzero(mask[0])[0]] = False              # clip 0 keeps one extra
    mask[2, torch.nonzero(~mask[2])[-1]] = True             # clip 2 keeps one fewer
    n = 1 + keep
    ref, flags = er.visible_indices(mask, n)
    assert flags == {1, 3}
    idx, err = _visible(ll, mask, n)
    assert int(err.item()) in flags, int(err.item())
    assert int(idx[2, -1]) == 1
    _exact(f"visible_indices ragged N={N}", idx, ref)


# ---------------------------------------------------------------- im2col_visible
@pytest.mark.parametrize("tub,P", [(1, 14), (2, 16), (2, 14)])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("pad", [0, 8])
@pytest.mark.parametrize("j0", [0, 1])
def test_im2col_visible_bit_exact(cuda_lib, tub, P, C, pad, j0):
    """The patch rows of the tokens idx[:, j0:] names, zero-padded to Kpad (K rounded up to 8, and 8 more), from a
    non-square frame, with an index row pitch wider than the rows."""
    ll = cuda_lib
    B, T, H, W = 3, 2 * tub, 2 * P, 3 * P
    L = (T // tub) * (H // P) * (W // P)
    video = torch.randn(B, C, T, H, W, device="cuda", generator=_gen(P + C)).to(bf16)
    keep = 5
    mask = _keep_mask(B, 1 + L, keep, P + tub)
    vis, _ = er.visible_indices(mask, 1 + keep)
    ibuf = torch.full((B, 1 + keep + 5), -7, dtype=i32, device="cuda")
    ibuf[:, :1 + keep] = vis.cuda()
    idx = ibuf[:, 1 - j0:1 + keep]                        # j0 = 0: the patch columns alone; j0 = 1: behind the cls slot
    rows = keep
    K = C * tub * P * P
    kpad = (K + 7) // 8 * 8 + pad
    fr = Frame()
    buf = fr.buf((B * rows * kpad + 16,), bf16)
    cols = fr.out(buf, buf[8:8 + B * rows * kpad]).view(B * rows, kpad)
    fr.arm()

    def call():
        ll._call("im2col_visible", video, idx, idx.stride(0), j0, rows, B, C, T, H, W, tub, P, kpad, cols)
    call()
    fr.check("im2col_visible")
    _exact(f"im2col tub={tub} P={P} C={C} kpad={kpad} j0={j0}", cols, er.im2col(video, idx, j0, rows, tub, P, kpad))
    _twice("im2col_visible", call, [cols])


# ---------------------------------------------------------------- gather_add
GATHER_FORMS = [("src_table_idx", 0), ("src_table_idx", -1), ("src", 0), ("table", 0), ("cls", 0)]


@pytest.mark.parametrize("form,off", GATHER_FORMS)
@pytest.mark.parametrize("D", [8, 264, 1408, 3200])
@pytest.mark.parametrize("out_dtype", [f32, bf16])
def test_gather_add_bit_exact(cuda_lib, form, off, D, out_dtype):
    """Every form the towers call: position rows gathered onto a strided fp32 source (EmbedFn, GatherAddFn), the
    source alone rounded to bf16 (EmbedFn's demb), a table read without an index, and the cls row broadcast to every
    clip (source clip stride 0).  Source and output are strided views, as EmbedFn passes x0[:, 1:] and dx0[:, 1:]."""
    ll = cuda_lib
    g = _gen(D + off)
    B, rows, Ntab = 3, 1 if form == "cls" else 37, 50
    use_src, use_table = form != "table", form in ("src_table_idx", "table")
    sbuf = torch.randn(B, rows + 1, D, device="cuda", generator=g)
    src = (sbuf[:1, 1:].expand(B, -1, -1) if form == "cls" else sbuf[:, 1:]) if use_src else None
    src_bstride = 0 if form == "cls" else (rows + 1) * D
    table = torch.randn(Ntab, D, device="cuda", generator=g).to(bf16) if use_table else None
    idx = None
    if form == "src_table_idx":
        ibuf = torch.zeros(B, rows + 2, dtype=i32, device="cuda")
        for b in range(B):
            ibuf[b, 2:] = torch.randperm(Ntab - 1, device="cuda", generator=g)[:rows].sort().values + 1
        idx = ibuf[:, 2:]
    fr = Frame()
    obuf = fr.buf((B, rows + 3, D), out_dtype)
    out = fr.out(obuf, obuf[:, 1:1 + rows])
    fr.arm()

    def call():
        ll._call("gather_add", src, src_bstride, table, idx, 0 if idx is None else idx.stride(0), off, B, rows, D, out,
                 int(out_dtype == f32), out.stride(0))
    call()
    fr.check(f"gather_add {form}")
    _exact(f"gather_add {form} off={off} D={D} {out_dtype}", out,
           er.gather_add(src, table, idx, off, B, rows, out_dtype))
    _twice("gather_add", call, [out])


# ---------------------------------------------------------------- scatter_add
@pytest.mark.parametrize("form,off", [("null_idx", 0), ("idx", 0), ("idx", -1)])
@pytest.mark.parametrize("g_dtype", [f32, bf16])
@pytest.mark.parametrize("B", [3, 32])
@pytest.mark.parametrize("D", [264, 1408])
def test_scatter_add_bit_exact(cuda_lib, form, off, g_dtype, B, D):
    """The table gradient after adding B clips' rows onto a non-zero table, against clip-ordered fp32 adds; equal
    bits on a second run.  Values stay in the normal range: red.add.f32 flushes subnormals."""
    ll = cuda_lib
    gen = _gen(B * D + off)
    rows, Ntab = 37, 50
    gbuf = torch.randn(B, rows + 1, D, device="cuda", generator=gen).to(g_dtype)
    gv = gbuf[:, 1:]
    idx = None
    if form == "idx":
        ibuf = torch.zeros(B, rows + 1, dtype=i32, device="cuda")
        for b in range(B):
            ibuf[b, 1:] = torch.randperm(Ntab - 1, device="cuda", generator=gen)[:rows] + 1
        idx = ibuf[:, 1:]
    t0 = torch.randn(Ntab, D, device="cuda", generator=gen)
    fr = Frame()
    tbuf = fr.buf((Ntab + 2, D), f32)
    tg = fr.out(tbuf, tbuf[1:1 + Ntab])

    def call():
        tg.copy_(t0)
        ll._call("scatter_add", gv, int(g_dtype == f32), gv.stride(0), idx, 0 if idx is None else idx.stride(0), off,
                 B, rows, D, tg)
    fr.arm()
    call()
    fr.check(f"scatter_add {form}")
    _exact(f"scatter_add {form} off={off} {g_dtype} B={B} D={D}", tg, er.scatter_add(gv, idx, off, t0))
    _twice("scatter_add", call, [tg])


def test_gather_scatter_full_size(cuda_lib):
    """The student's position add and its gradient at the pretraining step's size (32 clips keeping 410 of 2048
    patches behind the cls slot, D = 1408), called as EmbedFn calls them: gather_add of the patch rows onto x0[:, 1:]
    and scatter_add of dx0 over every token into the position-table gradient.  Both bit-exact, nothing outside the
    outputs written (x0's cls rows included), and the same bits on a second run."""
    ll = cuda_lib
    B, L, keep, D = 32, 2048, 410, 1408
    n = 1 + keep
    idx, err = ll.visible_indices(_keep_mask(B, 1 + L, keep, 11).cuda(), n)
    assert int(err.item()) == 0
    emb = torch.randn(B, n - 1, D, device="cuda", generator=_gen(12))
    pos = (torch.randn(1 + L, D, device="cuda", generator=_gen(13)) * 0.1).to(bf16)
    dx0 = torch.randn(B, n, D, device="cuda", generator=_gen(14))
    fr = Frame()
    xbuf = fr.buf((B, n, D), f32)
    x0 = fr.out(xbuf, xbuf[:, 1:])
    tbuf = fr.buf((L + 3, D), f32)
    dpos = fr.out(tbuf, tbuf[1:L + 2])
    fr.arm()

    def call():
        ll.gather_add(emb, (n - 1) * D, pos, idx[:, 1:], n, 0, B, n - 1, D, x0, n * D)
        dpos.zero_()
        ll.scatter_add(dx0, n * D, idx, n, 0, B, n, D, dpos)
    call()
    fr.check("gather_add / scatter_add at full size")
    _exact("gather_add at full size", x0, er.gather_add(emb, pos, idx[:, 1:], 0, B, n - 1, f32))
    _exact("scatter_add at full size", dpos, er.scatter_add(dx0, idx, 0, torch.zeros(1 + L, D, device="cuda")))
    _twice("gather_add / scatter_add at full size", call, [x0, dpos])


# ---------------------------------------------------------------- EmbedFn and GatherAddFn through autograd
def _conv_tokens(x, w, b, tub, P):
    """float64 Conv3d of video x, and of |x| with |w|, as [B, tokens, D]."""
    y = F.conv3d(x.double(), w.double(), None if b is None else b.double(), stride=(tub, P, P))
    ya = F.conv3d(x.double().abs(), w.double().abs(), stride=(tub, P, P))
    return y.flatten(2).transpose(1, 2), ya.flatten(2).transpose(1, 2)


def _embed_case(D, tub, P, seed):
    B, C, T, H, W = 3, 3, 4 * tub, 4 * P, 4 * P
    L = (T // tub) * (H // P) * (W // P)
    keep = 13
    g = _gen(seed)
    x = torch.randn(B, C, T, H, W, device="cuda", generator=g).to(bf16)
    w = (torch.randn(D, C, tub, P, P, device="cuda", generator=g) * 0.02).to(bf16)
    b = (torch.randn(D, device="cuda", generator=g) * 0.1).to(bf16)
    mask = _keep_mask(B, 1 + L, keep, seed)
    return x, w, b, mask, L, 1 + keep


def _embed_fwd_ref(x, w, b, idx, table, tub, P):
    """float64 patch embed + position rows at the tokens idx[:, 1:] names: (ref, scale) [B, n - 1, D].  scale: the
    GEMM's fp32 accumulation (gemm_ref's sqrt(K/16) growth), its fp32 store, and the one fp32 add of the position row."""
    y, ya = _conv_tokens(x, w, b, tub, P)
    tok = (idx[:, 1:].long() - 1)[:, :, None].expand(-1, -1, y.shape[-1])
    emb, emba = torch.gather(y, 1, tok), torch.gather(ya, 1, tok)
    K = w[0].numel()
    kpad = (K + 7) // 8 * 8
    ref = emb + table.double()[idx[:, 1:].long()]
    scale = U24 * (math.sqrt(math.ceil(kpad / 16)) * emba + b.double().abs() + emb.abs())
    return ref, scale


def _wgrad_ref(x, wshape, demb, idx, L, tub, P):
    """float64 Conv3d weight gradient of the bf16 demb rows at the tokens idx[:, 1:] names, and its scale."""
    B, rows, D = demb.shape
    G = torch.zeros(B, L, D, dtype=torch.float64, device="cuda")
    G.scatter_(1, (idx[:, 1:].long() - 1)[:, :, None].expand(-1, -1, D), demb.double())
    _, C, T, H, W = x.shape
    g5 = G.transpose(1, 2).reshape(B, D, T // tub, H // P, W // P)
    dw = torch.nn.grad.conv3d_weight(x.double(), wshape, g5, stride=(tub, P, P))
    dwa = torch.nn.grad.conv3d_weight(x.double().abs(), wshape, g5.abs(), stride=(tub, P, P))
    return dw, U24 * math.sqrt(math.ceil(B * rows / 16)) * dwa


@pytest.mark.parametrize("D,tub,P", [(384, 1, 14), (1408, 1, 14), (384, 2, 16)])
def test_embed_fn_autograd(cuda_lib, D, tub, P):
    """EmbedFn forward and backward: the stream against float64 Conv3d + cls + position gather; dw and db against
    float64 of the bf16-rounded demb (the design: the weight gradients read bf16 demb); dpos bit-exact; dcls float64."""
    ll = cuda_lib
    from internvideo_b200 import ops
    x, w, b, mask, L, n = _embed_case(D, tub, P, D + tub)
    B = x.shape[0]
    cls = (torch.randn(1, 1, D, device="cuda", generator=_gen(1)) * 0.1).to(bf16)
    pos = (torch.randn(1, 1 + L, D, device="cuda", generator=_gen(2)) * 0.1).to(bf16)
    w_, b_, cls_, pos_ = (t.clone().requires_grad_(True) for t in (w, b, cls, pos))
    idx, err = ll.visible_indices(mask.cuda(), n)
    h = ops.EmbedFn.apply(x, idx, w_, b_, cls_, pos_, tub, P)
    assert int(err.item()) == 0
    h3 = h.detach().reshape(B, n, D)
    ref, scale = _embed_fwd_ref(x, w, b, idx, pos[0], tub, P)
    _check(f"EmbedFn D={D} patch rows", "x0", h3[:, 1:], ref, scale)
    c0 = (cls.reshape(D).float() + pos[0, 0].float()).double()
    _check(f"EmbedFn D={D} cls row", "x0", h3[:, 0], c0.expand(B, D), torch.zeros(B, D, dtype=torch.float64))
    dx0 = torch.randn(B * n, D, device="cuda", generator=_gen(3))
    h.backward(dx0)
    d3 = dx0.reshape(B, n, D)
    demb = d3[:, 1:].to(bf16)
    dw, dws = _wgrad_ref(x, w.shape, demb, idx, L, tub, P)
    _check(f"EmbedFn D={D} dw", "dw", w_.grad, dw, dws)
    M = B * (n - 1)
    db = demb.double().sum((0, 1))
    _check(f"EmbedFn D={D} db", "db", b_.grad, db, 2 * U24 * (math.sqrt(M) + 4) * demb.double().abs().sum((0, 1)))
    dcls = d3[:, 0].double().sum(0)
    _check(f"EmbedFn D={D} dcls", "dcls", cls_.grad.reshape(D), dcls, 2 * U24 * B * d3[:, 0].double().abs().sum(0))
    dpos = er.scatter_add(d3, idx, 0, torch.zeros(1 + L, D, device="cuda"))
    _exact(f"EmbedFn D={D} dpos", pos_.grad.reshape(1 + L, D), dpos.to(bf16))


def test_embed_tokens_without_cls(cuda_lib):
    """modules.embed_tokens with no cls token: the stream of the patch tokens alone, and the table gradient bit-exact
    (the cls slot's row of the padded table is dropped)."""
    ll = cuda_lib
    from internvideo_b200 import modules
    D, tub, P = 384, 1, 14
    x, w, b, mask, L, n = _embed_case(D, tub, P, 7)
    B = x.shape[0]
    pe = torch.nn.Module()
    pe.proj = torch.nn.Conv3d(3, D, (tub, P, P), stride=(tub, P, P)).cuda().to(bf16)
    with torch.no_grad():
        pe.proj.weight.copy_(w)
        pe.proj.bias.copy_(b)
    table = (torch.randn(1, L, D, device="cuda", generator=_gen(4)) * 0.1).to(bf16).requires_grad_(True)
    idx, _ = ll.visible_indices(mask.cuda(), n)
    h = modules.embed_tokens(pe, x, idx, None, table)
    assert h.shape == (B * (n - 1), D)
    full = torch.cat([torch.zeros(1, D, device="cuda", dtype=bf16), table.detach()[0]])
    ref, scale = _embed_fwd_ref(x, w, b, idx, full, tub, P)
    _check("embed_tokens without cls", "x0", h.detach(), ref, scale)
    dh = torch.randn(B, n - 1, D, device="cuda", generator=_gen(5))
    h.backward(dh.reshape(B * (n - 1), D))
    dfull = torch.cat([torch.zeros(B, 1, D, device="cuda"), dh], 1)
    dt = er.scatter_add(dfull, idx, 0, torch.zeros(1 + L, D, device="cuda")).to(bf16)[1:]
    _exact("embed_tokens without cls: table gradient", table.grad.reshape(L, D), dt)


@pytest.mark.parametrize("j0,off", [(0, 0), (1, -1)])
@pytest.mark.parametrize("D", [384, 1408])
def test_gather_add_fn_autograd(cuda_lib, j0, off, D):
    """The pretraining model's two decoder position adds (modules.py _decoder_inputs): the clip decoder's over every
    token, the MAE decoder's over the patch tokens with the table shifted by one.  Output, source gradient and table
    gradient bit-exact."""
    ll = cuda_lib
    from internvideo_b200 import ops
    B, L, keep = 3, 64, 13
    n = 1 + keep
    mask = _keep_mask(B, 1 + L, keep, D + j0)
    idx, _ = ll.visible_indices(mask.cuda(), n)
    taps = torch.randn(B * n, D, device="cuda", generator=_gen(6)).requires_grad_(True)
    table = (torch.randn(1, L + 1 + off, D, device="cuda", generator=_gen(7)) * 0.1).to(bf16).requires_grad_(True)
    out = ops.GatherAddFn.apply(taps, table, idx, B, n, j0, off)
    rows = n - j0
    _exact(f"GatherAddFn j0={j0} D={D}", out,
           er.gather_add(taps.detach().reshape(B, n, D)[:, j0:], table.detach()[0], idx[:, j0:], off, B, rows, bf16))
    dout = torch.randn(B * rows, D, device="cuda", generator=_gen(8)).to(bf16)
    out.backward(dout)
    d3 = dout.reshape(B, rows, D)
    dsrc = torch.zeros(B, n, D, device="cuda")
    dsrc[:, j0:] = d3.float()
    _exact(f"GatherAddFn j0={j0} D={D} dsrc", taps.grad, dsrc.reshape(B * n, D))
    dt = er.scatter_add(d3, idx[:, j0:], off, torch.zeros(L + 1 + off, D, device="cuda")).to(bf16)
    _exact(f"GatherAddFn j0={j0} D={D} dtable", table.grad.reshape(L + 1 + off, D), dt)


# ---------------------------------------------------------------- pixel targets
def _pixel_video(tub, P, seed):
    """A video of 2 clips whose first masked patches are flat (white, mid-grey and black frames, a random constant per
    channel) and one near-flat patch (a random constant with one pixel per channel one bf16 step off); the rest random.
    Returns (video, midx [B * n_mask] int32, n_mask, flat [B * n_mask] bool)."""
    B, C, T, H, W = 2, 3, 2 * tub, 2 * P, 3 * P
    gh, gw = H // P, W // P
    L = (T // tub) * gh * gw
    n_mask = 8
    g = _gen(seed)
    video = torch.randn(B, C, T, H, W, device="cuda", generator=g).to(bf16)
    midx = torch.stack([torch.randperm(L, device="cuda", generator=g)[:n_mask].sort().values for _ in range(B)])
    flat = torch.zeros(B, n_mask, dtype=torch.bool)

    def region(b, tok):
        f, py, px = tok // (gh * gw), (tok // gw) % gh, tok % gw
        return video[b, :, f * tub:(f + 1) * tub, py * P:(py + 1) * P, px * P:(px + 1) * P]

    consts = [[(raw - m) / s for m, s in zip(MEAN3, STD3)] for raw in (1.0, 0.5, 0.0)]
    consts.append(torch.randn(3, generator=torch.Generator().manual_seed(seed)).tolist())
    for k, cv in enumerate(consts):
        for c in range(C):
            region(0, int(midx[0, k]))[c].fill_(cv[c])
        flat[0, k] = True
    near = region(0, int(midx[0, 4]))
    for c in range(C):
        near[c].fill_(float(torch.randn(1, generator=torch.Generator().manual_seed(seed + c))))
        dt, rest = divmod((37 * c + 11) % (tub * P * P), P * P)
        near[c].view(torch.int16)[dt, rest // P, rest % P] += 1
    return video, midx.to(i32).flatten(), n_mask, flat.flatten()


@pytest.mark.parametrize("tub,P", [(2, 16), (1, 16), (2, 14)])
@pytest.mark.parametrize("normalize", [True, False])
def test_pixel_targets(cuda_lib, tub, P, normalize):
    """Pixel labels of masked patches: un-normalised within one fp32 ulp of float64 x * std + mean; normalised within
    embed_ref's derived bound, and exactly 0 on flat patches."""
    ll = cuda_lib
    video, midx, n_mask, flat = _pixel_video(tub, P, 10 * P + tub)
    B, C, T, H, W = video.shape
    mean3 = torch.tensor(MEAN3, device="cuda")
    std3 = torch.tensor(STD3, device="cuda")
    rows, width = B * n_mask, tub * P * P * C
    fr = Frame()
    buf = fr.buf((rows * width + 16,), f32)
    lab = fr.out(buf, buf[8:8 + rows * width]).view(rows, width)
    fr.arm()

    def call():
        ll._call("pixel_targets", video, midx, n_mask, B, C, T, H, W, tub, P, int(normalize), mean3, std3, lab)
    call()
    fr.check("pixel_targets")
    _twice("pixel_targets", call, [lab])
    ref, scale = er.pixel_targets(video, midx, n_mask, tub, P, normalize, mean3, std3)
    what = f"pixel_targets tub={tub} P={P} normalize={normalize}"
    if normalize:
        fl = lab[flat.cuda()]
        assert (fl == 0).all(), f"{what}: flat patches give non-zero labels, up to {float(fl.abs().max()):.3g}"
    _check(what, "label" if normalize else "raw", lab, ref, scale)
