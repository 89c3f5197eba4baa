"""Every norm, LayerScale, column-sum, decoder-head, contrastive, MSE and AdamW kernel of ivb_norm.cu / ivb_loss.cu,
element by element against the float64 reference of tests/row_ref.py, at the shapes that select each kernel the
library can choose (grid sizes assume a 132-SM H100).

Each check is the largest per-element error divided by its tolerance (gemm_ref.elem_errors: half an ulp of the output
format plus row_ref's fp32 scale), so one element a bf16 ulp off, or a few wrong rows among thousands, fails it.  A
failure names the entry point, the case, and the worst row and column with its value, reference and limit.

Every output lives inside a wider NaN-filled buffer with a padded pitch, and every input inside one whose padding is
NaN: each output element must be finite (written, and computed from no padding), and every byte outside the outputs'
views -- padding, the untouched q/k/v slots, neighbouring rows -- must keep its bits.  Parameter-gradient and loss
outputs start from nonzero values, so the documented `+=` is checked too.

Each limit in LIMITS is at most twice the worst value measured over this file on an H100 80GB HBM3 (SXM, 700 W power
limit); the measured value is beside it.  The file (692 tests) runs in 20 to 30 s there.
"""
import math
import zlib

import pytest
import torch

import row_ref as rr
from gemm_ref import elem_errors

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32

# limit, and beside it the worst value measured over this file (H100 80GB HBM3 SXM, 700 W power limit)
LIMITS = {
    "y": 1.9,           # bf16 norm outputs (norm_fwd, pair, ln_l2_fwd, l2norm_rows_fwd)   measured 0.99969
    "rstd": 0.36,       # fp32 saved rstd, 1/||y||, 1/||x||                                measured 0.180
    "mean": 0.67,       # fp32 saved mean                                                  measured 0.336
    "dx32": 0.98,       # fp32 input gradients                                             measured 0.494
    "dx16": 1.9,        # bf16 input gradients, dyb, LayerScale dy, dcos, dpred            measured 0.999995
    "pgrad": 0.66,      # fp32 parameter gradients (fixed-order column sums)               measured 0.332
    "loss": 0.5,        # fp32 losses (atomic sums: their order varies), lse, dtemp        measured 0.260 (eight runs)
    "adamw": 1.5,       # fp32 master, exp_avg, exp_avg_sq                                 measured 0.751
    "fp8": 1.9,         # E4M3 row of norm_fwd_fp8, in half E4M3 ulps                      measured 0.99992
}


# ---------------------------------------------------------------- buffers and checks
class Frame:
    """NaN-filled buffers around the operands of one call.  arm() snapshots them; check() asserts that every element
    outside the views the call writes kept its bits."""

    def __init__(self):
        self.items = []

    def mat(self, rows, cols, dtype, fill=None, pad=8, writes=True):
        """A [rows, cols] view at row 1 of a [rows + 2, cols + pad] NaN buffer, filled with `fill` if given."""
        buf = torch.full((rows + 2, cols + pad), math.nan, device="cuda", dtype=dtype)
        v = buf[1:rows + 1, :cols]
        if fill is not None:
            v.copy_(fill)
        self.items.append((buf, [v] if writes else []))
        return v

    def vec(self, n, fill=None, dtype=f32, writes=True):
        """An [n] view at element 8 of an [n + 16] NaN buffer."""
        buf = torch.full((n + 16,), math.nan, device="cuda", dtype=dtype)
        v = buf[8:8 + n]
        if fill is not None:
            v.copy_(fill)
        self.items.append((buf, [v] if writes else []))
        return v

    def watch(self, buf, *views):
        self.items.append((buf, list(views)))

    def arm(self):
        self.snaps = [b.clone() for b, _ in self.items]

    def check(self, what):
        torch.cuda.synchronize()
        for (buf, views), snap in zip(self.items, self.snaps):
            keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
            for v in views:
                keep.as_strided(v.shape, v.stride(), v.storage_offset() - buf.storage_offset()).fill_(False)
            ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[buf.element_size()]
            changed = keep & (buf.view(ib) != snap.view(ib))
            assert not changed.any(), f"{what}: {int(changed.sum())} elements outside the outputs changed, first at " \
                                      f"{tuple(int(i) for i in changed.nonzero()[0])} of a {tuple(buf.shape)} buffer"


def _check(what, fam, got, ref_scale):
    ref, scale = ref_scale
    got = got.reshape(ref.shape)
    bad = ~torch.isfinite(got)
    if bad.any():
        pos = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} non-finite elements of {fam}, first at {pos}")
    errs = elem_errors(got, ref, scale)
    flat = int(errs.argmax())
    e = float(errs.reshape(-1)[flat])
    pos = divmod(flat, ref.shape[1]) if ref.dim() == 2 else (flat,)
    assert e <= LIMITS[fam], (f"{what}: {fam} error {e:.3g} x tol > {LIMITS[fam]} at row/col {pos}: got "
                              f"{float(got[pos]):.8g}, ref {float(ref[pos]):.8g}, scale {float(scale[pos]):.3g}")


def _outs(what, fams, got, ref):
    """Checks got[k] against ref[k] for every output k the reference has."""
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    for k in ref:
        _check(f"{what} {k}", fams.get(k, k), got[k], ref[k])


def _seed(*key):
    torch.manual_seed(zlib.crc32(repr(key).encode()))


def _weights(D, ln=False):
    w = (torch.randn(D, device="cuda") * 0.2 + 1).to(bf16)
    b = (torch.randn(D, device="cuda") * 0.1).to(bf16) if ln else None
    return w, b


def _rowscale(M):
    rs = (torch.rand(M, device="cuda") < 0.7).float() / 0.7
    rs[0] = 0.0 if M > 2 else rs[0]
    return rs


# ---------------------------------------------------------------- norm_fwd
RMS_REG_D = [8, 264, 384, 512, 520, 1024, 1032, 1408, 1536]
NORM_M = [1, 7, 417, 8449]
FWD_CASES = ([("rms", D, M) for D in RMS_REG_D for M in NORM_M] + [("rms", D, M) for D in (1544, 3200) for M in NORM_M]
             + [(k, D, M) for k in ("ln", "ln_nobias") for D in (8, 520, 1408, 3208) for M in (1, 417, 8449)])


def _norm_fwd(fr, x, w, b, eps, ln, want_stats=True, y=None):
    M, D = x.shape
    y = fr.mat(M, D, bf16) if y is None else y
    mean = fr.vec(M) if (ln and want_stats) else None
    rstd = fr.vec(M) if want_stats else None
    fr.arm()
    from internvideo_b200 import lowlevel as ll
    ll._call("norm_fwd", x, int(x.dtype == f32), x.stride(0), w, b, float(eps), int(ln), M, D, y, y.stride(0), mean, rstd)
    return y, mean, rstd


@pytest.mark.parametrize("kind,D,M", FWD_CASES)
@pytest.mark.parametrize("xdt", [f32, bf16])
def test_norm_fwd(cuda_lib, kind, D, M, xdt):
    _seed("fwd", kind, D, M, str(xdt))
    ln = kind != "rms"
    fr = Frame()
    x = fr.mat(M, D, xdt, torch.randn(M, D, device="cuda") * 2 + 0.3, writes=False)
    w, b = _weights(D, kind == "ln")
    eps = 1e-5 if ln else 1e-6
    y, mean, rstd = _norm_fwd(fr, x, w, b, eps, ln)
    what = f"norm_fwd [{kind} D={D} M={M} x={xdt}]"
    fr.check(what)
    got = {"y": y, "rstd": rstd} | ({"mean": mean} if ln else {})
    _outs(what, {}, got, rr.norm_fwd(x, w, b, eps, ln))


@pytest.mark.parametrize("kind,D", [("rms", 1408), ("ln", 3200)])
def test_norm_fwd_without_stats(cuda_lib, kind, D):
    _seed("fwd-nostats", kind, D)
    ln = kind == "ln"
    fr = Frame()
    x = fr.mat(417, D, f32, torch.randn(417, D, device="cuda"), writes=False)
    w, b = _weights(D, ln)
    y, _, _ = _norm_fwd(fr, x, w, b, 1e-6, ln, want_stats=False)
    fr.check(f"norm_fwd [{kind} D={D} no stats]")
    _check(f"norm_fwd [{kind} D={D} no stats]", "y", y, rr.norm_fwd(x, w, b, 1e-6, ln)["y"])


@pytest.mark.parametrize("D", [1544, 3200])
@pytest.mark.parametrize("M", [7, 8449])
def test_norm_fwd_strided_qk(cuda_lib, D, M):
    """The q- and k-norms above D = 1536 (two norm_fwd calls): views of a [M, 3D] qkv buffer into a [M, 2D] output."""
    _seed("fwd-qk", D, M)
    fr = Frame()
    qkv = fr.mat(M, 3 * D, bf16, torch.randn(M, 3 * D, device="cuda"), writes=False)
    qkn_buf = torch.full((M + 2, 2 * D + 8), math.nan, device="cuda", dtype=bf16)
    qkn = qkn_buf[1:M + 1, :2 * D]
    wq, _ = _weights(D)
    wk, _ = _weights(D)
    for part, w in ((0, wq), (1, wk)):
        f = Frame()
        f.items = list(fr.items)
        f.watch(qkn_buf, qkn[:, part * D:(part + 1) * D])
        x = qkv[:, part * D:(part + 1) * D]
        y, _, rstd = _norm_fwd(f, x, w, None, 1e-6, False, y=qkn[:, part * D:(part + 1) * D])
        what = f"norm_fwd [q/k slot {part} D={D} M={M}]"
        f.check(what)
        _outs(what, {}, {"y": y, "rstd": rstd}, rr.norm_fwd(x, w, None, 1e-6, False))


# ---------------------------------------------------------------- norm_bwd
BWD_D = [("rms", 264), ("rms", 520), ("rms", 1032), ("rms", 1536), ("rms", 1544), ("ln", 1408), ("ln", 3200),
         ("ln", 3208), ("ln", 6408), ("rms", 6408)]


def _stats(x, w, b, ln):
    from internvideo_b200 import lowlevel as ll
    _, mean, rstd = ll.norm_fwd(x, w, b, eps=1e-5 if ln else 1e-6, layernorm=ln)
    return mean, rstd


@pytest.mark.parametrize("kind,D", BWD_D)
@pytest.mark.parametrize("xdt", [f32, bf16])
@pytest.mark.parametrize("dxdt", [f32, bf16])
@pytest.mark.parametrize("with_in", [True, False])
@pytest.mark.parametrize("with_grads", [True, False])
def test_norm_bwd(cuda_lib, kind, D, xdt, dxdt, with_in, with_grads):
    _check_norm_bwd(kind, D, 1031, xdt, dxdt, with_in, with_grads)


@pytest.mark.parametrize("xdt", [f32, bf16])
@pytest.mark.parametrize("with_in", [True, False])
def test_norm_bwd_one_warp_per_cta(cuda_lib, xdt, with_in):
    """LayerNorm at D = 14 088 with weight gradients: a warp's two gradient rows take 110 KB of shared memory, so each
    CTA runs one warp.  At M = 400 the partials of its 200 CTAs fit the gradient scratch."""
    _check_norm_bwd("ln", 14088, 400, xdt, bf16, with_in, True)


def _check_norm_bwd(kind, D, M, xdt, dxdt, with_in, with_grads):
    from internvideo_b200 import lowlevel as ll
    _seed("bwd", kind, D, str(xdt), str(dxdt), with_in, with_grads)
    ln = kind == "ln"
    fr = Frame()
    x = fr.mat(M, D, xdt, torch.randn(M, D, device="cuda") * 2 + 0.3, writes=False)
    w, b = _weights(D, ln)
    mean, rstd = _stats(x, w, b, ln)
    dy = fr.mat(M, D, bf16, torch.randn(M, D, device="cuda"), writes=False)
    dx_in = fr.mat(M, D, f32, torch.randn(M, D, device="cuda"), pad=16, writes=False) if with_in else None
    dx = fr.mat(M, D, dxdt)
    dw = fr.vec(D, torch.randn(D, device="cuda")) if with_grads else None
    db = fr.vec(D, torch.randn(D, device="cuda")) if (with_grads and ln) else None
    ref = rr.norm_bwd(dy, x, w, mean, rstd, ln, dx_in, dw, db)
    fr.arm()
    ll.norm_bwd(dy, x, w, mean, rstd, layernorm=ln, dx_in=dx_in, dx_out=dx, dweight=dw, dbias=db)
    what = f"norm_bwd [{kind} D={D} x={xdt} dx={dxdt} dx_in={with_in} grads={with_grads}]"
    fr.check(what)
    got = {"dx": dx} | ({"dweight": dw} if with_grads else {}) | ({"dbias": db} if (with_grads and ln) else {})
    _outs(what, {"dx": "dx32" if dxdt == f32 else "dx16", "dweight": "pgrad", "dbias": "pgrad"}, got, ref)


@pytest.mark.parametrize("D", [1408, 3200])
def test_norm_bwd_in_place_qk_slots(cuda_lib, D):
    """The q/k-norm backward above D = 1536, as the block runs it: bf16 dx written over dy in the q and k slots of the
    [M, 3D] gradient buffer; the v slot and the padding keep their bits."""
    from internvideo_b200 import lowlevel as ll
    _seed("bwd-inplace", D)
    M = 2 * 417 + 1
    fr = Frame()
    qkv = fr.mat(M, 3 * D, bf16, torch.randn(M, 3 * D, device="cuda"), writes=False)
    dqkv_buf = torch.full((M + 2, 3 * D + 8), math.nan, device="cuda", dtype=bf16)
    dqkv = dqkv_buf[1:M + 1, :3 * D]
    dqkv.copy_(torch.randn(M, 3 * D, device="cuda"))
    fr.watch(dqkv_buf, dqkv[:, :2 * D])
    refs, gots = [], []
    for part in (0, 1):
        x = qkv[:, part * D:(part + 1) * D]
        w, _ = _weights(D)
        _, rstd = _stats(x, w, None, False)
        dw = fr.vec(D, torch.randn(D, device="cuda"))
        g = dqkv[:, part * D:(part + 1) * D]
        refs.append(rr.norm_bwd(g, x, w, None, rstd, False, None, dw))
        gots.append((g, dw, x, w, rstd))
    fr.arm()
    for g, dw, x, w, rstd in gots:
        ll.norm_bwd(g, x, w, None, rstd, dx_out=g, dweight=dw)
    what = f"norm_bwd [in place, q/k slots D={D}]"
    fr.check(what)
    for (g, dw, *_), ref in zip(gots, refs):
        _outs(what, {"dx": "dx16", "dweight": "pgrad"}, {"dx": g, "dweight": dw}, ref)


# ---------------------------------------------------------------- q-norm + k-norm pair
@pytest.mark.parametrize("D", [264, 384, 1024, 1408, 1536])
@pytest.mark.parametrize("M", [13, 417, 8449])
@pytest.mark.parametrize("with_grads", [True, False])
def test_rmsnorm_pair(cuda_lib, D, M, with_grads):
    from internvideo_b200 import lowlevel as ll
    _seed("pair", D, M, with_grads)
    fr = Frame()
    qkv = fr.mat(M, 3 * D, bf16, torch.randn(M, 3 * D, device="cuda"), writes=False)
    out = fr.mat(M, 2 * D, bf16)
    w0, _ = _weights(D)
    w1, _ = _weights(D)
    fr.arm()
    rstd = ll.rmsnorm_pair_fwd(qkv, D, w0, w1, out)
    what = f"rmsnorm_pair_fwd [D={D} M={M}]"
    fr.check(what)
    for part, w in ((0, w0), (1, w1)):
        ref = rr.norm_fwd(qkv[:, part * D:(part + 1) * D], w, None, 1e-6, False)
        _outs(f"{what} part {part}", {}, {"y": out[:, part * D:(part + 1) * D], "rstd": rstd[:, part]}, ref)
    fb = Frame()
    fb.items = [it for it in fr.items if not it[1]]                 # qkv: an input now
    dqkv_buf = torch.full((M + 2, 3 * D + 8), math.nan, device="cuda", dtype=bf16)
    dqkv = dqkv_buf[1:M + 1, :3 * D]
    dqkv.copy_(torch.randn(M, 3 * D, device="cuda"))
    fb.watch(dqkv_buf, dqkv[:, :2 * D])
    dws = [fb.vec(D, torch.randn(D, device="cuda")) if with_grads else None for _ in range(2)]
    refs = [rr.norm_bwd(dqkv[:, p * D:(p + 1) * D], qkv[:, p * D:(p + 1) * D], w, None, rstd[:, p], False, None, dws[p])
            for p, w in ((0, w0), (1, w1))]
    fb.arm()
    ll.rmsnorm_pair_bwd(dqkv, qkv, D, w0, w1, rstd, dws[0], dws[1])
    what = f"rmsnorm_pair_bwd [D={D} M={M} grads={with_grads}]"
    fb.check(what)
    for p in (0, 1):
        got = {"dx": dqkv[:, p * D:(p + 1) * D]} | ({"dweight": dws[p]} if with_grads else {})
        _outs(f"{what} part {p}", {"dx": "dx16", "dweight": "pgrad"}, got, refs[p])


# ---------------------------------------------------------------- fused RMSNorm + LayerScale backward
FUSED_CASES = ([(1408, M, fin, frs, absent) for M in (1, 5, 13344) for fin in (True, False) for frs in (True, False)
                for absent in (None, "dweight", "dgamma", "dcolsum")]
               + [(1600, M, True, True, None) for M in (5, 13344)] + [(2064, M, False, True, None) for M in (5, 13344)])


def _fused_call(fr, D, M, with_in, with_rs, absent):
    from internvideo_b200 import lowlevel as ll
    x = fr.mat(M, D, f32, torch.randn(M, D, device="cuda") * 2 + 0.3, pad=4, writes=False)
    w, _ = _weights(D)
    _, rstd = _stats(torch.empty((M, D), device="cuda").copy_(x), w, None, False)   # norm_fwd: fp32 pitches of 8
    dy = fr.mat(M, D, bf16, torch.randn(M, D, device="cuda"), writes=False)
    ybr = fr.mat(M, D, bf16, torch.randn(M, D, device="cuda"), writes=False)
    dx_in = fr.mat(M, D, f32, torch.randn(M, D, device="cuda"), pad=4, writes=False) if with_in else None
    gamma = (torch.randn(D, device="cuda") * 0.1).to(bf16)
    rs = fr.vec(M, _rowscale(M), writes=False) if with_rs else None
    dx = fr.mat(M, D, f32, pad=4)
    dyb = fr.mat(M, D, bf16)
    g = {k: (None if k == absent else fr.vec(D, torch.randn(D, device="cuda"))) for k in ("dweight", "dgamma", "dcolsum")}
    ref = rr.rmsnorm_bwd_layerscale(dy, x, w, rstd, dx_in, ybr, gamma, g["dweight"], g["dgamma"], g["dcolsum"], rs)
    fr.arm()
    ll._call("rmsnorm_bwd_layerscale", dy, dy.stride(0), x, x.stride(0), w, rstd, M, D, dx_in,
             dx_in.stride(0) if with_in else 0, dx, dx.stride(0), g["dweight"], ybr, ybr.stride(0), gamma, rs, dyb,
             dyb.stride(0), g["dgamma"], g["dcolsum"])
    return ref, {"dx": dx, "dyb": dyb} | {k: v for k, v in g.items() if v is not None}


@pytest.mark.parametrize("D,M,with_in,with_rs,absent", FUSED_CASES)
def test_rmsnorm_bwd_layerscale(cuda_lib, D, M, with_in, with_rs, absent):
    _seed("fused", D, M, with_in, with_rs, absent)
    fr = Frame()
    ref, got = _fused_call(fr, D, M, with_in, with_rs, absent)
    what = f"rmsnorm_bwd_layerscale [D={D} M={M} dx_in={with_in} rowscale={with_rs} without {absent}]"
    fr.check(what)
    _outs(what, {"dx": "dx32", "dyb": "dx16", "dweight": "pgrad", "dgamma": "pgrad", "dcolsum": "pgrad"}, got, ref)


@pytest.mark.parametrize("D,with_in", [(1608, True), (2072, False)])
def test_rmsnorm_bwd_layerscale_refuses_past_the_row_ring(cuda_lib, D, with_in):
    """One row per ring slot must fit shared memory: D <= 1600 with dx_in, D <= 2064 without; past that the call is
    refused, with nothing written."""
    from internvideo_b200 import _lib
    fr = Frame()
    with pytest.raises(_lib.IvbError, match="too large for the shared-memory row ring"):
        _fused_call(fr, D, 5, with_in, True, None)
    fr.check(f"rmsnorm_bwd_layerscale [refused D={D}]")


# ---------------------------------------------------------------- LayerScale backward, column sums
LS_D = [8, 264, 1408, 4224, 6144]
LS_M = [1, 63, 64, 65, 127, 129, 13344]
LS_CASES = ([(D, M, None) for D in LS_D for M in LS_M]
            + [(D, M, a) for D in (264, 6144) for M in (65, 13344) for a in ("y", "gamma", "rowscale", "dgamma", "dcolsum")])


@pytest.mark.parametrize("D,M,absent", LS_CASES)
def test_layerscale_bwd(cuda_lib, D, M, absent):
    from internvideo_b200 import lowlevel as ll
    _seed("ls", D, M, absent)
    fr = Frame()
    dx = fr.mat(M, D, f32, torch.randn(M, D, device="cuda"), writes=False)
    y = fr.mat(M, D, bf16, torch.randn(M, D, device="cuda"), writes=False) if absent != "y" else None
    gamma = (torch.randn(D, device="cuda") * 0.1).to(bf16) if absent != "gamma" else None
    rs = fr.vec(M, _rowscale(M), writes=False) if absent != "rowscale" else None
    # without y the call writes no dgamma: it must keep its bits
    dg = fr.vec(D, torch.randn(D, device="cuda"), writes=y is not None) if absent != "dgamma" else None
    dc = fr.vec(D, torch.randn(D, device="cuda")) if absent != "dcolsum" else None
    out = fr.mat(M, D, bf16)
    ref = rr.layerscale_bwd(dx, y, gamma, dg, dc, rs)
    fr.arm()
    ll.layerscale_bwd(dx, y, gamma, dg, dc, out=out, rowscale=rs)
    what = f"layerscale_bwd [D={D} M={M} without {absent}]"
    fr.check(what)
    got = {"dy": out} | ({"dgamma": dg} if (y is not None and dg is not None) else {}) | ({"dcolsum": dc} if dc is not None else {})
    _outs(what, {"dy": "dx16", "dgamma": "pgrad", "dcolsum": "pgrad"}, got, ref)


@pytest.mark.parametrize("N", LS_D)
@pytest.mark.parametrize("M", LS_M)
def test_colsum(cuda_lib, N, M):
    from internvideo_b200 import lowlevel as ll
    _seed("colsum", N, M)
    fr = Frame()
    x = fr.mat(M, N, bf16, torch.randn(M, N, device="cuda"), writes=False)
    out = fr.vec(N, torch.randn(N, device="cuda"))
    ref = rr.colsum(x, out)
    fr.arm()
    ll.colsum(x, out=out)
    what = f"colsum_bf16 [N={N} M={M}]"
    fr.check(what)
    _outs(what, {"out": "pgrad"}, {"out": out}, ref)


# ---------------------------------------------------------------- LayerNorm -> L2 (decoder heads)
LNL2_CASES = [(768, bf16), (1408, bf16), (3200, bf16), (3328, bf16), (3336, bf16), (3200, f32), (3208, f32), (264, f32)]


def _ln_l2_fwd(fr, z, w, b, tgt, with_out, loss):
    from internvideo_b200 import lowlevel as ll
    M, C = z.shape
    out = fr.mat(M, C, bf16) if with_out else None
    sbuf = torch.full((3 * M + 8,), math.nan, device="cuda")
    stats = sbuf[4:4 + 3 * M]
    fr.watch(sbuf, stats)
    fr.arm()
    ll._call("ln_l2_fwd", z, z.stride(0), w, b, 1e-5, M, C, out, out.stride(0) if with_out else 0, stats, tgt,
             int(tgt is not None and tgt.dtype == f32), tgt.stride(0) if tgt is not None else 0, loss)
    return out, stats.view(M, 3)


@pytest.mark.parametrize("C", [8, 768, 1408, 3200, 3336])
@pytest.mark.parametrize("tdt", [bf16, f32, None])
@pytest.mark.parametrize("with_out", [True, False])
@pytest.mark.parametrize("M", [1, 417])
def test_ln_l2_fwd(cuda_lib, C, tdt, with_out, M):
    _seed("lnl2f", C, str(tdt), with_out, M)
    fr = Frame()
    z = fr.mat(M, C, bf16, torch.randn(M, C, device="cuda") * 1.5 + 0.2, writes=False)
    w, b = _weights(C, True)
    tgt = (fr.mat(M, C, tdt, torch.nn.functional.normalize(torch.randn(M, C, device="cuda"), dim=-1), writes=False)
           if tdt is not None else None)
    loss = fr.vec(1, torch.full((1,), 1.5, device="cuda")) if tdt is not None else None
    ref = rr.ln_l2_fwd(z, w, b, 1e-5, tgt, loss)
    out, stats = _ln_l2_fwd(fr, z, w, b, tgt, with_out, loss)
    what = f"ln_l2_fwd [C={C} M={M} target={tdt} out={with_out}]"
    fr.check(what)
    got = {"mean": stats[:, 0], "rstd": stats[:, 1], "inv_n": stats[:, 2]}
    got |= ({"out": out} if with_out else {}) | ({"loss": loss} if tdt is not None else {})
    if not with_out:
        ref.pop("out")
    _outs(what, {"out": "y", "inv_n": "rstd"}, got, ref)


@pytest.mark.parametrize("C,ddt", LNL2_CASES)
@pytest.mark.parametrize("grads", ["both", "dweight", "none"])
@pytest.mark.parametrize("M", [1, 2049])
def test_ln_l2_bwd(cuda_lib, C, ddt, grads, M):
    """Register-resident kernels (bf16 dout, C <= 3328: NCH 3, 6, 13), the streaming kernel (bf16 at C = 3336, fp32
    at any C; wpb 8 at C = 3200, 4 at 3208) with the alignment loss's dout = target, gscale_host = -2/M and a device
    scale != 1."""
    from internvideo_b200 import lowlevel as ll
    _seed("lnl2b", C, str(ddt), grads, M)
    fr = Frame()
    z = fr.mat(M, C, bf16, torch.randn(M, C, device="cuda") * 1.5 + 0.2, writes=False)
    w, b = _weights(C, True)
    _, stats = ll.ln_l2_fwd(z, w, b, want_out=False)
    dout = fr.mat(M, C, ddt, torch.nn.functional.normalize(torch.randn(M, C, device="cuda"), dim=-1), writes=False)
    gd = torch.full((1,), 0.75, device="cuda")
    dw = fr.vec(C, torch.randn(C, device="cuda")) if grads != "none" else None
    db = fr.vec(C, torch.randn(C, device="cuda")) if grads == "both" else None
    dz = fr.mat(M, C, bf16)
    ref = rr.ln_l2_bwd(z, w, b, stats, dout, -2.0 / M, gd, dw, db)
    fr.arm()
    ll._call("ln_l2_bwd", z, z.stride(0), w, b, stats, M, C, dout, int(ddt == f32), dout.stride(0), -2.0 / M, gd, dz,
             dz.stride(0), dw, db)
    what = f"ln_l2_bwd [C={C} M={M} dout={ddt} grads={grads}]"
    fr.check(what)
    got = {"dz": dz} | ({"dweight": dw} if dw is not None else {}) | ({"dbias": db} if db is not None else {})
    _outs(what, {"dz": "dx16", "dweight": "pgrad", "dbias": "pgrad"}, got, ref)


# ---------------------------------------------------------------- F.normalize rows
@pytest.mark.parametrize("C", [8, 264, 768])
@pytest.mark.parametrize("xdt", [f32, bf16])
def test_l2norm_rows(cuda_lib, C, xdt):
    from internvideo_b200 import lowlevel as ll
    _seed("l2n", C, str(xdt))
    M = 37
    fr = Frame()
    xv = torch.randn(M, C, device="cuda")
    xv[5] = 0.0                                                      # the 1e-12 clamp
    x = fr.mat(M, C, xdt, xv, writes=False)
    out = fr.mat(M, C, bf16)
    inv = fr.vec(M)
    ref = rr.l2norm_rows_fwd(x)
    fr.arm()
    ll._call("l2norm_rows_fwd", x, int(xdt == f32), x.stride(0), M, C, out, out.stride(0), inv)
    what = f"l2norm_rows_fwd [C={C} x={xdt}]"
    fr.check(what)
    _outs(what, {"out": "y", "inv": "rstd"}, {"out": out, "inv": inv}, ref)
    fb = Frame()
    dy = fb.mat(M, C, f32, torch.randn(M, C, device="cuda"), writes=False)
    dx = fb.mat(M, C, f32)
    refb = rr.l2norm_rows_bwd(dy, out, inv)
    fb.arm()
    ll._call("l2norm_rows_bwd", dy, dy.stride(0), out, out.stride(0), inv, M, C, dx, dx.stride(0))
    what = f"l2norm_rows_bwd [C={C} x={xdt}]"
    fb.check(what)
    _outs(what, {"dx": "dx32"}, {"dx": dx}, refb)


# ---------------------------------------------------------------- video-text contrastive loss
def _vtc_idx(G, mode):
    if mode == "distinct":
        return torch.arange(G, device="cuda") * 3 + 1
    if mode == "equal":
        return torch.full((G,), 5, device="cuda", dtype=torch.int64)
    return torch.randint(0, max(1, G // 3), (G,), device="cuda")


@pytest.mark.parametrize("G", [1, 2, 31, 256, 257, 1024])
@pytest.mark.parametrize("mode", ["distinct", "repeats", "equal"])
@pytest.mark.parametrize("dev_temp", [False, True])
def test_vtc_loss(cuda_lib, G, mode, dev_temp):
    from internvideo_b200 import lowlevel as ll
    _seed("vtc", G, mode, dev_temp)
    idx = _vtc_idx(G, mode).to(torch.int64)
    v = torch.nn.functional.normalize(torch.randn(G, 64, device="cuda"), dim=-1)
    t = torch.nn.functional.normalize(v + 0.7 * torch.randn(G, 64, device="cuda"), dim=-1)
    cos = (v @ t.t()).contiguous()
    temp = 0.07
    temp_dev = torch.full((1,), 0.0625, device="cuda") if dev_temp else None
    fr = Frame()
    lse_r, lse_c = fr.vec(G), fr.vec(G)
    loss = fr.vec(1, torch.full((1,), 0.5, device="cuda"))
    ref = rr.vtc_loss_fwd(cos, idx, temp, temp_dev, loss)
    fr.arm()
    ll._call("vtc_loss_fwd", cos, idx, G, temp, temp_dev, lse_r, lse_c, loss)
    what = f"vtc_loss_fwd [G={G} idx {mode} temp_dev={dev_temp}]"
    fr.check(what)
    _outs(what, {"lse_r": "loss", "lse_c": "loss"}, {"lse_r": lse_r, "lse_c": lse_c, "loss": loss}, ref)
    fb = Frame()
    dcos = fb.mat(G, G, bf16, pad=0)
    dtemp = fb.vec(1, torch.full((1,), -0.25, device="cuda"))
    gd = torch.full((1,), 1.5, device="cuda")
    refb = rr.vtc_loss_bwd(cos, idx, temp, lse_r, lse_c, 0.5, gd, temp_dev, dtemp)
    fb.arm()
    ll._call("vtc_loss_bwd", cos, idx, G, temp, temp_dev, lse_r, lse_c, 0.5, gd, dcos, dtemp)
    what = f"vtc_loss_bwd [G={G} idx {mode} temp_dev={dev_temp}]"
    fb.check(what)
    _outs(what, {"dcos": "dx16", "dtemp": "loss"}, {"dcos": dcos, "dtemp": dtemp}, refb)


# ---------------------------------------------------------------- MSE
MSE_N = [1, 255, 2 * 132 * 8 * 256 + 17]                             # the last: more than one persistent grid


@pytest.mark.parametrize("n", MSE_N)
@pytest.mark.parametrize("absent", [None, "dpred", "loss_sum"])
def test_mse_loss(cuda_lib, n, absent):
    from internvideo_b200 import lowlevel as ll
    _seed("mse", n, absent)
    fr = Frame()
    pred = fr.vec(n, torch.randn(n, device="cuda"), dtype=bf16, writes=False)
    label = fr.vec(n, torch.randn(n, device="cuda"), writes=False)
    loss = fr.vec(1, torch.full((1,), 3.0, device="cuda")) if absent != "loss_sum" else None
    dpred = fr.vec(n, dtype=bf16) if absent != "dpred" else None
    gd = torch.full((1,), 0.375, device="cuda")
    ref = rr.mse_loss(pred, label, loss, 1.0 / n, gd, dpred)
    fr.arm()
    ll.mse_loss(pred, label, loss, gscale_host=1.0 / n, gscale_dev=gd, dpred=dpred)
    what = f"mse_loss [n={n} without {absent}]"
    fr.check(what)
    got = ({"loss": loss} if loss is not None else {}) | ({"dpred": dpred} if dpred is not None else {})
    _outs(what, {"dpred": "dx16"}, got, ref)


# ---------------------------------------------------------------- AdamW
HP = dict(lr=1e-3, beta1=0.9, beta2=0.95, eps=1e-8, wd=0.05)


def _adamw_state(n, off, gdt):
    """master, m, v, grad and the bf16 copy as [n] slices at element `off` of larger buffers, as the engine's flat
    buckets hand them over (off = 1..3 selects the kernel's scalar path)."""
    bufs = [torch.full((n + 8,), math.nan, device="cuda") for _ in range(3)]
    master, m, v = (b[off:off + n] for b in bufs)
    master.copy_(torch.randn(n, device="cuda"))
    m.copy_(torch.randn(n, device="cuda") * 1e-3)
    v.copy_(torch.rand(n, device="cuda") * 1e-5)
    gbuf = torch.full((n + 8,), math.nan, device="cuda", dtype=gdt)
    grad = gbuf[off:off + n]
    pbuf = torch.full((n + 8,), math.nan, device="cuda", dtype=bf16)
    pb = pbuf[off:off + n]
    return bufs + [gbuf, pbuf], (master, m, v, grad, pb)


@pytest.mark.parametrize("n", [1, 3, 4, 10007])
@pytest.mark.parametrize("off", [0, 1, 2, 3])
@pytest.mark.parametrize("gdt", [f32, bf16])
def test_adamw_step(cuda_lib, n, off, gdt):
    from internvideo_b200 import lowlevel as ll
    _seed("adamw", n, off, str(gdt))
    bufs, (master, m, v, grad, pb) = _adamw_state(n, off, gdt)
    gsd = torch.full((1,), 0.5, device="cuda")
    for step in (1, 2, 7):
        grad.copy_(torch.randn(n, device="cuda"))
        ref = rr.adamw_step(master, m, v, grad, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], HP["wd"], step, 0.8, gsd)
        fr = Frame()
        for b in bufs:
            fr.watch(b, *[t for t in (master, m, v, pb) if t.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()])
        fr.arm()
        ll.adamw_step(master, m, v, grad, pb, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], HP["wd"], step,
                      grad_scale=0.8, grad_scale_dev=gsd)
        what = f"adamw_step [n={n} offset={off} grad={gdt} step={step}]"
        fr.check(what)
        _outs(what, {"master": "adamw", "exp_avg": "adamw", "exp_avg_sq": "adamw"},
              {"master": master, "exp_avg": m, "exp_avg_sq": v}, ref)
        assert torch.equal(pb, master.to(bf16)), what


@pytest.mark.parametrize("n,off", [(10007, 0), (10007, 1), (3, 0)])
def test_adamw_dyn_lr_step_matches_host(cuda_lib, n, off):
    """A device-resident {lr, step} gives the bits the host lr and step give, step after step."""
    from internvideo_b200 import lowlevel as ll
    _seed("adamw-dyn", n, off)
    _, host = _adamw_state(n, off, f32)
    _, dev = _adamw_state(n, off, f32)
    for a, b in zip(host, dev):
        b.copy_(a)
    for step, lr in ((1, 1e-3), (2, 7.5e-4), (3, 3e-4), (10, 1e-4), (1000, 2e-5)):
        g = torch.randn(n, device="cuda")
        host[3].copy_(g); dev[3].copy_(g)
        ll.adamw_step(*host[:4], host[4], lr, HP["beta1"], HP["beta2"], HP["eps"], HP["wd"], step)
        dyn = torch.tensor([lr, float(step)], device="cuda")
        ll.adamw_step(*dev[:4], dev[4], 123.0, HP["beta1"], HP["beta2"], HP["eps"], HP["wd"], 99, dyn_lr_step=dyn)
        for name, a, b in zip(("master", "exp_avg", "exp_avg_sq", "grad", "param_bf16"), host, dev):
            assert torch.equal(a.view(torch.int32 if a.dtype == f32 else torch.int16),
                               b.view(torch.int32 if b.dtype == f32 else torch.int16)), f"step {step}: {name} differs"


@pytest.mark.parametrize("bad", [0.0, -1.0, math.nan, math.inf])
@pytest.mark.parametrize("n,off", [(10007, 0), (10007, 1)])
def test_adamw_bad_step_leaves_state(cuda_lib, bad, n, off):
    """A device gradient scale that is not a positive finite number marks a bad step: master, m, v and the bf16 copy
    keep their bits."""
    from internvideo_b200 import lowlevel as ll
    bufs, (master, m, v, grad, pb) = _adamw_state(n, off, bf16)
    pb.copy_(master.to(bf16))
    grad.copy_(torch.randn(n, device="cuda"))
    fr = Frame()
    for b in bufs:
        fr.watch(b)
    fr.arm()
    ll.adamw_step(master, m, v, grad, pb, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], HP["wd"], 3,
                  grad_scale_dev=torch.full((1,), bad, device="cuda"))
    fr.check(f"adamw_step [grad_scale_dev={bad}]")


# ---------------------------------------------------------------- norm_fwd_fp8
@pytest.mark.parametrize("kind", ["rms", "ln"])
@pytest.mark.parametrize("D", [264, 1024, 1536, 3200])
def test_norm_fwd_fp8_row_is_the_norm_fwd_row(cuda_lib, kind, D):
    """At each NCH (2, 4, 6, 16) the E4M3 row times its scale is the fp32 row norm_fwd rounds to bf16, rounded to
    E4M3 instead: within half an E4M3 ulp plus row_ref's fp32 scale of the float64 row."""
    from internvideo_b200 import lowlevel as ll
    _seed("fp8", kind, D)
    ln = kind == "ln"
    M = 417
    x = torch.randn(M, D, device="cuda") * 2 + 0.3
    w, b = _weights(D, ln)
    q, sinv = ll.norm_fwd_fp8(x, w, b, eps=1e-5 if ln else 1e-6, layernorm=ln)
    ref, scale = rr.norm_fwd(x, w, b, 1e-5 if ln else 1e-6, ln)["y"]
    s = sinv.double()[:, None]
    ys = ref / s                                                      # the row in the E4M3 grid's units
    e = torch.floor(torch.log2(ys.abs().clamp_min(2.0 ** -6)))
    half = torch.exp2(e - 4)                                          # half an E4M3 ulp (3 mantissa bits)
    errs = (q.double() - ys).abs() / (half + scale / s)
    i = int(errs.argmax())
    assert float(errs.reshape(-1)[i]) <= LIMITS["fp8"], f"norm_fwd_fp8 [{kind} D={D}]: {float(errs.reshape(-1)[i]):.3g} at {divmod(i, D)}"
