"""Every fused GEMM epilogue, element by element against float64 (tests/gemm_ref.py), on every kernel ivb_gemm_bf16 can
select: the cooperative kernel (IVB_FLAG_1CTA) at tile_n 128 / 176 / 192 / 256, the ping-pong kernel, the CTA pair
(IVB_FLAG_2CTA) at the same four widths, and the default selection (gpu).

Each check is the largest per-element error divided by its tolerance (gemm_ref.elem_errors: half an ulp of the output
format plus the accumulation, evaluation and GELU-form error bounds); a failure names the kernel tile, warpgroup band
and 16-column epilogue chunk of the worst element.  Every output is written as a view into a NaN-filled buffer wider
than N, and nothing outside the view may change.

The tolerance is a bound, not a fit: the worst element of every family measured below 1 on the H100.  The elementwise
check cannot see an error smaller than the tanh form's own budget (tanh.approx.f32, about 2^-11 of t), such as the erf
derivative in place of the tanh one (at most 8.7e-4 off); gemm_ref.binned_bias, the mean signed error per bin of the
pre-activation, checks the GELU derivative outputs for such systematic errors.

Each limit in LIMITS is at most twice the worst value measured over this file on an H100 80GB HBM3 (SXM, 700 W power
limit); the measured value is beside it.  The file (792 tests) runs in about 20 s there.
"""
import pytest
import torch

from gemm_ref import binned_bias, elem_errors, gemm_ref, half_ulp, worst

pytestmark = pytest.mark.gpu

bf, f32 = torch.bfloat16, torch.float32
PAD = 24

# limit, and beside it the worst value measured over this file (H100 80GB HBM3 SXM, 700 W power limit)
LIMITS = {
    "bf16": 1.9,        # out0 of EPI_BF16 (bias, ACCUM)                 measured 0.99999
    "f32": 1.4,         # out0 of EPI_F32 (bias, ACCUM)                  measured 0.742
    "gelu": 1.9,        # out0 of EPI_BIAS_GELU                          measured 0.99947
    "gelu_h": 1.9,      # out1 = h                                       measured 0.99931
    "gelu_d": 1.9,      # out1 = gelu'(h) (FLAG_GELU_SAVE_GRAD)          measured 0.99972
    "resid": 1.9,       # out0 of EPI_RESID                              measured 0.99933
    "resid_y": 1.9,     # out1 = y of EPI_RESID                          measured 0.99998
    "gelu_bwd": 1.9,    # out0 of EPI_GELU_BWD                           measured 0.99997
    # largest mean signed error over a 0.25-wide bin of h, in units of the tolerance (gemm_ref.binned_bias)
    "gelu_d_bias": 0.0097,   # out1 = gelu'(h)                           measured 0.00489
    "gelu_bwd_bias": 0.045,  # out0 of EPI_GELU_BWD, erf and tanh forms  measured 0.0227
}


def _within(family, e, msg):
    assert e <= LIMITS[family], msg


# ---------------------------------------------------------------- kernels
class Kernel:
    def __init__(self, name, flag, tile_n, bm, bn):
        self.name, self.flag, self.tile_n, self.bm, self.bn = name, flag, tile_n, bm, bn

    def __repr__(self):
        return self.name


def _kernels():
    FL_1CTA, FL_2CTA, FL_PP = 4, 8, 32
    ks = [Kernel(f"coop{bn}", FL_1CTA, bn, 128, bn) for bn in (128, 176, 192, 256)]
    ks.append(Kernel("pingpong", FL_PP, 0, 128, 128))
    ks += [Kernel(f"pair{bn}", FL_2CTA, bn, 256, bn) for bn in (128, 176, 192, 256)]
    ks.append(Kernel("default", 0, 0, 128, 128))     # tiles named as 128 x 128; bands and chunks do not depend on it
    return ks


KERNELS = _kernels()


# ---------------------------------------------------------------- operands and epilogues
def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(bf)


def _bits(t):
    return t.view(torch.int16) if t.dtype == bf else t.view(torch.int32)


def _operands(layout, M, N, K, seed):
    if layout == "nt":       # y = x W^T
        return _mk((M, K), seed), _mk((N, K), seed + 1, 0.05), False, False
    if layout == "dgrad":    # dx = dy W
        return _mk((M, K), seed), _mk((K, N), seed + 1, 0.05), False, True
    # wgrad dW = dy^T x, dy a view whose pitch is a multiple of 8 whatever M is
    return _mk((K, (M + 7) // 8 * 8 + 8), seed)[:, :M], _mk((K, N), seed + 1, 0.05), True, True


def _view(rows, N, dtype, narrow, init=None):
    """A [rows, N] view into a NaN-filled buffer.  Wide: pitch N + PAD (rows 32-byte aligned when N + PAD is a
    multiple of 16).  Narrow: bf16 rows at a pitch of 8 (mod 16) elements, so every other row is 16- but not 32-byte
    aligned; fp32 rows start 4 columns into the buffer (16- but not 32-byte aligned)."""
    if not narrow:
        buf = torch.full((rows, N + PAD), float("nan"), device="cuda", dtype=dtype)
        v = buf[:, :N]
    elif dtype == bf:
        pitch = N + 8 if N % 16 == 0 else N + 16
        buf = torch.full((rows, pitch), float("nan"), device="cuda", dtype=dtype)
        v = buf[:, :N]
    else:
        buf = torch.full((rows, N + 16), float("nan"), device="cuda", dtype=dtype)
        v = buf[:, 4:4 + N]
    if init is not None:
        v.copy_(init)
    return buf, v


def _vec(N, seed, scale, narrow):
    """bias / gamma: a length-N bf16 vector, 16- but not 32-byte aligned when narrow."""
    buf = torch.full((N + 16,), float("nan"), device="cuda", dtype=bf)
    off = 8 if narrow else 0
    buf[off:off + N] = _mk((N,), seed, scale)
    return buf[off:off + N]


def _gelu_grad_bf16(h, tanh):
    x = h.double().requires_grad_(True)
    (d,) = torch.autograd.grad(torch.nn.functional.gelu(x, approximate="tanh" if tanh else "none").sum(), x)
    return d.to(bf)


EPI_BF16, EPI_F32, EPI_BIAS_GELU, EPI_RESID, EPI_GELU_BWD = 0, 1, 2, 3, 4
F_TANH, F_ACCUM, F_SAVE = 1, 2, 16

EPILOGUES = ["bf16", "bf16_bias", "accum_bf16", "accum_bf16_bias", "f32", "f32_bias", "accum_f32", "accum_f32_bias",
             "gelu_erf", "gelu_tanh", "gelu_erf_save", "gelu_tanh_save",
             "resid", "resid_gamma", "resid_rowscale", "resid_gamma_rowscale_out1",
             "gelu_bwd_erf", "gelu_bwd_tanh", "gelu_bwd_save"]
EDGE_EPILOGUES = ["bf16_bias", "gelu_tanh_save", "resid_gamma_rowscale_out1", "gelu_bwd_save", "accum_bf16"]


def _rowscale(M, seed, keep=0.75):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(M, device="cuda", generator=g) < keep).float() / keep


def _epilogue(name, M, N, seed, narrow):
    """(epi, flags, kwargs of lowlevel.gemm except out0/out1, out0 init or None, writes out1, output families)."""
    kw = {}
    if "bias" in name or (name.startswith("gelu_") and not name.startswith("gelu_bwd")) or name.startswith("resid"):
        kw["bias"] = _vec(N, seed + 10, 0.1, narrow)
    if name.startswith(("bf16", "accum_bf16", "f32", "accum_f32")):
        epi = EPI_F32 if "f32" in name else EPI_BF16
        flags, init = (F_ACCUM, None) if name.startswith("accum") else (0, None)
        if flags:
            init = torch.randn((M, N), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed + 13))
            init = init.to(bf) if epi == EPI_BF16 else init
        return epi, flags, kw, init, False, ["f32" if epi == EPI_F32 else "bf16"]
    if name.startswith("gelu_bwd"):
        flags = {"gelu_bwd_erf": 0, "gelu_bwd_tanh": F_TANH, "gelu_bwd_save": F_TANH | F_SAVE}[name]
        h = _mk((M, N), seed + 12, 1.5)
        aux = _gelu_grad_bf16(h, True) if flags & F_SAVE else h
        kw["aux"] = _view(M, N, bf, narrow, aux)[1]
        return EPI_GELU_BWD, flags, kw, None, False, ["gelu_bwd"]
    if name.startswith("gelu"):
        flags = (F_TANH if "tanh" in name else 0) | (F_SAVE if "save" in name else 0)
        return EPI_BIAS_GELU, flags, kw, None, True, ["gelu", "gelu_d" if flags & F_SAVE else "gelu_h"]
    if name.startswith("resid"):
        kw["aux"] = _view(M, N, f32, narrow, torch.randn((M, N), device="cuda"))[1]
        if "gamma" in name:
            kw["gamma"] = _vec(N, seed + 11, 0.5, narrow)
        if "rowscale" in name:
            kw["rowscale"] = _rowscale(M, seed)
        out1 = "out1" in name
        return EPI_RESID, 0, kw, None, out1, ["resid"] + (["resid_y"] if out1 else [])
    raise ValueError(name)


_CASES = {}


def _case(layout, name, M, N, K, seed, narrow):
    """Inputs and float64 references of one (layout, epilogue, shape), shared by every kernel."""
    key = (layout, name, M, N, K, seed, narrow)
    if key not in _CASES:
        if len(_CASES) > 64:
            _CASES.clear()
        a, b, a_t, b_t = _operands(layout, M, N, K, seed)
        epi, flags, kw, init, out1, fams = _epilogue(name, M, N, seed, narrow)
        refs = gemm_ref(a, b, a_t=a_t, b_t=b_t, epi=epi, flags=flags, out0=init,
                        out1=torch.empty(1) if out1 else None, **kw)
        hpre = None     # the pre-activation of a GELU derivative output, for binned_bias
        if epi == EPI_GELU_BWD and not flags & F_SAVE:
            hpre = kw["aux"].double()
        elif epi == EPI_BIAS_GELU and flags & F_SAVE:
            hpre = gemm_ref(a, b, a_t=a_t, b_t=b_t, epi=epi, flags=flags & ~F_SAVE, out1=torch.empty(1), **kw)[1][0]
        _CASES[key] = (a, b, a_t, b_t, epi, flags, kw, init, out1, fams, refs, hpre)
    return _CASES[key]


def _run_and_check(ll, kern, layout, name, M, N, K, seed=100, narrow=False):
    a, b, a_t, b_t, epi, flags, kw, init, want_out1, fams, refs, hpre = _case(layout, name, M, N, K, seed, narrow)
    out_dtype = f32 if epi in (EPI_F32, EPI_RESID) else bf
    bufs = [_view(M, N, out_dtype, narrow, init)]
    if want_out1:
        bufs.append(_view(M, N, bf, narrow))
    before = [_bits(buf).clone() for buf, _ in bufs]
    try:
        ll.gemm(a, b, a_t=a_t, b_t=b_t, epi=epi, flags=flags | kern.flag, out0=bufs[0][1],
                out1=bufs[1][1] if want_out1 else None, tile_n=kern.tile_n, **kw)
    except ll._lib.IvbError as e:
        pytest.skip(f"{kern}: refused by the library: {e}")
    torch.cuda.synchronize()
    what = f"{kern} {layout} {name} M={M} N={N} K={K}{' narrow' if narrow else ''}"
    for (buf, v), old, fam, (ref, scale) in zip(bufs, before, fams, refs):
        inside = torch.zeros_like(buf, dtype=torch.bool)
        inside[:, v.storage_offset() - buf.storage_offset():][:, :N] = True
        assert torch.equal(_bits(buf)[~inside], old[~inside]), f"{what}: {fam} written outside the output view"
        assert torch.isfinite(v).all(), f"{what}: {fam} has non-finite values"
        e, where = worst(elem_errors(v, ref, scale), kern.bm, kern.bn)
        _within(fam, e, f"{what}: {fam} error {e:.3g} x tol > {LIMITS[fam]} at {where}")
        if hpre is not None and fam in ("gelu_d", "gelu_bwd") and v.numel() >= 100000:
            e, edge = binned_bias(v, ref, scale, hpre)
            _within(fam + "_bias", e, f"{what}: {fam} mean error {e:.3g} x tol > {LIMITS[fam + '_bias']} "
                                      f"for h in [{edge}, {edge + 0.25})")


# ---------------------------------------------------------------- epilogue x layout matrix
@pytest.mark.parametrize("kern", KERNELS, ids=str)
@pytest.mark.parametrize("layout", ["nt", "dgrad", "wgrad"])
@pytest.mark.parametrize("epilogue", EPILOGUES)
def test_epilogue_matrix(cuda_lib, epilogue, layout, kern):
    _run_and_check(cuda_lib, kern, layout, epilogue, 417, 1000, 592)


# ---------------------------------------------------------------- edges of the tiling
@pytest.mark.parametrize("kern", KERNELS, ids=str)
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 129, 255, 257])
def test_tile_edges_rows(cuda_lib, M, kern):
    """Rows around the 64-row warpgroup bands and the 128- / 256-row tiles (the CTA pair's rank-1 CTA has no rows for
    M <= 128).  N = 440 leaves a ragged last tile for every tile width."""
    for layout in ("nt", "dgrad", "wgrad"):
        for name in EDGE_EPILOGUES:
            _run_and_check(cuda_lib, kern, layout, name, M, 440, 72)


def _edge_widths(bn):
    """N such that the last tile holds 8, 16, 24, 40 or bn - 8 valid columns, and N = 8."""
    return [8] + [bn + w for w in (8, 16, 24, 40, bn - 8)]


@pytest.mark.parametrize("kern", KERNELS, ids=str)
@pytest.mark.parametrize("wi", range(6))
def test_tile_edges_columns_narrow(cuda_lib, wi, kern):
    """The epilogue's half-chunk path (nvalid < 16) and its 16-byte (not 32-byte) row accesses: every output, aux,
    bias and gamma view is 16- but not 32-byte aligned on at least every other row."""
    N = _edge_widths(kern.bn)[wi]
    for K in (8, 56, 72):
        for layout in ("nt", "dgrad", "wgrad"):
            for name in EDGE_EPILOGUES:
                _run_and_check(cuda_lib, kern, layout, name, 129, N, K, seed=200 + K, narrow=True)


# ---------------------------------------------------------------- GELU over every bf16 value
def _ftz(x):
    return torch.where(x.abs() < 2.0 ** -126, torch.zeros_like(x), x)


def _all_bf16():
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(bf)


@pytest.mark.parametrize("kern", KERNELS, ids=str)
@pytest.mark.parametrize("flags", [0, F_TANH, F_SAVE, F_TANH | F_SAVE], ids=["erf", "tanh", "erf_save", "tanh_save"])
def test_gelu_every_bf16_value(cuda_lib, flags, kern):
    """EPI_BIAS_GELU with A = 0 and bias = h, so acc + bias is exactly h, over all 65536 bf16 patterns.  The bound holds
    for |h| <= 2^10; beyond it the forward stays finite, and so does gelu'(h) except the tanh form's for |h| >= 2^64
    (documented in ivb_ptx.cuh).  NaN propagates."""
    ll = cuda_lib
    h = _all_bf16()
    N, M, K = h.numel(), 2, 8
    a = torch.zeros((M, K), device="cuda", dtype=bf)
    b = torch.zeros((N, K), device="cuda", dtype=bf)
    g = torch.empty((M, N), device="cuda", dtype=bf)
    o1 = torch.empty((M, N), device="cuda", dtype=bf)
    try:
        ll.gemm(a, b, epi=EPI_BIAS_GELU, flags=flags | kern.flag, bias=h, out0=g, out1=o1, tile_n=kern.tile_n)
    except ll._lib.IvbError as e:
        pytest.skip(f"{kern}: refused by the library: {e}")
    torch.cuda.synchronize()
    assert torch.equal(_bits(g[0]), _bits(g[1])) and torch.equal(_bits(o1[0]), _bits(o1[1]))
    hd = h.double()
    fin = torch.isfinite(hd)
    live = fin & (hd.abs() <= 2.0 ** 10)
    (gr, gs), (dr, ds) = gemm_ref(a, b, epi=EPI_BIAS_GELU, flags=flags, bias=h, out1=o1)
    for got, ref, scale, fam in ((g[0], gr[0], gs[0], "gelu"),
                                 (o1[0], dr[0], ds[0], "gelu_d" if flags & F_SAVE else "gelu_h")):
        errs = elem_errors(got[live], ref[live], scale[live])
        i = int(errs.argmax())
        _within(fam, float(errs[i]), f"{kern} flags={flags}: {fam} error {float(errs[i]):.3g} x tol at h = "
                                     f"{float(hd[live][i]):.6g} (got {float(got[live][i]):.6g}, want {float(ref[live][i]):.6g})")
    assert torch.isfinite(g[0][fin]).all(), "gelu(h) is not finite for some finite h"
    if flags & F_SAVE:
        dom = fin & (hd.abs() < 2.0 ** 64) if flags & F_TANH else fin
        assert torch.isfinite(o1[0][dom]).all(), "gelu'(h) is not finite inside its documented domain"
        if flags & F_TANH:
            assert torch.isnan(o1[0][fin & ~dom]).all(), "the tanh gelu'(h) domain in ivb_ptx.cuh is out of date"
    else:                       # h = 0 + bias comes back exactly; subnormals flush to zero (--use_fast_math)
        assert (o1[0].double()[fin] == _ftz(hd)[fin]).all()
    nan = torch.isnan(hd)
    assert torch.isnan(g[0][nan]).all() and torch.isnan(o1[0][nan]).all()


@pytest.mark.parametrize("kern", KERNELS, ids=str)
@pytest.mark.parametrize("flags", [0, F_TANH, F_SAVE], ids=["erf", "tanh", "save"])
def test_gelu_bwd_every_bf16_value(cuda_lib, flags, kern):
    """EPI_GELU_BWD with acc = 1 exactly (one unit product per element) and aux = every bf16 pattern."""
    ll = cuda_lib
    aux = _all_bf16().reshape(256, 256)
    M, N, K = 256, 256, 8
    a = torch.zeros((M, K), device="cuda", dtype=bf)
    b = torch.zeros((N, K), device="cuda", dtype=bf)
    a[:, 0] = 1
    b[:, 0] = 1
    out = torch.empty((M, N), device="cuda", dtype=bf)
    try:
        ll.gemm(a, b, epi=EPI_GELU_BWD, flags=flags | kern.flag, aux=aux, out0=out, tile_n=kern.tile_n)
    except ll._lib.IvbError as e:
        pytest.skip(f"{kern}: refused by the library: {e}")
    torch.cuda.synchronize()
    hd = aux.double()
    fin = torch.isfinite(hd)
    nan = torch.isnan(hd)
    assert torch.isnan(out[nan]).all()
    if flags & F_SAVE:          # out = 1 * aux: every value but NaN comes back exactly, subnormals flushed to zero
        assert (out.double()[~nan] == _ftz(hd)[~nan]).all()
        return
    live = fin & (hd.abs() <= 2.0 ** 10)
    (ref, scale), = gemm_ref(a, b, epi=EPI_GELU_BWD, flags=flags, aux=aux)
    errs = elem_errors(out[live], ref[live], scale[live])
    i = int(errs.argmax())
    _within("gelu_bwd", float(errs[i]), f"{kern} flags={flags}: gelu_bwd error {float(errs[i]):.3g} x tol at h = "
                                        f"{float(hd[live][i]):.6g}")
    dom = fin & (hd.abs() < 2.0 ** 64) if flags & F_TANH else fin
    assert torch.isfinite(out[dom]).all()
    if flags & F_TANH:
        assert torch.isnan(out[fin & ~dom]).all(), "the tanh gelu'(h) domain in ivb_ptx.cuh is out of date"


# ---------------------------------------------------------------- LayerScale at its real size
@pytest.mark.parametrize("kern", KERNELS, ids=str)
def test_layerscale_real_size(cuda_lib, kern):
    """gamma = 1e-5 (1 + 0.1 noise), as the model initialises LayerScale; the residual stream of unit scale; rowscale
    of zeros and 1/keep.  out0 - aux, formed exactly in float64, is checked against rowscale * gamma * y: at this
    scale the branch is 1e-5 of out0, so a relative check of out0 could not see it.  Rows dropped by DropPath come
    back as the residual, bit for bit."""
    ll = cuda_lib
    M, N, K = 417, 1408, 592
    a, w = _mk((M, K), 500), _mk((N, K), 501, 0.05)
    bias = _mk((N,), 502, 0.1)
    gn = torch.Generator(device="cuda").manual_seed(503)
    gamma = (1e-5 * (1 + 0.1 * torch.randn(N, device="cuda", generator=gn))).to(bf)
    aux = torch.randn((M, N), device="cuda", generator=gn)
    rs = _rowscale(M, 504)
    buf, out = _view(M, N, f32, False)
    y = torch.empty((M, N), device="cuda", dtype=bf)
    try:
        ll.gemm(a, w, epi=EPI_RESID, bias=bias, gamma=gamma, aux=aux, rowscale=rs, out0=out, out1=y,
                flags=kern.flag, tile_n=kern.tile_n)
    except ll._lib.IvbError as e:
        pytest.skip(f"{kern}: refused by the library: {e}")
    torch.cuda.synchronize()
    (r0, s0), (r1, s1) = gemm_ref(a, w, epi=EPI_RESID, bias=bias, gamma=gamma, aux=aux, rowscale=rs, out1=y)
    branch_got = out.double() - aux.double()                  # exact: both are fp32
    branch_ref = r0 - aux.double()
    errs = (branch_got - branch_ref).abs() / (s0 + half_ulp(f32, r0))
    e, where = worst(errs, kern.bm, kern.bn)
    _within("resid", e, f"{kern}: LayerScale branch error {e:.3g} x tol at {where}")
    drop = rs == 0
    assert drop.any() and (~drop).any()
    assert torch.equal(_bits(out[drop]), _bits(aux[drop])), "a dropped row is not the residual bit for bit"
    e, where = worst(elem_errors(y, r1, s1), kern.bm, kern.bn)
    _within("resid_y", e, f"{kern}: y error {e:.3g} x tol at {where}")
    assert torch.isnan(buf[:, N:]).all()


# ---------------------------------------------------------------- the step's own GEMMs at full size
TOK, D, HD = 13344, 1408, 6144        # cfg-2: 32 clips x 417 tokens, InternVideo2-1B widths
STEP_GELU = F_TANH | F_SAVE           # FusedMLP's tanh GELU, gelu'(h) saved for the backward
FULL_CHUNK = 2048


def _check_full(fam, got, ref_args, what, out_index=0, **kw):
    """Whole-tensor check of a full-size output, reference computed 2048 rows at a time."""
    M = got.shape[0]
    worst_e, worst_where = -1.0, ""
    for r0 in range(0, M, FULL_CHUNK):
        rows = slice(r0, min(M, r0 + FULL_CHUNK))
        ref, scale = gemm_ref(*ref_args[0], rows=rows, **ref_args[1])[out_index]
        e, where = worst(elem_errors(got[rows], ref, scale), row0=r0, **kw)
        if e > worst_e:
            worst_e, worst_where = e, where
        del ref, scale
    _within(fam, worst_e, f"{what}: {fam} error {worst_e:.3g} x tol > {LIMITS[fam]} at {worst_where}")


def test_step_forward_full_size(cuda_lib):
    """proj and fc2 (EPI_RESID with gamma, rowscale and y saved) and fc1 (EPI_BIAS_GELU, tanh, gelu' saved), with the
    step's flags and the library's default kernel selection, as ops.block_forward launches them."""
    ll = cuda_lib
    rs = _rowscale(TOK, 600, keep=0.9)
    x = torch.randn((TOK, D), device="cuda", generator=torch.Generator(device="cuda").manual_seed(601))
    a = _mk((TOK, D), 602)
    projw, projb = _mk((D, D), 603, 0.03), _mk((D,), 604, 0.1)
    g1 = (1e-5 * (1 + 0.1 * torch.randn(D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(605)))).to(bf)
    y1 = torch.empty((TOK, D), device="cuda", dtype=bf)
    kw = dict(epi=EPI_RESID, bias=projb, gamma=g1, aux=x, rowscale=rs)
    x1 = ll.gemm(a, projw, out1=y1, **kw)
    torch.cuda.synchronize()
    _check_full("resid", x1, ((a, projw), dict(out1=y1, **kw)), "proj x1")
    _check_full("resid_y", y1, ((a, projw), dict(out1=y1, **kw)), "proj y1", out_index=1)
    del x, y1

    n2 = _mk((TOK, D), 606)
    fc1w, fc1b = _mk((HD, D), 607, 0.03), _mk((HD,), 608, 0.1)
    h = torch.empty((TOK, HD), device="cuda", dtype=bf)
    kw = dict(epi=EPI_BIAS_GELU, flags=STEP_GELU, bias=fc1b)
    g = ll.gemm(n2, fc1w, out1=h, **kw)
    torch.cuda.synchronize()
    _check_full("gelu", g, ((n2, fc1w), dict(out1=h, **kw)), "fc1 gelu(h)")
    _check_full("gelu_d", h, ((n2, fc1w), dict(out1=h, **kw)), "fc1 gelu'(h)", out_index=1)
    del h, n2

    fc2w, fc2b = _mk((D, HD), 609, 0.02), _mk((D,), 610, 0.1)
    g2 = _mk((D,), 611, 0.1)
    y2 = torch.empty((TOK, D), device="cuda", dtype=bf)
    kw = dict(epi=EPI_RESID, bias=fc2b, gamma=g2, aux=x1, rowscale=rs)
    x2 = ll.gemm(g, fc2w, out1=y2, **kw)
    torch.cuda.synchronize()
    _check_full("resid", x2, ((g, fc2w), dict(out1=y2, **kw)), "fc2 x2")
    _check_full("resid_y", y2, ((g, fc2w), dict(out1=y2, **kw)), "fc2 y2", out_index=1)


def test_step_backward_full_size(cuda_lib):
    """dh (EPI_GELU_BWD on the saved gelu') and the four weight gradients, accumulated (FLAG_ACCUM) into views of one
    flat bf16 gradient buffer laid out by the engine's plan_layout, as ops.block_backward launches them."""
    from internvideo_b200.engine import plan_layout
    ll = cuda_lib
    dy2 = _mk((TOK, D), 700)
    fc2w = _mk((D, HD), 701, 0.02)
    hsave = _gelu_grad_bf16(_mk((TOK, HD), 702, 1.5), True)
    kw = dict(b_t=True, epi=EPI_GELU_BWD, flags=STEP_GELU, aux=hsave)
    dh = ll.gemm(dy2, fc2w, **kw)
    torch.cuda.synchronize()
    _check_full("gelu_bwd", dh, ((dy2, fc2w), kw), "dh")
    del hsave, fc2w

    shapes = [("blocks.0.attn.qkv.weight", (3 * D, D)), ("blocks.0.attn.proj.weight", (D, D)),
              ("blocks.0.mlp.fc1.weight", (HD, D)), ("blocks.0.mlp.fc2.weight", (D, HD)),
              ("blocks.0.attn.qkv.bias", (3 * D,)), ("blocks.0.ls1.gamma", (D,))]
    entries, _, total = plan_layout(shapes)
    base = 8          # a block further down the buffer: 16- but not 32-byte aligned (the engine aligns to 8 elements)
    flat = _mk((base + total,), 703, 0.01)
    off = {name: base + o for name, o, _, _ in entries}
    n1, a, n2 = _mk((TOK, D), 704), _mk((TOK, D), 705), _mk((TOK, D), 706)
    g = _mk((TOK, HD), 707)
    dqkv, dy1 = _mk((TOK, 3 * D), 708), _mk((TOK, D), 709)
    for name, dy, act in (("blocks.0.mlp.fc2.weight", dy2, g), ("blocks.0.mlp.fc1.weight", dh, n2),
                          ("blocks.0.attn.proj.weight", dy1, a), ("blocks.0.attn.qkv.weight", dqkv, n1)):
        shape = dict(shapes)[name]
        view = flat[off[name]:off[name] + shape[0] * shape[1]].view(shape)
        old = view.clone()
        before = _bits(flat).clone()
        ll.gemm(dy, act, a_t=True, b_t=True, out0=view, flags=F_ACCUM)
        torch.cuda.synchronize()
        changed = _bits(flat) != before
        changed[off[name]:off[name] + view.numel()] = False
        assert not changed.any(), f"wgrad {name} wrote outside its slice of the flat buffer"
        _check_full("bf16", view, ((dy, act), dict(a_t=True, b_t=True, flags=F_ACCUM, out0=old)), f"wgrad {name}")
