"""The ping-pong GEMM kernel (IVB_FLAG_PINGPONG) against the cooperative kernel at tile_n = 128 (gpu).

Both run the same m64n128k16 wgmma in the same k order and the same epilogue code, so every output must be
bit-identical: every epilogue, every operand layout, tile counts per CTA of 1, odd, even and fewer tiles than SMs,
ragged M / N / K, and outputs written as views with a wider pitch into NaN-filled buffers (nothing outside a view
may change)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

bf, f32 = torch.bfloat16, torch.float32
PAD = 24          # extra columns of every output buffer beyond N (pitch N + PAD, a multiple of 8 when N is)


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(bf)


def _bits(t):
    return t.view(torch.int16) if t.dtype == bf else t.view(torch.int32)


def _nan_buf(M, N, dtype, init=None):
    """[M, N + PAD] buffer of NaN; the [:, :N] view holds `init` when given."""
    buf = torch.full((M, N + PAD), float("nan"), device="cuda", dtype=dtype)
    if init is not None:
        buf[:, :N] = init
    return buf


def _run(ll, kernel_flags, tile_n, a, b, a_t, b_t, M, N, epi, flags, want_out1, init0, **kw):
    out_dtype = f32 if epi in (ll.EPI_F32, ll.EPI_RESID) else bf
    o0 = _nan_buf(M, N, out_dtype, init0)
    o1 = _nan_buf(M, N, bf) if want_out1 else None
    ll.gemm(a, b, a_t=a_t, b_t=b_t, epi=epi, flags=flags | kernel_flags, out0=o0[:, :N],
            out1=None if o1 is None else o1[:, :N], tile_n=tile_n, **kw)
    return [o for o in (o0, o1) if o is not None]


def _check_pair(ll, a, b, a_t, b_t, M, N, epi=0, flags=0, want_out1=False, init0=None, **kw):
    ref = _run(ll, ll.FLAG_1CTA, 128, a, b, a_t, b_t, M, N, epi, flags, want_out1, init0, **kw)
    got = _run(ll, ll.FLAG_PINGPONG, 0, a, b, a_t, b_t, M, N, epi, flags, want_out1, init0, **kw)
    torch.cuda.synchronize()
    for r, g in zip(ref, got):
        assert torch.equal(_bits(g), _bits(r)), (M, N, epi, flags)
        assert torch.isnan(g[:, N:]).all(), "written outside the output view"
        assert torch.isfinite(g[:, :N]).all()
    return got


def _operands(layout, M, N, K, seed):
    if layout == "nt":       # y = x W^T
        return _mk((M, K), seed), _mk((N, K), seed + 1, 0.05), False, False
    if layout == "dgrad":    # dx = dy W
        return _mk((M, K), seed), _mk((K, N), seed + 1, 0.05), False, True
    # wgrad dW = dy^T x; dy is a view with a pitch that is a multiple of 8 whatever M is
    return _mk((K, (M + 7) // 8 * 8 + 8), seed)[:, :M], _mk((K, N), seed + 1, 0.05), True, True


# ---------------------------------------------------------------- every epilogue, every layout
EPILOGUES = ["bf16", "bf16_bias", "f32", "gelu_erf", "gelu_tanh", "gelu_erf_save", "gelu_tanh_save",
             "resid", "resid_gamma", "resid_gamma_rowscale_out1", "resid_rowscale", "gelu_bwd_erf", "gelu_bwd_tanh",
             "gelu_bwd_save", "accum_bf16", "accum_f32"]


def _epilogue_args(ll, name, M, N, seed):
    bias = _mk((N,), seed + 10, 0.1)
    gamma = _mk((N,), seed + 11, 0.5)
    rs = (torch.rand(M, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)) > 0.25).float() / 0.75
    if name == "bf16":
        return dict()
    if name == "bf16_bias":
        return dict(bias=bias)
    if name == "f32":
        return dict(epi=ll.EPI_F32, bias=bias)
    if name.startswith("gelu_bwd"):
        fl = {"gelu_bwd_erf": 0, "gelu_bwd_tanh": ll.FLAG_GELU_TANH, "gelu_bwd_save": ll.FLAG_GELU_SAVE_GRAD}[name]
        aux = torch.full((M, N + 8), float("nan"), device="cuda", dtype=bf)
        aux[:, :N] = _mk((M, N), seed + 12)
        return dict(epi=ll.EPI_GELU_BWD, flags=fl, aux=aux[:, :N])
    if name.startswith("gelu"):
        fl = (ll.FLAG_GELU_TANH if "tanh" in name else 0) | (ll.FLAG_GELU_SAVE_GRAD if "save" in name else 0)
        return dict(epi=ll.EPI_BIAS_GELU, flags=fl, bias=bias, want_out1=True)
    if name.startswith("resid"):
        aux = torch.full((M, N + 16), float("nan"), device="cuda", dtype=f32)
        aux[:, :N] = torch.randn((M, N), device="cuda")
        kw = dict(epi=ll.EPI_RESID, bias=bias, aux=aux[:, :N])
        if "gamma" in name:
            kw["gamma"] = gamma
        if "rowscale" in name:
            kw["rowscale"] = rs
        if "out1" in name:
            kw["want_out1"] = True
        return kw
    if name == "accum_bf16":
        return dict(flags=ll.FLAG_ACCUM, init0=_mk((M, N), seed + 13))
    if name == "accum_f32":
        return dict(epi=ll.EPI_F32, flags=ll.FLAG_ACCUM, init0=torch.randn((M, N), device="cuda"))
    raise ValueError(name)


@pytest.mark.parametrize("layout", ["nt", "dgrad", "wgrad"])
@pytest.mark.parametrize("epilogue", EPILOGUES)
def test_pingpong_epilogues_bitwise(cuda_lib, layout, epilogue):
    ll = cuda_lib
    M, N, K = 417, 1000, 592          # ragged in M, N (8 tiles of 128, the last 104 wide) and K (9.25 k-blocks)
    a, b, a_t, b_t = _operands(layout, M, N, K, 100)
    _check_pair(ll, a, b, a_t, b_t, M, N, **_epilogue_args(ll, epilogue, M, N, 200))


# ---------------------------------------------------------------- tile counts per CTA and ragged shapes
# 132 SMs: 1 tile; 3 tiles (odd, fewer than SMs: warpgroup 1 of most CTAs has nothing); 4 tiles; 136 tiles (some
# CTAs 2, some 1); 17 x 8 = 136; the step's shapes at 105 x 11 = 1155 tiles (8 or 9 per CTA) and wider.
SHAPES = [
    (128, 128, 64), (384, 128, 128), (256, 256, 64), (200, 200, 1000), (417, 1408, 1408), (2049, 1024, 1024),
    (1000, 6144, 592), (13344, 1408, 1408), (834, 3200, 1408), (417, 1408, 6144), (130, 768, 200),
]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("layout", ["nt", "dgrad", "wgrad"])
def test_pingpong_shapes_bitwise(cuda_lib, M, N, K, layout):
    ll = cuda_lib
    a, b, a_t, b_t = _operands(layout, M, N, K, 300)
    out = _check_pair(ll, a, b, a_t, b_t, M, N, epi=ll.EPI_F32)[0][:, :N]
    # and against fp32 torch on a few rows (same tolerance as the cooperative kernel's tests)
    idx = torch.tensor(sorted({0, M // 2, M - 1}), device="cuda")
    af = (a.t() if a_t else a).float()[idx]
    bf_ = (b if b_t else b.t()).float()
    ref = af @ bf_
    rel = ((out[idx] - ref).norm() / ref.norm()).item()
    assert rel < 1e-4, rel


def test_pingpong_repeat_bitwise(cuda_lib):
    ll = cuda_lib
    M, N, K = 13344, 6144, 1408
    a, b = _mk((M, K), 400), _mk((N, K), 401, 0.03)
    bias = _mk((N,), 402, 0.1)
    fl = ll.FLAG_GELU_TANH | ll.FLAG_GELU_SAVE_GRAD | ll.FLAG_PINGPONG
    outs = []
    for _ in range(2):
        h = torch.empty((M, N), device="cuda", dtype=bf)
        g = ll.gemm(a, b, epi=ll.EPI_BIAS_GELU, flags=fl, bias=bias, out1=h)
        outs.append((g, h))
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0][0]), _bits(outs[1][0])) and torch.equal(_bits(outs[0][1]), _bits(outs[1][1]))


def test_pingpong_full_size_fp32(cuda_lib):
    """A full-size cfg-2 GEMM (fc1 forward, 1155 tiles) against fp32 on spot rows, and the default selection."""
    ll = cuda_lib
    M, N, K = 13344, 6144, 1408
    a = _mk((M, K), 20); w = _mk((N, K), 21, 0.03)
    out = ll.gemm(a, w, epi=ll.EPI_F32, flags=ll.FLAG_PINGPONG)
    idx = torch.tensor([0, 1, 63, 64, 127, 128, 5000, 13343], device="cuda")
    ref = a[idx].float() @ w.float().t()
    assert ((out[idx] - ref).norm() / ref.norm()).item() < 1e-4
    assert torch.equal(ll.gemm(a, w, epi=ll.EPI_F32), out)   # the step's own selection runs the same kernel


def test_pingpong_flag_refusals(cuda_lib):
    ll = cuda_lib
    a = _mk((128, 64), 1)
    with pytest.raises(ll._lib.IvbError):
        ll.gemm(a, a, flags=ll.FLAG_PINGPONG, tile_n=176)
    with pytest.raises(ll._lib.IvbError):
        ll.gemm(a, a, flags=ll.FLAG_PINGPONG | ll.FLAG_1CTA)
    with pytest.raises(ll._lib.IvbError):
        ll.gemm(a, a, flags=ll.FLAG_PINGPONG | ll.FLAG_2CTA)
