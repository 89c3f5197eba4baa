"""Per-token FP8 training of the ViT blocks (modules.set_fp8(model, scaling="token")) on the H100 (gpu).

- ivb_norm_fwd_fp8_train: bf16 row, mean and rstd bit-identical to ivb_norm_fwd; E4M3 rows and scales bit-identical
  to ivb_norm_fwd_fp8; padding of every output keeps its bits.
- ivb_fp8_quantize_cols_t: element by element against a float64 restatement of the scale rule, with tails in both
  dimensions, a zero column, an Inf column and a NaN column; the same bits on two runs.
- Row independence of the input-gradient GEMM: scaling one gradient row by a power of two leaves every other row of dx
  bit-identical.
The block and the model in this mode: test_fp8_modes_gpu.py.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, e4m3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
NAN8 = 0x7f    # an E4M3 NaN byte


def _pad16(n):
    return (n + 15) // 16 * 16


# ------------------------------------------------------------------------------------------------ kernel (a)
@pytest.mark.parametrize("layernorm", [False, True], ids=["rms", "ln"])
@pytest.mark.parametrize("x_f32", [True, False], ids=["xf32", "xbf16"])
@pytest.mark.parametrize("D", [8, 384, 1408, 1544, 4096])
def test_norm_fwd_fp8_train_bits(cuda_lib, layernorm, x_f32, D):
    ll = cuda_lib
    M = 333
    g = torch.Generator(device="cuda").manual_seed(D + 7 * layernorm + 3 * x_f32)
    xb = torch.randn((M, D + 24), device="cuda", generator=g) * 3 + 0.5
    x = (xb if x_f32 else xb.to(bf16))[:, :D]                     # padded pitch ldx = D + 24
    w = (1 + 0.2 * torch.randn(D, device="cuda", generator=g)).to(bf16)
    b = (0.1 * torch.randn(D, device="cuda", generator=g)).to(bf16) if layernorm else None
    eps = 1e-5 if layernorm else 1e-6
    ldy, ldo = D + 8, _pad16(D) + 16
    y = torch.full((M, ldy), float("nan"), device="cuda", dtype=bf16)
    q = torch.full((M, ldo), NAN8, device="cuda", dtype=torch.uint8)
    stats = torch.full((3, M + 1), float("nan"), device="cuda", dtype=f32)   # sinv, mean, rstd; one guard element each
    ll._call("norm_fwd_fp8_train", x, int(x_f32), x.stride(0), w, b, eps, int(layernorm), M, D, q, ldo, stats[0], y,
             ldy, stats[1], stats[2])
    y_ref, mean_ref, rstd_ref = ll.norm_fwd(x, w, b, eps=eps, layernorm=layernorm)
    q_ref, s_ref = ll.norm_fwd_fp8(x, w, b, eps=eps, layernorm=layernorm)
    torch.cuda.synchronize()
    assert torch.equal(y[:, :D].view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(stats[2, :M].view(torch.int32), rstd_ref.view(torch.int32))
    if layernorm:
        assert torch.equal(stats[1, :M].view(torch.int32), mean_ref.view(torch.int32))
    else:
        assert torch.isnan(stats[1]).all()                       # RMSNorm writes no mean
    assert torch.equal(q[:, :D], q_ref.view(torch.uint8))
    assert torch.equal(stats[0, :M].view(torch.int32), s_ref.view(torch.int32))
    assert torch.isnan(y[:, D:].float()).all() and (q[:, D:] == NAN8).all() and torch.isnan(stats[:, M]).all()
    # the lowlevel form returns the same bits
    q2, s2, y2, mean2, rstd2 = ll.norm_fwd_fp8(x, w, b, eps=eps, layernorm=layernorm, save=True)
    assert torch.equal(q2.view(torch.uint8), q[:, :D]) and torch.equal(y2.view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(rstd2, rstd_ref) and (mean2 is None) == (not layernorm)


# ------------------------------------------------------------------------------------------------ kernel (b)
def _cols_reference(w):
    """float64 restatement: per column k, scale 2^e with e the largest integer such that amax_k * 2^e <= 448 (e in
    [-126, 126]; 1 for a zero column), q_t[k] = RNE_e4m3(w[:, k] * scale), scale_inv NaN for a non-finite column."""
    w64 = w.double()
    amax = w64.abs().amax(0)
    e = torch.floor(torch.log2(448.0 / amax.clamp_min(1e-300)))
    e = torch.where(amax * torch.exp2(e + 1) <= 448.0, e + 1, e)
    e = torch.where(amax * torch.exp2(e) > 448.0, e - 1, e)
    e = torch.where(amax == 0, torch.zeros_like(e), e.clamp(-126, 126))
    finite = torch.isfinite(amax)
    e = torch.where(finite, e, torch.zeros_like(e))
    scale = torch.exp2(e)
    q_t = (w64 * scale).float().t().contiguous().to(e4m3)
    sinv = torch.where(finite, 1.0 / scale, torch.full_like(scale, float("nan")))
    return q_t, sinv, amax


@pytest.mark.parametrize("N,K", [(197, 133), (64, 64), (6144, 1408), (1408, 6144), (77, 4224)])
def test_quantize_cols_t_against_float64(cuda_lib, N, K):
    ll = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(N * 31 + K)
    ldx = (K + 7) // 8 * 8 + 8
    wb = (torch.randn((N, ldx), device="cuda", generator=g) * 0.02)
    wb[:, : K // 2] *= torch.exp2(torch.randint(-20, 20, (K // 2,), device="cuda", generator=g).float())
    wb = wb.to(bf16)
    w = wb[:, :K]
    w[:, 5] = 0                                       # a zero column
    w[N // 2, 7] = float("inf")                       # an Inf column
    w[N // 3, 7] = -float("inf")
    w[1, 9] = float("nan")                            # a NaN column
    ldt = _pad16(N) + 16
    runs = []
    for _ in range(2):
        q_t = torch.full((K, ldt), NAN8, device="cuda", dtype=torch.uint8)
        amax = torch.full((K + 1,), float("nan"), device="cuda", dtype=f32)
        sinv = torch.full((K + 1,), float("nan"), device="cuda", dtype=f32)
        ll._call("fp8_quantize_cols_t", w, ldx, N, K, q_t, ldt, amax, sinv)
        runs.append((q_t, amax, sinv))
    torch.cuda.synchronize()
    (q_t, amax, sinv), (q_t2, amax2, sinv2) = runs
    assert torch.equal(q_t, q_t2) and torch.equal(sinv.view(torch.int32), sinv2.view(torch.int32))
    q_ref, s_ref, a_ref = _cols_reference(w)
    fin = torch.isfinite(a_ref)
    assert not bool(fin[7]) and bool(torch.isnan(sinv[7]))
    assert torch.equal(sinv[:K][fin].double(), s_ref[fin])
    assert torch.equal(amax[:K].double()[fin], a_ref[fin]) and float(sinv[5]) == 1.0
    assert torch.equal(q_t[:, :N][fin], q_ref.view(torch.uint8)[fin])
    assert (q_t[:, N:] == NAN8).all() and torch.isnan(amax[K]) and torch.isnan(sinv[K])
    # the non-finite columns: scale 1 and a satfinite cast, so an Inf becomes +-448 and a NaN stays NaN
    for k in (7, 9):
        col, nan = w[:, k].float(), torch.isnan(w[:, k].float())
        assert torch.equal(q_t[k, :N][~nan], col.clamp(-448, 448).to(e4m3).view(torch.uint8)[~nan])
        assert bool(((q_t[k, :N][nan] & 0x7f) == 0x7f).all()) and bool(torch.isnan(sinv[k]))
    # the lowlevel form: the rows of w^T, the same bits as the per-row cast of w^T
    qt3, s3 = ll.fp8_quantize_rows(w, transposed=True)
    assert torch.equal(qt3.view(torch.uint8), q_t[:, :N])
    wt = torch.zeros((K, (N + 7) // 8 * 8), device="cuda", dtype=bf16)   # the row cast wants a pitch of 8 elements
    wt[:, :N] = w.t()
    q_rows, s_rows = ll.fp8_quantize_rows(wt[:, :N])
    assert torch.equal(q_rows.view(torch.uint8)[fin], q_t[:, :N][fin]) and torch.equal(s_rows[fin], sinv[:K][fin])


# ------------------------------------------------------------------------------------------------ row independence
def test_dgrad_rows_are_independent(cuda_lib):
    ll = cuda_lib
    M, N, K = 777, 1408, 640
    g = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn((M, N), device="cuda", generator=g).to(bf16)
    w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(bf16)
    w_t, ws = ll.fp8_quantize_rows(w, transposed=True)

    def dgrad(d):
        q, s = ll.fp8_quantize_rows(d)
        return ll.gemm_fp8(q, s, w_t, ws, epi=ll.EPI_F32)
    dx = dgrad(dy)
    dy2 = dy.clone()
    r = 300
    dy2[r] *= 2.0 ** 12
    dx2 = dgrad(dy2)
    others = torch.arange(M, device="cuda") != r
    assert torch.equal(dx2[others], dx[others])
    assert torch.equal(dx2[r], dx[r] * 2.0 ** 12)
