"""wgmma GEMM vs torch fp32 matmul on the same bf16-rounded operands (gpu)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


SHAPES = [
    (128, 256, 64), (128, 128, 128), (200, 384, 384), (412, 1152, 384), (417, 1408, 1408),
    (1000, 4224, 1408), (834, 1408, 6144), (130, 6144, 1408), (64, 768, 592), (2049, 1024, 1024),
]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("tile_n", [0, 128, 176, 192, 256])
def test_gemm_nt(cuda_lib, M, N, K, tile_n):
    ll = cuda_lib
    a = _mk((M, K), 1); b = _mk((N, K), 2, 0.05)
    ref = a.float() @ b.float().t()
    out = ll.gemm(a, b, tile_n=tile_n)
    torch.cuda.synchronize()
    assert _rel(out, ref) < 6e-3, (M, N, K, tile_n, _rel(out, ref))
    out32 = ll.gemm(a, b, epi=ll.EPI_F32, tile_n=tile_n)
    assert _rel(out32, ref) < 1e-4


@pytest.mark.parametrize("M,N,K", [(417, 1408, 4224), (300, 384, 1152), (1000, 6144, 1408), (128, 192, 64)])
@pytest.mark.parametrize("tile_n", [0, 128, 176, 256])
def test_gemm_dgrad_layout(cuda_lib, M, N, K, tile_n):
    """dx[M,N] = dy[M,K] @ W[K,N]  (B operand MN-major, read straight from the row-major weight)."""
    ll = cuda_lib
    dy = _mk((M, K), 3); w = _mk((K, N), 4, 0.05)
    ref = dy.float() @ w.float()
    out = ll.gemm(dy, w, b_t=True, epi=ll.EPI_F32, tile_n=tile_n)
    assert _rel(out, ref) < 1e-4, _rel(out, ref)


@pytest.mark.parametrize("M,N,K", [(1408, 1408, 417), (384, 1152, 824), (6144, 1408, 1000), (128, 128, 64), (592, 768, 200)])
@pytest.mark.parametrize("tile_n", [0, 128, 176, 256])
def test_gemm_wgrad_layout(cuda_lib, M, N, K, tile_n):
    """dW[M,N] = dy[K,M]^T @ x[K,N]  (both operands MN-major)."""
    ll = cuda_lib
    dy = _mk((K, M), 5); x = _mk((K, N), 6)
    ref = dy.float().t() @ x.float()
    out = ll.gemm(dy, x, a_t=True, b_t=True, epi=ll.EPI_F32, tile_n=tile_n)
    assert _rel(out, ref) < 1e-4, _rel(out, ref)
    acc = torch.ones_like(out)
    ll.gemm(dy, x, a_t=True, b_t=True, epi=ll.EPI_F32, flags=ll.FLAG_ACCUM, out0=acc, tile_n=tile_n)
    assert _rel(acc, ref + 1) < 1e-4


def test_gemm_epilogues(cuda_lib):
    ll = cuda_lib
    M, N, K = 417, 1536, 384
    a = _mk((M, K), 7); w = _mk((N, K), 8, 0.05); bias = _mk((N,), 9, 0.1)
    h_ref = a.float() @ w.float().t() + bias.float()
    for flags, fn in ((0, lambda t: torch.nn.functional.gelu(t)),
                      (ll.FLAG_GELU_TANH, lambda t: torch.nn.functional.gelu(t, approximate="tanh"))):
        h = torch.empty((M, N), device="cuda", dtype=torch.bfloat16)
        g = ll.gemm(a, w, epi=ll.EPI_BIAS_GELU, flags=flags, bias=bias, out1=h)
        assert _rel(h, h_ref) < 6e-3
        assert _rel(g, fn(h_ref)) < 6e-3
        # gelu backward epilogue: out = acc * gelu'(h)
        dy = _mk((M, K), 10)  # pretend upstream grad of shape [M,K]; contraction over K again
        w2 = _mk((N, K), 11, 0.05)
        acc_ref = dy.float() @ w2.float().t()
        hh = h.float().requires_grad_(True)
        fn(hh).backward(torch.ones_like(hh))
        dh = ll.gemm(dy, w2, epi=ll.EPI_GELU_BWD, flags=flags, aux=h)
        assert _rel(dh, acc_ref * hh.grad) < 8e-3
        # training form: the forward saves gelu'(h), the backward epilogue is a plain multiply
        fl = flags | ll.FLAG_GELU_SAVE_GRAD
        dsave = torch.empty((M, N), device="cuda", dtype=torch.bfloat16)
        g2 = ll.gemm(a, w, epi=ll.EPI_BIAS_GELU, flags=fl, bias=bias, out1=dsave)
        assert torch.equal(g2, g)
        h32 = h_ref.clone().requires_grad_(True)
        fn(h32).backward(torch.ones_like(h32))
        assert _rel(dsave, h32.grad) < 6e-3
        dh2 = ll.gemm(dy, w2, epi=ll.EPI_GELU_BWD, flags=fl, aux=dsave)
        assert _rel(dh2, acc_ref * h32.grad) < 8e-3
    # residual epilogue
    N2 = 384
    w3 = _mk((N2, K), 12, 0.05); b3 = _mk((N2,), 13, 0.1); gamma = _mk((N2,), 14, 0.5)
    resid = torch.randn((M, N2), device="cuda")
    y = torch.empty((M, N2), device="cuda", dtype=torch.bfloat16)
    out = ll.gemm(a, w3, epi=ll.EPI_RESID, bias=b3, gamma=gamma, aux=resid, out1=y)
    y_ref = a.float() @ w3.float().t() + b3.float()
    assert _rel(y, y_ref) < 6e-3
    assert _rel(out, resid + gamma.float() * y_ref) < 1e-4
    out2 = ll.gemm(a, w3, epi=ll.EPI_RESID, bias=b3, gamma=None, aux=resid)
    assert _rel(out2, resid + y_ref) < 1e-4


def test_gemm_large_full_size(cuda_lib):
    """cfg-2 sized GEMMs: linearity property at full size + spot-check rows against fp32."""
    ll = cuda_lib
    M, N, K = 13344, 6144, 1408
    a = _mk((M, K), 20); w = _mk((N, K), 21, 0.03)
    out = ll.gemm(a, w, epi=ll.EPI_F32)
    idx = torch.tensor([0, 1, 127, 128, 5000, 13343], device="cuda")
    ref = a[idx].float() @ w.float().t()
    assert _rel(out[idx], ref) < 1e-4
    # linearity: (2a) W^T == 2 (a W^T) exactly in fp32 (power-of-two scaling)
    out2 = ll.gemm((a.float() * 2).to(torch.bfloat16), w, epi=ll.EPI_F32)
    assert torch.equal(out2, out * 2)


# ---------------------------------------------------------------- CTA-pair (cluster of 2, multicast B) kernel
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 1408, 1408), (1000, 4224, 1408), (417, 6144, 1408),
                                   (834, 1408, 6144), (130, 768, 592), (2049, 1024, 1024)])
@pytest.mark.parametrize("tile_n", [0, 128, 176, 192, 256])
def test_gemm2_nt(cuda_lib, M, N, K, tile_n):
    ll = cuda_lib
    a = _mk((M, K), 31); b = _mk((N, K), 32, 0.05)
    ref = a.float() @ b.float().t()
    out32 = ll.gemm(a, b, epi=ll.EPI_F32, flags=ll.FLAG_2CTA, tile_n=tile_n)
    torch.cuda.synchronize()
    assert _rel(out32, ref) < 1e-4, (M, N, K, tile_n, _rel(out32, ref))


@pytest.mark.parametrize("M,N,K", [(417, 1408, 4224), (300, 384, 1152), (1000, 6144, 1408), (256, 256, 64)])
@pytest.mark.parametrize("tile_n", [0, 128, 256])
def test_gemm2_dgrad_layout(cuda_lib, M, N, K, tile_n):
    ll = cuda_lib
    dy = _mk((M, K), 33); w = _mk((K, N), 34, 0.05)
    out = ll.gemm(dy, w, b_t=True, epi=ll.EPI_F32, flags=ll.FLAG_2CTA, tile_n=tile_n)
    assert _rel(out, dy.float() @ w.float()) < 1e-4


@pytest.mark.parametrize("M,N,K", [(1408, 1408, 417), (384, 1152, 824), (6144, 1408, 1000), (256, 128, 64), (592, 768, 200)])
@pytest.mark.parametrize("tile_n", [0, 128, 256])
def test_gemm2_wgrad_layout(cuda_lib, M, N, K, tile_n):
    ll = cuda_lib
    dy = _mk((K, M), 35); x = _mk((K, N), 36)
    out = ll.gemm(dy, x, a_t=True, b_t=True, epi=ll.EPI_F32, flags=ll.FLAG_2CTA, tile_n=tile_n)
    assert _rel(out, dy.float().t() @ x.float()) < 1e-4


def test_gemm2_epilogue_resid(cuda_lib):
    ll = cuda_lib
    M, N, K = 1000, 1408, 384
    a = _mk((M, K), 37); w = _mk((N, K), 38, 0.05); b = _mk((N,), 39, 0.1); gamma = _mk((N,), 40, 0.5)
    resid = torch.randn((M, N), device="cuda")
    rs = (torch.rand(M, device="cuda") > 0.25).float() / 0.75
    y = torch.empty((M, N), device="cuda", dtype=torch.bfloat16)
    out = ll.gemm(a, w, epi=ll.EPI_RESID, bias=b, gamma=gamma, aux=resid, out1=y, rowscale=rs, flags=ll.FLAG_2CTA)
    y_ref = a.float() @ w.float().t() + b.float()
    assert _rel(y, y_ref) < 6e-3
    assert _rel(out, resid + rs[:, None] * gamma.float() * y_ref) < 1e-4
    out1 = ll.gemm(a, w, epi=ll.EPI_RESID, bias=b, gamma=gamma, aux=resid, rowscale=rs, flags=ll.FLAG_1CTA)
    assert _rel(out1, out) < 1e-6
