"""Row-kernel properties the element-wise checks of test_rows_gpu.py do not cover: the same bits on every run, and a
raised shared-memory limit on every device (gpu)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def _equal_twice(run):
    """run() zeroes fresh gradient buffers, calls the library and returns them: two calls must agree bit for bit."""
    first, second = run(), run()
    for a, b in zip(first, second):
        assert torch.equal(a, b)


@pytest.mark.parametrize("case", ["rms 1408", "rms 3200", "ln 1408", "ln 3200", "pair", "fused layerscale",
                                  "layerscale", "colsum", "ln_l2 reg", "ln_l2 stream"])
def test_parameter_gradients_are_deterministic(cuda_lib, case):
    """include/ivb200.h promises the same bits on every run: every entry point that writes parameter gradients sums
    them in a fixed order, on the register-resident and the streaming kernels."""
    ll = cuda_lib
    torch.manual_seed(4)
    M = 13344
    zeros = lambda n: torch.zeros(n, device="cuda")
    if case.startswith(("rms", "ln ")):
        D = int(case.split()[1]); ln = case.startswith("ln")
        x = torch.randn(M, D, device="cuda"); w = (torch.rand(D, device="cuda") + 0.5).to(torch.bfloat16)
        b = torch.zeros(D, device="cuda", dtype=torch.bfloat16) if ln else None
        _, mean, rstd = ll.norm_fwd(x, w, b, layernorm=ln)
        dy = torch.randn(M, D, device="cuda").to(torch.bfloat16)

        def run():
            dw, db = zeros(D), (zeros(D) if ln else None)
            ll.norm_bwd(dy, x, w, mean, rstd, layernorm=ln, dweight=dw, dbias=db)
            return [dw, db] if ln else [dw]
    elif case == "pair":
        D = 1408
        qkv = torch.randn(M, 3 * D, device="cuda").to(torch.bfloat16)
        wq, wk = ((torch.rand(D, device="cuda") + 0.5).to(torch.bfloat16) for _ in range(2))
        rstd = ll.rmsnorm_pair_fwd(qkv, D, wq, wk, torch.empty(M, 2 * D, device="cuda", dtype=torch.bfloat16))
        dqkv = torch.randn(M, 3 * D, device="cuda").to(torch.bfloat16)

        def run():
            dwq, dwk = zeros(D), zeros(D)
            ll.rmsnorm_pair_bwd(dqkv.clone(), qkv, D, wq, wk, rstd, dwq, dwk)
            return [dwq, dwk]
    elif case in ("fused layerscale", "layerscale", "colsum"):
        D = 1408
        x = torch.randn(M, D, device="cuda"); w = (torch.rand(D, device="cuda") + 0.5).to(torch.bfloat16)
        _, _, rstd = ll.norm_fwd(x, w)
        dy, ybr = (torch.randn(M, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        dx_in = torch.randn(M, D, device="cuda")
        gamma = (torch.randn(D, device="cuda") * 0.1).to(torch.bfloat16)
        rs = (torch.rand(M, device="cuda") < 0.7).float() / 0.7

        def run():
            g = [zeros(D), zeros(D), zeros(D)]
            if case == "fused layerscale":
                ll.rmsnorm_bwd_layerscale(dy, x, w, rstd, dx_in, ybr, gamma, *g, rowscale=rs)
            elif case == "layerscale":
                ll.layerscale_bwd(dx_in, ybr, gamma, g[0], g[1], rowscale=rs)
            else:
                ll.colsum(ybr, out=g[0])
            return g
    else:
        C = 3200
        z = torch.randn(M, C, device="cuda").to(torch.bfloat16)
        w = (torch.rand(C, device="cuda") + 0.5).to(torch.bfloat16); b = (torch.randn(C, device="cuda") * 0.1).to(torch.bfloat16)
        tgt = torch.randn(M, C, device="cuda").to(torch.bfloat16 if case.endswith("reg") else torch.float32)
        _, stats = ll.ln_l2_fwd(z, w, b, want_out=False)

        def run():
            dw, db = zeros(C), zeros(C)
            ll.ln_l2_bwd(z, w, b, stats, tgt, -2.0 / M, None, dw, db)
            return [dw, db]
    _equal_twice(run)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_layernorm_bwd_on_every_device(cuda_lib):
    """The LayerNorm backward at D = 1408 with weight and bias gradients needs 88 KB of shared memory, a limit that is
    raised per device: it must run on the second GPU of a process as well as on the first."""
    ll = cuda_lib
    M, D = 417, 1408
    for dev in (0, 1):
        with torch.cuda.device(dev):
            torch.manual_seed(5)
            x = torch.randn(M, D, device="cuda")
            w = (torch.randn(D, device="cuda") * 0.2 + 1).to(torch.bfloat16)
            b = (torch.randn(D, device="cuda") * 0.1).to(torch.bfloat16)
            xr = x.clone().requires_grad_(True); wr = w.float().requires_grad_(True); br = b.float().requires_grad_(True)
            yr = torch.nn.functional.layer_norm(xr, (D,), wr, br, 1e-5)
            _, mean, rstd = ll.norm_fwd(x, w, b, eps=1e-5, layernorm=True)
            dy = torch.randn(M, D, device="cuda").to(torch.bfloat16)
            yr.backward(dy.float())
            dw = torch.zeros(D, device="cuda"); db = torch.zeros(D, device="cuda")
            dx = ll.norm_bwd(dy, x, w, mean, rstd, layernorm=True, dweight=dw, dbias=db)
            torch.cuda.synchronize()
            assert _rel(dx, xr.grad) < 1e-4 and _rel(dw, wr.grad) < 1e-4 and _rel(db, br.grad) < 1e-4
