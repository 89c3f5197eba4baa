"""RMSNorm / LayerNorm / LayerScale-backward / colsum kernels vs torch fp32 (gpu)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


@pytest.mark.parametrize("M,D", [(1, 384), (417, 1408), (1000, 3200), (33, 768), (2049, 1024)])
@pytest.mark.parametrize("xf32", [True, False])
@pytest.mark.parametrize("ln", [False, True])
def test_norm_fwd_bwd(cuda_lib, M, D, xf32, ln):
    ll = cuda_lib
    torch.manual_seed(0)
    x = torch.randn(M, D, device="cuda") * 2 + 0.3
    if not xf32:
        x = x.to(torch.bfloat16)
    w = (torch.randn(D, device="cuda") * 0.2 + 1).to(torch.bfloat16)
    b = (torch.randn(D, device="cuda") * 0.1).to(torch.bfloat16) if ln else None
    eps = 1e-5 if ln else 1e-6
    xr = x.float().requires_grad_(True)
    wr = w.float().requires_grad_(True)
    br = b.float().requires_grad_(True) if ln else None
    if ln:
        yr = torch.nn.functional.layer_norm(xr, (D,), wr, br, eps)
    else:
        yr = wr * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + eps))
    y, mean, rstd = ll.norm_fwd(x, w, b, eps=eps, layernorm=ln)
    assert _rel(y, yr) < 5e-3
    dy = torch.randn(M, D, device="cuda").to(torch.bfloat16)
    yr.backward(dy.float())
    dw = torch.zeros(D, device="cuda"); db = torch.zeros(D, device="cuda") if ln else None
    dx_in = torch.randn(M, D, device="cuda")
    dx = ll.norm_bwd(dy, x, w, mean, rstd, layernorm=ln, dx_in=dx_in, dweight=dw, dbias=db)
    assert _rel(dx - dx_in, xr.grad) < 1e-4
    assert _rel(dw, wr.grad) < 1e-4
    if ln:
        assert _rel(db, br.grad) < 1e-4
    # bf16 in-place variant (as used for the q/k-norm backward)
    dyc = dy.clone()
    ll.norm_bwd(dyc, x, w, mean, rstd, layernorm=ln, dx_out=dyc)
    assert _rel(dyc, xr.grad) < 6e-3


def test_norm_strided_qk(cuda_lib):
    ll = cuda_lib
    M, D = 417, 1408
    qkv = torch.randn(M, 3 * D, device="cuda").to(torch.bfloat16)
    wq = (torch.rand(D, device="cuda") + 0.5).to(torch.bfloat16)
    out = torch.empty(M, 2 * D, device="cuda", dtype=torch.bfloat16)
    y, _, rstd = ll.norm_fwd(qkv[:, D:2 * D], wq, out=out[:, D:])
    k = qkv[:, D:2 * D].float()
    ref = wq.float() * k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + 1e-6)
    assert _rel(out[:, D:], ref) < 5e-3


def test_layerscale_bwd_and_colsum(cuda_lib):
    ll = cuda_lib
    M, D = 1000, 1408
    dx = torch.randn(M, D, device="cuda")
    y = torch.randn(M, D, device="cuda").to(torch.bfloat16)
    gamma = (torch.randn(D, device="cuda") * 0.1).to(torch.bfloat16)
    dg = torch.zeros(D, device="cuda"); dc = torch.zeros(D, device="cuda")
    dy = ll.layerscale_bwd(dx, y, gamma, dg, dc)
    assert _rel(dy, dx * gamma.float()) < 5e-3
    assert _rel(dg, (dx * y.float()).sum(0)) < 1e-4
    assert _rel(dc, dx.sum(0) * gamma.float()) < 1e-4     # bias gradient: gamma * column sums
    dc.zero_()
    dy2 = ll.layerscale_bwd(dx, None, None, None, dc)
    assert _rel(dy2, dx) < 5e-3
    cs = ll.colsum(y)
    assert _rel(cs, y.float().sum(0)) < 1e-4


@pytest.mark.parametrize("M,D", [(417, 1408), (13344, 1408), (33, 384), (1025, 1024)])
def test_rmsnorm_pair_matches_separate_calls(cuda_lib, M, D):
    """q-norm + k-norm in ONE launch (forward, and the in-place backward with both weight gradients) against fp32
    torch RMSNorm of the two column slices of the [M, 3D] projection buffer (internvideo2_pretrain.py:198-206)."""
    ll = cuda_lib
    torch.manual_seed(1)
    qkv = torch.randn(M, 3 * D, device="cuda").to(torch.bfloat16)
    wq = (torch.rand(D, device="cuda") + 0.5).to(torch.bfloat16)
    wk = (torch.rand(D, device="cuda") + 0.5).to(torch.bfloat16)
    out = torch.empty(M, 2 * D, device="cuda", dtype=torch.bfloat16)
    rstd = ll.rmsnorm_pair_fwd(qkv, D, wq, wk, out)
    assert rstd.shape == (M, 2)
    refs, leaves = [], []
    for part, w in ((0, wq), (1, wk)):
        x = qkv[:, part * D:(part + 1) * D].float().requires_grad_(True)
        wr = w.float().requires_grad_(True)
        r = wr * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6))
        refs.append(r); leaves.append((x, wr))
        assert _rel(out[:, part * D:(part + 1) * D], r) < 5e-3
    dqkv = torch.randn(M, 3 * D, device="cuda").to(torch.bfloat16)
    dv_before = dqkv[:, 2 * D:].clone()
    for part in (0, 1):
        refs[part].backward(dqkv[:, part * D:(part + 1) * D].float())
    dwq = torch.zeros(D, device="cuda"); dwk = torch.zeros(D, device="cuda")
    ll.rmsnorm_pair_bwd(dqkv, qkv, D, wq, wk, rstd, dwq, dwk)
    for part, dw in ((0, dwq), (1, dwk)):
        assert _rel(dqkv[:, part * D:(part + 1) * D], leaves[part][0].grad) < 6e-3
        assert _rel(dw, leaves[part][1].grad) < 2e-4
    assert torch.equal(dqkv[:, 2 * D:], dv_before)            # the v slot of the gradient buffer is untouched


@pytest.mark.parametrize("M,C", [(834, 3200), (417, 1408), (32, 768), (100, 3208), (64, 3456)])
def test_ln_l2_register_resident_paths(cuda_lib, M, C):
    """Decoder tail LN -> L2 -> (2-2cos) loss, forward and backward, on the register-resident kernels (bf16 target,
    C <= 3328) and on the streaming fallback (fp32 target, or C > 3328) against fp32 torch."""
    ll = cuda_lib
    torch.manual_seed(2)
    z = (torch.randn(M, C, device="cuda") * 1.5 + 0.2).to(torch.bfloat16)
    w = (torch.randn(C, device="cuda") * 0.2 + 1).to(torch.bfloat16)
    b = (torch.randn(C, device="cuda") * 0.1).to(torch.bfloat16)
    tgt = torch.nn.functional.normalize(torch.randn(M, C, device="cuda"), dim=-1)
    zr = z.float().requires_grad_(True); wr = w.float().requires_grad_(True); br = b.float().requires_grad_(True)
    y = torch.nn.functional.layer_norm(zr, (C,), wr, br, 1e-5)
    o = y / y.norm(dim=-1, keepdim=True)
    for tdt in (torch.bfloat16, torch.float32):
        t = tgt.to(tdt)
        loss_ref = (2 - 2 * (o * t.float()).sum(-1)).sum()
        ls = torch.zeros(1, device="cuda")
        out, stats = ll.ln_l2_fwd(z, w, b, 1e-5, want_out=True, target=t, loss_sum=ls)
        assert _rel(out, o) < 5e-3
        assert abs(float(ls) - float(loss_ref)) < 2e-3 * abs(float(loss_ref))
        for p_ in (zr, wr, br):
            p_.grad = None
        (loss_ref / M).backward(retain_graph=True)
        dw = torch.zeros(C, device="cuda"); db = torch.zeros(C, device="cuda")
        gd = torch.ones(1, device="cuda")
        dz = ll.ln_l2_bwd(z, w, b, stats, t, -2.0 / M, gd, dw, db)
        assert _rel(dz, zr.grad) < 1e-2
        assert _rel(dw, wr.grad) < 2e-3 and _rel(db, br.grad) < 2e-3


@pytest.mark.parametrize("M,D", [(13344, 1408), (1025, 1024), (2049, 384), (4100, 1536)])
def test_rms_tma_row_pipeline_and_fused_layerscale(cuda_lib, M, D):
    """fp32 stream, M >= 1024: RMSNorm forward and backward (+ residual gradient in) on the register-resident kernels,
    and the backward fused with the LayerScale backward on the bulk-copy row ring (rowscale = DropPath factors incl.
    dropped rows; with and without the residual gradient in and the rowscale) vs fp32 torch."""
    ll = cuda_lib
    torch.manual_seed(3)
    x = torch.randn(M, D, device="cuda") * 2 + 0.3
    w = (torch.randn(D, device="cuda") * 0.2 + 1).to(torch.bfloat16)
    xr = x.clone().requires_grad_(True); wr = w.float().requires_grad_(True)
    yr = wr * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-6))
    y, _, rstd = ll.norm_fwd(x, w)
    assert _rel(y, yr) < 5e-3
    assert _rel(rstd, torch.rsqrt(x.pow(2).mean(-1) + 1e-6)) < 1e-5
    dy = torch.randn(M, D, device="cuda").to(torch.bfloat16)
    dx_in = torch.randn(M, D, device="cuda")
    yr.backward(dy.float())
    dw = torch.zeros(D, device="cuda")
    dx = ll.norm_bwd(dy, x, w, None, rstd, dx_in=dx_in, dweight=dw)
    assert _rel(dx - dx_in, xr.grad) < 1e-4 and _rel(dw, wr.grad) < 2e-4
    # fused: + LayerScale backward of the branch feeding the stream
    ybr = torch.randn(M, D, device="cuda").to(torch.bfloat16)
    gamma = (torch.randn(D, device="cuda") * 0.1).to(torch.bfloat16)
    rs = (torch.rand(M, device="cuda") < 0.7).float() / 0.7
    for fin, frs in ((dx_in, rs), (None, rs), (dx_in, None)):
        dw2 = torch.zeros(D, device="cuda"); dg = torch.zeros(D, device="cuda"); dc = torch.zeros(D, device="cuda")
        dx2, dyb = ll.rmsnorm_bwd_layerscale(dy, x, w, rstd, fin, ybr, gamma, dw2, dg, dc, rowscale=frs)
        ref_dx = xr.grad + dx_in if fin is not None else xr.grad
        assert _rel(dx2, ref_dx) < 1e-4 and _rel(dw2, wr.grad) < 2e-4
        d = ref_dx * rs[:, None] if frs is not None else ref_dx
        assert _rel(dyb, d * gamma.float()) < 5e-3
        assert _rel(dg, (d * ybr.float()).sum(0)) < 2e-4
        assert _rel(dc, d.sum(0) * gamma.float()) < 2e-4


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
