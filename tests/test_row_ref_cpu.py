"""tests/row_ref.py against torch.autograd in float64 on small shapes (CPU): every backward formula, the contrastive
loss's temperature gradient and AdamW over a few steps; and every scale positive and finite, all-zero rows included."""
import math

import pytest
import torch
import torch.nn.functional as F

import row_ref as rr

dt = torch.float64


def _close(got, want, tol=1e-10):
    assert torch.allclose(got, want, rtol=tol, atol=tol), float((got - want).abs().max())


def _scales_ok(out):
    for name, (ref, scale) in out.items():
        assert torch.isfinite(ref).all(), name
        assert torch.isfinite(scale).all() and (scale > 0).all(), name


def _rand(*shape, seed=0, s=1.0, off=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=dt) * s + off


@pytest.mark.parametrize("ln", [False, True])
def test_norm_fwd_bwd_match_autograd(ln):
    M, D = 7, 24
    x = _rand(M, D, seed=1, s=2.0, off=0.3)
    x[3] = 0.0                                                     # an all-zero row
    w, b = _rand(D, seed=2, s=0.2, off=1.0), _rand(D, seed=3, s=0.1)
    eps = 1e-5 if ln else 1e-6
    xr, wr, br = (t.clone().requires_grad_(True) for t in (x, w, b))
    if ln:
        y = F.layer_norm(xr, (D,), wr, br, eps)
    else:
        y = wr * xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + eps)
    fw = rr.norm_fwd(x, w, b if ln else None, eps, ln)
    _close(fw["y"][0], y.detach())
    _scales_ok(fw)
    dy, dx_in = _rand(M, D, seed=4), _rand(M, D, seed=5)
    y.backward(dy)
    mean = fw["mean"][0] if ln else None
    dw0, db0 = _rand(D, seed=6), _rand(D, seed=7)
    bw = rr.norm_bwd(dy, x, w, mean, fw["rstd"][0], ln, dx_in=dx_in, dweight=dw0, dbias=db0 if ln else None)
    _close(bw["dx"][0], xr.grad + dx_in)
    _close(bw["dweight"][0], wr.grad + dw0)
    if ln:
        _close(bw["dbias"][0], br.grad + db0)
    _scales_ok(bw)


@pytest.mark.parametrize("with_y,with_gamma,with_rs", [(True, True, True), (False, True, False), (True, False, True)])
def test_layerscale_bwd_matches_autograd(with_y, with_gamma, with_rs):
    """dy, dgamma and the branch bias gradient dcolsum are the gradients of out = rs * gamma * (ybr + bias)."""
    M, D = 9, 16
    dx = _rand(M, D, seed=1)
    y, gamma, bias = _rand(M, D, seed=2), _rand(D, seed=3, s=0.1), torch.zeros(D, dtype=dt)
    rs = (torch.arange(M) % 3 != 0).to(dt) / 0.7                   # dropped rows: rs = 0
    yr, gr, brr = (t.clone().requires_grad_(True) for t in (y, gamma, bias))
    r = rs[:, None] if with_rs else 1.0
    out = r * (gr if with_gamma else 1.0) * (yr + brr)
    out.backward(dx)
    dg0, dc0 = _rand(D, seed=4), _rand(D, seed=5)
    res = rr.layerscale_bwd(dx, y if with_y else None, gamma if with_gamma else None, dg0, dc0, rs if with_rs else None)
    _close(res["dy"][0], yr.grad)
    _close(res["dcolsum"][0], brr.grad + dc0)
    if with_y and with_gamma:
        _close(res["dgamma"][0], gr.grad + dg0)
    _scales_ok(res)
    cs = rr.colsum(y, out=dc0)
    _close(cs["out"][0], y.sum(0) + dc0)
    _scales_ok(cs)


def test_rmsnorm_bwd_layerscale_matches_autograd():
    M, D = 6, 32
    x = _rand(M, D, seed=1, s=2.0)
    x[2] = 0.0
    w, gamma = _rand(D, seed=2, s=0.2, off=1.0), _rand(D, seed=3, s=0.1)
    dy, dx_in, ybr = _rand(M, D, seed=4), _rand(M, D, seed=5), _rand(M, D, seed=6)
    rs = torch.tensor([1.0, 0.0, 1.25, 1.25, 0.0, 1.25], dtype=dt)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    (wr * xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-6)).backward(dy)
    dxt = xr.grad + dx_in
    yr, gr, br = ybr.clone().requires_grad_(True), gamma.clone().requires_grad_(True), torch.zeros(D, dtype=dt, requires_grad=True)
    (rs[:, None] * gr * (yr + br)).backward(dxt)
    rstd = torch.rsqrt(x.pow(2).mean(-1) + 1e-6)
    z = torch.zeros(D, dtype=dt)
    res = rr.rmsnorm_bwd_layerscale(dy, x, w, rstd, dx_in, ybr, gamma, z, z, z, rowscale=rs)
    _close(res["dx"][0], dxt)
    _close(res["dweight"][0], wr.grad)
    _close(res["dyb"][0], yr.grad)
    _close(res["dgamma"][0], gr.grad)
    _close(res["dcolsum"][0], br.grad)
    _scales_ok(res)


@pytest.mark.parametrize("gs", [1.0, -0.37])
def test_ln_l2_fwd_bwd_match_autograd(gs):
    M, C = 5, 40
    z = _rand(M, C, seed=1, s=1.5, off=0.2)
    z[1] = 0.0                                                      # y = b on this row
    w, b = _rand(C, seed=2, s=0.2, off=1.0), _rand(C, seed=3, s=0.1)
    tgt = F.normalize(_rand(M, C, seed=4), dim=-1)
    zr, wr, br = (t.clone().requires_grad_(True) for t in (z, w, b))
    y = F.layer_norm(zr, (C,), wr, br, 1e-5)
    o = y / y.norm(dim=-1, keepdim=True)
    old = torch.tensor([0.5], dtype=dt)
    fw = rr.ln_l2_fwd(z, w, b, 1e-5, target=tgt, loss_sum=old)
    _close(fw["out"][0], o.detach())
    _close(fw["loss"][0], old + (2 - 2 * (o * tgt).sum(-1)).sum().detach())
    _close(fw["inv_n"][0], 1.0 / y.detach().norm(dim=-1))
    _scales_ok(fw)
    dout = _rand(M, C, seed=5)
    (o * dout).sum().mul(gs).backward()
    stats = torch.stack([fw["mean"][0], fw["rstd"][0], fw["inv_n"][0]], 1)
    z0 = torch.zeros(C, dtype=dt)
    bw = rr.ln_l2_bwd(z, w, b, stats, dout, gscale_host=gs / 2, gscale_dev=torch.tensor([2.0], dtype=dt),
                      dweight=z0, dbias=z0)
    _close(bw["dz"][0], zr.grad)
    _close(bw["dweight"][0], wr.grad)
    _close(bw["dbias"][0], br.grad)
    _scales_ok(bw)


def test_l2norm_rows_match_autograd():
    M, C = 4, 16
    x = _rand(M, C, seed=1)
    x[2] = 0.0                                                      # the 1e-12 clamp
    xr = x.clone().requires_grad_(True)
    y = F.normalize(xr, dim=-1)
    fw = rr.l2norm_rows_fwd(x)
    _close(fw["out"][0], y.detach())
    assert fw["inv"][0][2] == 1e12
    _scales_ok(fw)
    dy = _rand(M, C, seed=2)
    y.backward(dy)
    bw = rr.l2norm_rows_bwd(dy, fw["out"][0], fw["inv"][0])
    _close(bw["dx"][0], xr.grad)
    _scales_ok(bw)


@pytest.mark.parametrize("idx", [[0, 1, 2, 3, 4, 5], [0, 1, 1, 2, 2, 2], [7] * 6])
@pytest.mark.parametrize("gs", [1.0, 0.25])
def test_vtc_loss_and_dtemp_match_autograd(idx, gs):
    G = len(idx)
    idx = torch.tensor(idx)
    cos = torch.tanh(_rand(G, G, seed=3))
    temp = 0.07
    cr = cos.clone().requires_grad_(True)
    tr = torch.tensor(float(torch.tensor(temp, dtype=torch.float32)), dtype=dt, requires_grad=True)
    s = cr / tr
    tg = (idx[:, None] == idx[None, :]).to(dt)
    tg = tg / tg.sum(1, keepdim=True)
    loss = (-(torch.log_softmax(s, 1) * tg).sum(1).mean() - (torch.log_softmax(s.t(), 1) * tg).sum(1).mean()) / 2
    (loss * gs).backward()
    old = torch.tensor([0.25], dtype=dt)
    fw = rr.vtc_loss_fwd(cos, idx, temp, loss=old)
    _close(fw["loss"][0], old + loss.detach())
    _close(fw["lse_r"][0], torch.logsumexp(s.detach(), 1))
    _close(fw["lse_c"][0], torch.logsumexp(s.detach(), 0))
    _scales_ok(fw)
    for temp_dev in (None, tr.detach().reshape(1)):
        bw = rr.vtc_loss_bwd(cos, idx, temp, fw["lse_r"][0], fw["lse_c"][0], gscale_host=gs / 4,
                             gscale_dev=torch.tensor([4.0], dtype=dt), temp_dev=temp_dev, dtemp=old)
        _close(bw["dcos"][0], cr.grad)
        _close(bw["dtemp"][0], old + tr.grad)
        _scales_ok(bw)


def test_mse_matches_autograd():
    pred, label = _rand(300, seed=1), _rand(300, seed=2)
    pr = pred.clone().requires_grad_(True)
    loss = ((pr - label) ** 2).sum()
    (loss * 0.125).backward()
    old = torch.tensor([2.0], dtype=dt)
    res = rr.mse_loss(pred, label, loss_sum=old, gscale_host=0.5, gscale_dev=torch.tensor([0.25], dtype=dt),
                      dpred=torch.empty(300))
    _close(res["loss"][0], old + loss.detach())
    _close(res["dpred"][0], pr.grad)
    _scales_ok(res)


@pytest.mark.parametrize("gscale", [1.0, 0.5])
def test_adamw_matches_torch_over_steps(gscale):
    n = 37
    p0 = _rand(n, seed=1)
    ref = torch.nn.Parameter(p0.clone())
    lr, b1, b2, eps, wd = (float(torch.tensor(v, dtype=torch.float32)) for v in (1e-3, 0.9, 0.95, 1e-8, 0.05))
    opt = torch.optim.AdamW([ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    master, m, v = p0.clone(), torch.zeros(n, dtype=dt), torch.zeros(n, dtype=dt)
    for step in range(1, 5):
        g = _rand(n, seed=10 + step)
        g[:3] = 0.0                                                  # v stays 0: the update is 0, its scale finite
        ref.grad = g * gscale
        opt.step()
        res = rr.adamw_step(master, m, v, g, lr, b1, b2, eps, wd, step, grad_scale=gscale)
        _scales_ok(res)
        master, m, v = res["master"][0], res["exp_avg"][0], res["exp_avg_sq"][0]
        _close(master, ref.detach(), tol=1e-12)
        _close(m, opt.state[ref]["exp_avg"], tol=1e-12)
        _close(v, opt.state[ref]["exp_avg_sq"], tol=1e-12)
    assert not math.isnan(float(master.sum()))


def test_model_formulas_match_the_oracle():
    """The reference's model-level formulas agree with oracle/restate.py: RMSNorm, LayerNorm, the decoder heads'
    alignment loss, the contrastive loss and the pixel MSE."""
    from oracle import restate
    M, C = 6, 32
    x = _rand(M, C, seed=1, s=2.0)
    w, b = _rand(C, seed=2, s=0.2, off=1.0), _rand(C, seed=3, s=0.1)
    # restate.rmsnorm takes its statistics in fp32, as the reference module does
    _close(rr.norm_fwd(x, w, None, 1e-6, False)["y"][0], restate.rmsnorm(x, w, 1e-6), tol=1e-6)
    _close(rr.norm_fwd(x, w, b, 1e-5, True)["y"][0], restate.layernorm(x, w, b, 1e-5))
    tgt = F.normalize(_rand(M, C, seed=4), dim=-1)
    loss = rr.ln_l2_fwd(x, w, b, 1e-5, target=tgt)["loss"][0]
    _close(loss / M, restate.align_loss(restate.l2n(restate.layernorm(x, w, b)), tgt).reshape(1))
    v, t = _rand(8, 16, seed=5), _rand(8, 16, seed=6)
    idx = torch.tensor([0, 1, 1, 2, 3, 3, 3, 4])
    cos = F.normalize(v, dim=-1) @ F.normalize(t, dim=-1).t()
    _close(rr.vtc_loss_fwd(cos, idx, 0.07)["loss"][0], restate.vtc_loss(v, t, idx, 0.07).reshape(1), tol=1e-7)
    pred, label = _rand(50, seed=7), _rand(50, seed=8)
    _close(rr.mse_loss(pred, label, loss_sum=torch.zeros(1, dtype=dt))["loss"][0] / 50,
           restate.mse_loss(pred, label).reshape(1))
