"""float64 reference of the row kernels (ivb_norm.cu, ivb_loss.cu) and the per-element error metric their tests use.

Each function takes the arguments of the lowlevel wrapper of one entry point and returns, for every output the call
writes, a pair (ref, scale) of float64 tensors: the reference, and a per-element tolerance `scale`, the fp32 error a
correct kernel may make before the output is rounded to its storage format.  gemm_ref.elem_errors adds half an ulp of
that format and divides, so 1 is the edge of what a correct kernel can produce.

`scale` is U24 = 2^-24 times the magnitudes of the terms that produce the element, times a constant for the depth of
the fp32 sums behind it:
  - a row statistic (a warp's sum over D columns: D / 32 sequential adds per lane, then five shuffle levels) carries
    ROW x sqrt(D) x the sum of its terms' magnitudes;
  - a column sum over M rows (per-warp partials in shared memory, then per-CTA slots added in order) carries
    COL x sqrt(M) x the sum of its terms' magnitudes;
  - every elementwise multiply or add of the kernel's expression adds U24 times the magnitude it rounds, and the
    fast-math exp2 / log2 / rsqrt / divide approximations add a few ulps (EVAL).
The sqrt depth factors are the growth of a rounding random walk; the kernels' measured errors stay well inside them.

A reference of a backward pass takes the statistics the forward kernel saved (mean, rstd, stats, lse) as exact inputs:
it checks the backward kernel alone.  Everything runs in float64 on the inputs' device, in row chunks, so the full
training shapes fit.
"""
from __future__ import annotations

import math

import torch

U24 = 2.0 ** -24
ROW = 2.0          # row statistics: x sqrt(D) x sum |terms|
COL = 2.0          # parameter gradients: x sqrt(M) x sum_m |term|
EVAL = 8.0         # fast-math rsqrt / exp2 / log2 / divide, in fp32 ulps
POWF = 2.0 ** -22  # fast-math powf(b, s) = ex2.approx(s lg2.approx(b)): relative error POWF (1 + s)
ROW_CHUNK = 4096
TINY = 2.0 ** -149  # the smallest fp32 step: no scale is zero, even on an all-zero row


def _d(t):
    return None if t is None else t.double()


def _chunks(M):
    for r0 in range(0, M, ROW_CHUNK):
        yield slice(r0, min(M, r0 + ROW_CHUNK))


def _rowdepth(D):
    return ROW * math.sqrt(D) * U24


def _coldepth(M):
    return COL * (math.sqrt(M) + 4.0) * U24


def _fin(out):
    """Every scale at least TINY."""
    return {k: (r, s.clamp_min(TINY)) for k, (r, s) in out.items()}


def _cat(parts):
    """[{name: (ref, scale)} per row chunk] -> {name: (ref, scale)} over all rows."""
    return {k: (torch.cat([p[k][0] for p in parts]), torch.cat([p[k][1] for p in parts])) for k in parts[0]}


def _accum(old, total, total_abs, M):
    """old + total (a column sum over M rows, fp32 [N]) and its scale; old None: the output starts at 0."""
    o = _d(old) if old is not None else torch.zeros_like(total)
    return o + total, _coldepth(M) * total_abs + U24 * (o.abs() + (o + total).abs())


# ---------------------------------------------------------------- RMSNorm / LayerNorm
def norm_fwd(x, weight, bias=None, eps=1e-6, layernorm=False):
    """ivb_norm_fwd: y = (x - mean) * rstd * w (+ b); {"y", "rstd"[, "mean"]}."""
    M, D = x.shape
    w, b = _d(weight), _d(bias)
    parts = []
    for rs in _chunks(M):
        xv = x[rs].double()
        mu = xv.mean(1, keepdim=True) if layernorm else torch.zeros_like(xv[:, :1])
        xc = xv - mu
        ms = (xc * xc).mean(1, keepdim=True)
        r = 1.0 / torch.sqrt(ms + eps)
        xh = xc * r
        y = xh * w + (b if (layernorm and b is not None) else 0.0)
        # mean: a row sum of |x|; rstd: a row sum of xc^2 (relative error halves through the square root)
        e_mu = _rowdepth(D) * xv.abs().mean(1, keepdim=True) if layernorm else torch.zeros_like(mu)
        rel_r = _rowdepth(D) + EVAL * U24 + 2.0 * e_mu * xc.abs().mean(1, keepdim=True) / (ms + eps)
        sy = (rel_r + 3 * U24) * (xh * w).abs() + e_mu * r * w.abs() + U24 * y.abs()
        out = {"y": (y, sy), "rstd": (r[:, 0], (rel_r * r)[:, 0])}
        if layernorm:
            out["mean"] = (mu[:, 0], (e_mu + U24 * mu.abs())[:, 0])
        parts.append(out)
    return _fin(_cat(parts))


def norm_bwd(dy, x, weight, mean, rstd, layernorm=False, dx_in=None, dweight=None, dbias=None):
    """ivb_norm_bwd with the forward's mean / rstd as given: dx = rstd (g w - s1 - xh s2) (+ dx_in), xh = (x - mean)
    rstd, s1 = mean(g w) (LayerNorm only), s2 = mean(g w xh); dweight += sum_m g xh, dbias += sum_m g.
    dweight / dbias are read (their values before the call) and say whether the call writes them.
    {"dx"[, "dweight"][, "dbias"]}."""
    M, D = x.shape
    w = _d(weight)
    gw_sum = torch.zeros(D, dtype=torch.float64, device=x.device)
    gw_abs = torch.zeros_like(gw_sum)
    gb_sum, gb_abs = torch.zeros_like(gw_sum), torch.zeros_like(gw_sum)
    dxs, sdx = [], []
    for rs in _chunks(M):
        g = dy[rs].double()
        r = rstd[rs].double()[:, None]
        mu = mean[rs].double()[:, None] if layernorm else 0.0
        xh = (x[rs].double() - mu) * r
        gwt = g * w
        s1 = gwt.mean(1, keepdim=True) if layernorm else torch.zeros_like(r)
        s2 = (gwt * xh).mean(1, keepdim=True)
        dx = r * (gwt - s1 - xh * s2)
        e1 = _rowdepth(D) * gwt.abs().mean(1, keepdim=True) if layernorm else 0.0
        e2 = _rowdepth(D) * (gwt * xh).abs().mean(1, keepdim=True) + 3 * U24 * (gwt * xh).abs().mean(1, keepdim=True)
        s = r * (3 * U24 * (gwt.abs() + s1.abs() + (xh * s2).abs()) + e1 + xh.abs() * e2) + U24 * dx.abs()
        if dx_in is not None:
            dx = dx + dx_in[rs].double()
            s = s + U24 * dx.abs()
        dxs.append(dx); sdx.append(s)
        gw_sum += (g * xh).sum(0); gw_abs += (g * xh).abs().sum(0)
        gb_sum += g.sum(0); gb_abs += g.abs().sum(0)
    out = {"dx": (torch.cat(dxs), torch.cat(sdx))}
    if dweight is not None:
        out["dweight"] = _accum(dweight, gw_sum, gw_abs, M)
        if layernorm and dbias is not None:
            out["dbias"] = _accum(dbias, gb_sum, gb_abs, M)
    return _fin(out)


# ---------------------------------------------------------------- LayerScale backward, column sums
def layerscale_bwd(dx, y=None, gamma=None, dgamma=None, dcolsum=None, rowscale=None):
    """ivb_layerscale_bwd: d = rowscale dx; dy = gamma d; dgamma += sum_m d y; dcolsum += gamma sum_m d.
    {"dy"[, "dgamma"][, "dcolsum"]}."""
    return _fin(_layerscale(dx.double(), torch.zeros_like(dx, dtype=torch.float64), y, gamma, dgamma, dcolsum, rowscale))


def _layerscale(dxv, sdx, y, gamma, dgamma, dcolsum, rowscale):
    M, D = dxv.shape
    rs = rowscale.double()[:, None] if rowscale is not None else torch.ones_like(dxv[:, :1])
    d = rs * dxv
    sd = rs.abs() * sdx + U24 * d.abs()
    gm = _d(gamma) if gamma is not None else torch.ones_like(dxv[0])
    dyv = d * gm
    out = {"dy": (dyv, gm.abs() * sd + U24 * dyv.abs())}
    if y is not None and dgamma is not None:
        yv = y.double()
        t, ta = (d * yv).sum(0), (d * yv).abs().sum(0) + (sd * yv.abs()).sum(0) / _coldepth(M)
        out["dgamma"] = _accum(dgamma, t, ta, M)
    if dcolsum is not None:
        t, ta = d.sum(0) * gm, (d.abs().sum(0) + sd.sum(0) / _coldepth(M) + U24 * d.sum(0).abs() / _coldepth(M)) * gm.abs()
        out["dcolsum"] = _accum(dcolsum, t, ta, M)
    return out


def colsum(x, out=None):
    """ivb_colsum_bf16: out += sum_m x.  {"out"}."""
    xv = x.double()
    return _fin({"out": _accum(out, xv.sum(0), xv.abs().sum(0), x.shape[0])})


def rmsnorm_bwd_layerscale(dy, x, weight, rstd, dx_in, ybr, gamma, dweight, dgamma, dcolsum, rowscale=None):
    """ivb_rmsnorm_bwd_layerscale: the RMSNorm backward (norm_bwd) followed by the LayerScale backward of its dx.
    {"dx", "dyb"[, "dweight"][, "dgamma"][, "dcolsum"]}."""
    n = norm_bwd(dy, x, weight, None, rstd, dx_in=dx_in, dweight=dweight)
    dxv, sdx = n["dx"]
    ls = _layerscale(dxv, sdx, ybr, gamma, dgamma, dcolsum, rowscale)
    out = {"dx": n["dx"], "dyb": ls["dy"]}
    if "dweight" in n:
        out["dweight"] = n["dweight"]
    for k in ("dgamma", "dcolsum"):
        if k in ls:
            out[k] = ls[k]
    return _fin(out)


# ---------------------------------------------------------------- LayerNorm -> L2 (decoder heads)
def ln_l2_fwd(z, weight, bias, eps=1e-5, target=None, loss_sum=None):
    """ivb_ln_l2_fwd: y = LN(z) w + b, out = y / ||y||, stats = (mean, rstd, 1/||y||), loss_sum += sum_rows
    (2 - 2 <out, target>).  {"out", "mean", "rstd", "inv_n"[, "loss"]}."""
    M, C = z.shape
    n = norm_fwd(z, weight, bias, eps, layernorm=True)
    y, sy = n["y"]
    nn2 = (y * y).sum(1, keepdim=True)
    inv = 1.0 / torch.sqrt(nn2)
    rel_n = (_rowdepth(C) + EVAL * U24) + (sy * y.abs()).sum(1, keepdim=True) / nn2
    o = y * inv
    so = (sy + U24 * y.abs()) * inv + rel_n * o.abs()
    out = {"out": (o, so), "mean": n["mean"], "rstd": n["rstd"], "inv_n": (inv[:, 0], (rel_n * inv)[:, 0])}
    if target is not None:
        t = target.double()
        dot = (o * t).sum(1)
        sdot = (so * t.abs()).sum(1) + _rowdepth(C) * (o * t).abs().sum(1)
        per = 2.0 - 2.0 * dot
        out["loss"] = _accum(loss_sum, per.sum()[None], (2.0 * sdot.sum() / _coldepth(M) + per.abs().sum())[None], M)
    return _fin(out)


def ln_l2_bwd(z, weight, bias, stats, dout, gscale_host=1.0, gscale_dev=None, dweight=None, dbias=None):
    """ivb_ln_l2_bwd with the forward's stats as given: xh = (z - mean) rstd, o = (xh w + b) inv_n, g = gs dout,
    a = <g, o>, dy = inv_n (g - o a), dz = rstd (dy w - s1 - xh s2) with s1 = mean(dy w), s2 = mean(dy w xh);
    dweight += sum_m dy xh, dbias += sum_m dy.  {"dz"[, "dweight"][, "dbias"]}."""
    M, C = z.shape
    w, b = weight.double(), bias.double()
    gs = float(gscale_host) * (float(gscale_dev.item()) if gscale_dev is not None else 1.0)
    dw_s = torch.zeros(C, dtype=torch.float64, device=z.device)
    dw_a, db_s, db_a = torch.zeros_like(dw_s), torch.zeros_like(dw_s), torch.zeros_like(dw_s)
    dzs, sdz = [], []
    for rs in _chunks(M):
        st = stats[rs].double()
        mu, r, inv = st[:, :1], st[:, 1:2], st[:, 2:3]
        xh = (z[rs].double() - mu) * r
        o = (xh * w + b) * inv
        g = gs * dout[rs].double()
        a = (g * o).sum(1, keepdim=True)
        dyv = inv * (g - o * a)
        ea = (_rowdepth(C) + 4 * U24) * (g * o).abs().sum(1, keepdim=True)
        sdy = inv * (4 * U24 * (g.abs() + (o * a).abs()) + o.abs() * ea) + U24 * dyv.abs()
        dyw = dyv * w
        s1 = dyw.mean(1, keepdim=True)
        s2 = (dyw * xh).mean(1, keepdim=True)
        e1 = _rowdepth(C) * dyw.abs().mean(1, keepdim=True) + (sdy * w.abs()).mean(1, keepdim=True)
        e2 = _rowdepth(C) * (dyw * xh).abs().mean(1, keepdim=True) + (sdy * (w * xh).abs()).mean(1, keepdim=True)
        dz = r * (dyw - s1 - xh * s2)
        s = r * (3 * U24 * (dyw.abs() + s1.abs() + (xh * s2).abs()) + sdy * w.abs() + e1 + xh.abs() * e2)
        dzs.append(dz); sdz.append(s + U24 * dz.abs())
        dw_s += (dyv * xh).sum(0); dw_a += (dyv * xh).abs().sum(0) + (sdy * xh.abs()).sum(0) / _coldepth(M)
        db_s += dyv.sum(0); db_a += dyv.abs().sum(0) + sdy.sum(0) / _coldepth(M)
    out = {"dz": (torch.cat(dzs), torch.cat(sdz))}
    if dweight is not None:
        out["dweight"] = _accum(dweight, dw_s, dw_a, M)
        if dbias is not None:
            out["dbias"] = _accum(dbias, db_s, db_a, M)
    return _fin(out)


# ---------------------------------------------------------------- F.normalize rows
def l2norm_rows_fwd(x):
    """ivb_l2norm_rows_fwd: out = x / max(||x||, 1e-12), inv_norm = 1 / max(||x||, 1e-12).  {"out", "inv"}."""
    C = x.shape[1]
    xv = x.double()
    nrm = torch.sqrt((xv * xv).sum(1, keepdim=True))
    inv = 1.0 / nrm.clamp_min(1e-12)
    rel = _rowdepth(C) + EVAL * U24
    o = xv * inv
    return _fin({"out": (o, (rel + U24) * o.abs()), "inv": (inv[:, 0], (rel * inv)[:, 0])})


def l2norm_rows_bwd(dy, xn, inv):
    """ivb_l2norm_rows_bwd with xn, inv as given: dx = inv (dy - xn <dy, xn>).  {"dx"}."""
    C = dy.shape[1]
    g, v, iv = dy.double(), xn.double(), inv.double()[:, None]
    dot = (g * v).sum(1, keepdim=True)
    edot = (_rowdepth(C) + U24) * (g * v).abs().sum(1, keepdim=True)
    dx = iv * (g - v * dot)
    return _fin({"dx": (dx, iv * (2 * U24 * (g.abs() + (v * dot).abs()) + v.abs() * edot) + U24 * dx.abs())})


# ---------------------------------------------------------------- video-text contrastive loss
def _vtc_s(cosm, idx, temp, temp_dev):
    t = float(temp_dev.item()) if temp_dev is not None else float(torch.tensor(temp, dtype=torch.float32))
    S = cosm.double() / t
    eq = (idx[:, None] == idx[None, :]).double()
    tg = eq / eq.sum(1, keepdim=True)
    return t, S, tg


def vtc_loss_fwd(cosm, idx, temp, temp_dev=None, loss=None):
    """ivb_vtc_loss_fwd: S = cos / temp, lse_row / lse_col = logsumexp of S's rows / columns, loss += 1/(2G)
    sum_i [(lse_r[i] - sum_j tg[i,j] S[i,j]) + (lse_c[i] - sum_j tg[i,j] S[j,i])], tg = (idx == idx^T) / rowcount.
    temp_dev overrides temp.  {"lse_r", "lse_c", "loss"}."""
    G = cosm.shape[0]
    _, S, tg = _vtc_s(cosm, idx, temp, temp_dev)
    lse_r, lse_c = torch.logsumexp(S, 1), torch.logsumexp(S, 0)
    ts_r, ts_c = (tg * S).sum(1), (tg * S.t()).sum(1)
    mx_r, mx_c = S.abs().amax(1), S.abs().amax(0)
    # S itself carries 2 ulps (cos * 1/temp); exp(s - max) an EVAL-ulp error growing with |s - max|
    e_r = U24 * (EVAL + 4 * mx_r + math.sqrt(G) * ROW + lse_r.abs())
    e_c = U24 * (EVAL + 4 * mx_c + math.sqrt(G) * ROW + lse_c.abs())
    per = (lse_r - ts_r) + (lse_c - ts_c)
    sper = e_r + e_c + U24 * (math.sqrt(G) * ROW + 2) * ((tg * S.abs()).sum(1) + (tg * S.t().abs()).sum(1))
    total = per.sum() / (2 * G)
    tabs = (sper.sum() + U24 * per.abs().sum()) / (2 * G) / _coldepth(G) + per.abs().sum() / (2 * G)
    return _fin({"lse_r": (lse_r, e_r), "lse_c": (lse_c, e_c), "loss": _accum(loss, total[None], tabs[None], G)})


def vtc_loss_bwd(cosm, idx, temp, lse_r, lse_c, gscale_host=1.0, gscale_dev=None, temp_dev=None, dtemp=None):
    """ivb_vtc_loss_bwd with lse_r / lse_c as given: dS = gs / (2G) (exp(S - lse_r[a]) + exp(S - lse_c[b]) - 2 tg),
    dcos = dS / temp, dtemp += sum dS (-S / temp).  {"dcos", "dtemp"}."""
    G = cosm.shape[0]
    t, S, tg = _vtc_s(cosm, idx, temp, temp_dev)
    gs = float(gscale_host) * (float(gscale_dev.item()) if gscale_dev is not None else 1.0) / (2 * G)
    lr, lc = lse_r.double()[:, None], lse_c.double()[None, :]
    pr, pc = torch.exp(S - lr), torch.exp(S - lc)
    ds = gs * (pr + pc - 2.0 * tg)
    # exp of an argument that carries ulps of |S| and |lse|, evaluated by ex2.approx
    e_arg_r = U24 * (EVAL + 4 * (S.abs() + lr.abs()))
    e_arg_c = U24 * (EVAL + 4 * (S.abs() + lc.abs()))
    sds = abs(gs) * (pr * e_arg_r + pc * e_arg_c + 3 * U24 * (pr + pc + 2.0 * tg))
    dcos = ds / t
    term = ds * (-S / t)
    tsum = term.sum()
    tabs = term.abs().sum() + ((S / t).abs() * sds).sum() / _coldepth(G * G) + 3 * U24 * term.abs().sum() / _coldepth(G * G)
    return _fin({"dcos": (dcos, (sds + 2 * U24 * ds.abs()) / t),
            "dtemp": _accum(dtemp, tsum[None], tabs[None], G * G)})


# ---------------------------------------------------------------- MSE
def mse_loss(pred, label, loss_sum=None, gscale_host=0.0, gscale_dev=None, dpred=None):
    """ivb_mse_loss: loss_sum += sum (pred - label)^2, dpred = gs 2 (pred - label).  {"loss"[, "dpred"]}."""
    d = pred.double().reshape(-1) - label.double().reshape(-1)
    gs = float(gscale_host) * (float(gscale_dev.item()) if gscale_dev is not None else 1.0)
    n = d.numel()
    out = {}
    if loss_sum is not None:
        out["loss"] = _accum(loss_sum, (d * d).sum()[None], (3 * d * d).sum()[None], n)
    if dpred is not None:
        out["dpred"] = (2.0 * gs * d, 3 * U24 * (2.0 * gs * d).abs() + 2.0 * abs(gs) * U24 * label.double().reshape(-1).abs())
    return _fin(out)


# ---------------------------------------------------------------- AdamW
def adamw_step(master, exp_avg, exp_avg_sq, grad, lr, beta1, beta2, eps, wd, step, grad_scale=1.0, grad_scale_dev=None):
    """One ivb_adamw_step from the state BEFORE the call (torch.optim.AdamW semantics, bias corrections from `step`):
    g = grad_scale (*grad_scale_dev) grad; p *= 1 - lr wd; m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2;
    p -= lr (m / bc1) / (sqrt(v / bc2) + eps).  lr, betas, eps, wd are taken at their fp32 values.
    {"master", "exp_avg", "exp_avg_sq"}."""
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))
    lr, b1, b2, eps, wd = (f32(v) for v in (lr, beta1, beta2, eps, wd))
    gsc = f32(grad_scale) * (float(grad_scale_dev.item()) if grad_scale_dev is not None else 1.0)
    g = grad.double() * gsc
    p0, m0, v0 = master.double(), exp_avg.double(), exp_avg_sq.double()
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    decay = 1.0 - lr * wd
    p = p0 * decay
    m = b1 * m0 + (1 - b1) * g
    v = b2 * v0 + (1 - b2) * g * g
    sm = 3 * U24 * ((b1 * m0).abs() + ((1 - b1) * g).abs())
    sv = 4 * U24 * ((b2 * v0).abs() + (1 - b2) * g * g)
    den = torch.sqrt(v / bc2) + eps
    upd = lr * (m / bc1) / den
    # relative error of the update: the bias corrections 1 - b^step (the kernel's fast-math powf: an error of
    # POWF (1 + step) b^step, relative to 1 - b^step), sqrt and divide, and m's and v's own errors
    e_bc1 = (b1 ** step * POWF * (1 + step) + U24) / bc1
    e_bc2 = (b2 ** step * POWF * (1 + step) + U24) / bc2
    rel = EVAL * U24 + e_bc1 + 0.5 * e_bc2
    s_upd = (rel * upd.abs() + lr * (sm / bc1) / den
             + upd.abs() * torch.sqrt(v / bc2) / den * sv / (2 * v).clamp_min(1e-300))
    pn = p - upd
    return _fin({"master": (pn, s_upd + 2 * U24 * (p.abs() + pn.abs())), "exp_avg": (m, sm), "exp_avg_sq": (v, sv)})
