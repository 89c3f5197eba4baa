"""The InternVideo2 RMSNorm block (modules.Block: ops.block_forward, ops.block_backward, ops.BlockFn) against float64, on
every path the host code takes: the q/k norms in one launch (D <= 1536), in two (D > 1536) or not at all; the fused
norm2 + LayerScale backward (D <= 1536, M >= 1024, LayerScale on) or its two calls; with and without LayerScale and qkv
bias; tanh and erf GELU; DropPath factors with and without plans; saved activations and the checkpoint recompute.

Call by call (test_rmsnorm_block_calls_match_float64): every library call block_forward(save=True) and block_backward
make is recorded with its outputs, and each stage is compared element by element with the float64 reference of that
stage (tests/row_ref.py, tests/gemm_ref.py, tests/attn_ref.py) at the limits of tests/test_rows_gpu.py,
tests/test_gemm_epilogue_gpu.py and tests/test_attn_gpu.py.  A stage's reference is built from what the math needs --
the block input, the parameters, the DropPath factors and the recorded outputs of the stages before it -- never from
the operands the call received, so a call handed the wrong buffer, pitch, gamma, rowscale, aux or flags fails at its
own stage.  A failure names the stage, the worst error and where it lies.  Rows a DropPath plan lets a GEMM skip
(zeros, or values no later stage reads) are left out of the bf16 activations' checks; the attention rows and gradient
rows of a dropped clip must be exactly 0.  The call sequence is checked last: it shows which of the paths above ran.

End to end (test_rmsnorm_block_matches_float64): Block.forward_stream through BlockFn against oracle.restate.block in
float64, on the GPU.  The output and the input gradient are compared without their identity part (x, dy), so the
bounds hold on what the two branches add: per tensor at 1e-2 (3e-2 for the parameter gradients), as in
tests/test_layernorm_block_gpu.py, and per slice (tests/local_err.py) -- every token row of the branch and of dx - dy,
every output channel of a weight gradient, every head of the q/k-norm weight gradients -- so an error confined to one
clip, head or channel cannot hide in a tensor norm.  Each slice bound in LOCAL is about twice the worst value measured
over this file on an H100 80GB HBM3 (SXM, 700 W power limit); the measured value is beside it.

Bit relations (test_rmsnorm_block_bit_relations): the checkpointed block gives the saved block's output, input gradient
and parameter gradients bit for bit, and forward_infer (no grad, nothing saved, no plans) the training forward's output.

The file (30 tests) runs in about 20 s on the H100.
"""
import inspect
import math
from typing import NamedTuple

import pytest
import torch

import row_ref as rr
from attn_ref import attn_ref_bwd, attn_ref_fwd, tile_errors
from attn_ref import worst as tile_worst
from gemm_ref import EPI_BIAS_GELU, EPI_GELU_BWD, EPI_RESID, elem_errors, gemm_ref
from gemm_ref import worst as gemm_worst
from local_err import rel, slice_errors, worst_slice
from test_attn_gpu import LIMITS as ATTN_LIMITS
from test_gemm_epilogue_gpu import LIMITS as GEMM_LIMITS
from test_rows_gpu import LIMITS as ROW_LIMITS


class Cfg(NamedTuple):
    D: int
    H: int
    hidden: int
    B: int
    n: int
    qk: bool = True            # qk_normalization
    ls: bool = True            # LayerScale (init_values)
    qkv_bias: bool = True
    tanh: bool = True          # use_fused_mlp: tanh GELU
    droppath: str = "none"     # "none"; "clip": per-clip factors; "plan": the same factors with their DropPath plans
    checkpoint: bool = False


# M = B n.  The fused norm2 + LayerScale backward runs at D <= 1536 with M >= 1024 and LayerScale on; the q/k norms run
# in one launch at D <= 1536 and in two above.
CONFIGS = {
    "d384_m834": Cfg(384, 6, 1536, 2, 417),
    "d384_m834_plain_erf": Cfg(384, 6, 1536, 2, 417, qk=False, ls=False, qkv_bias=False, tanh=False),
    "d384_m1023_clip": Cfg(384, 6, 1536, 3, 341, droppath="clip"),
    "d384_m1024_erf_plan_ckpt": Cfg(384, 6, 1536, 4, 256, qkv_bias=False, tanh=False, droppath="plan", checkpoint=True),
    "d1408_m834_erf_clip_ckpt": Cfg(1408, 16, 6144, 2, 417, tanh=False, droppath="clip", checkpoint=True),
    "d1408_m1251_plan": Cfg(1408, 16, 6144, 3, 417, droppath="plan"),
    "d1536_m1024_clip": Cfg(1536, 12, 6144, 4, 256, droppath="clip"),
    "d1536_m1023_nols_noqk_plan": Cfg(1536, 12, 6144, 3, 341, qk=False, ls=False, droppath="plan"),
    "d1600_m834_clip": Cfg(1600, 25, 6400, 2, 417, droppath="clip"),
    "d3200_m258_plan_ckpt": Cfg(3200, 25, 12800, 2, 129, qkv_bias=False, droppath="plan", checkpoint=True),
}

# Slice bounds of the end-to-end comparison, and beside each the worst value measured over this file (H100 80GB HBM3
# SXM, 700 W power limit).
LOCAL = {
    "branch_row": 6e-3,           # every token row of y - x                       measured 2.97e-3 (d384_m1023_clip)
    "dx_row": 1.1e-2,             # every token row of dx - dy                     measured 5.57e-3 (d384_m1023_clip)
    "attn.qkv.weight": 2.7e-2,    # every output channel (row) of the weight       measured 1.33e-2 (d3200)
    "attn.proj.weight": 2e-2,     #   gradients                                    measured 9.91e-3 (d3200)
    "mlp.fc1.weight": 1.25e-2,    #                                                measured 6.19e-3 (d3200)
    "mlp.fc2.weight": 1e-2,       #                                                measured 4.83e-3 (d3200)
    "attn.q_norm.weight": 2e-2,   # every head's d entries of the q/k-norm weight  measured 9.67e-3 (d1600)
    "attn.k_norm.weight": 1.8e-2,  # gradients                                     measured 8.81e-3 (d1600)
}

# Per-stage limit families: the element-wise limits of the row kernels and the GEMM epilogues, the tile limits of
# attention.
LIMITS = {**{"row_" + k: v for k, v in ROW_LIMITS.items()}, **{"gemm_" + k: v for k, v in GEMM_LIMITS.items()},
          **{"attn_" + k: v for k, v in ATTN_LIMITS.items()}}


# ---------------------------------------------------------------- the block and its inputs
def _block(cfg):
    from internvideo_b200.modules import Block
    torch.manual_seed(0)
    blk = Block(cfg.D, cfg.H, (cfg.hidden + 0.5) / cfg.D, qkv_bias=cfg.qkv_bias, init_values=0.1 if cfg.ls else None,
                use_fused_mlp=cfg.tanh, with_cp=cfg.checkpoint, qk_normalization=cfg.qk)
    assert blk.mlp.fc1.out_features == cfg.hidden
    with torch.no_grad():
        for nm, p in blk.named_parameters():
            if nm.endswith("weight") and p.ndim == 1:          # norm weights
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif nm.endswith("bias"):
                p.normal_(0, 0.1)
            elif nm.endswith("gamma"):
                p.mul_(1 + 0.5 * torch.rand_like(p))
    return blk.bfloat16().cuda().train()


def _inputs(cfg):
    """x, dy fp32 [M, D]; rs1 / rs2 fp32 [M] (None without DropPath): each branch drops one clip (the attention branch
    the first, the MLP branch the last) and scales the others by 1 / 0.8; plans (plan1, plan2) or None."""
    M = cfg.B * cfg.n
    g = torch.Generator().manual_seed(1)
    x = torch.randn((M, cfg.D), generator=g).cuda()
    dy = torch.randn((M, cfg.D), generator=g).cuda()
    rs1 = rs2 = plans = None
    if cfg.droppath != "none":
        f1, f2 = torch.full((cfg.B,), 1.25), torch.full((cfg.B,), 1.25)
        f1[0], f2[-1] = 0.0, 0.0
        rs1, rs2 = f1.repeat_interleave(cfg.n).cuda(), f2.repeat_interleave(cfg.n).cuda()
        if cfg.droppath == "plan":
            from internvideo_b200 import ops
            plans = tuple(ops.droppath_plan(torch.stack([rs1, rs2])))
    return x, dy, rs1, rs2, plans


# ---------------------------------------------------------------- recording the library calls
RECORDED = ("gemm", "norm_fwd", "rmsnorm_pair_fwd", "attn_fwd", "layerscale_bwd", "colsum", "norm_bwd",
            "rmsnorm_bwd_layerscale", "attn_bwd", "rmsnorm_pair_bwd")


class Call(NamedTuple):
    name: str
    before: dict      # tensor arguments by parameter name, as they were before the call
    after: dict       # ... and after it (outputs written in place, accumulators)
    ret: object       # the return value, cloned


def _clone(v):
    if torch.is_tensor(v):
        return v.clone()
    if isinstance(v, tuple):
        return tuple(_clone(t) for t in v)
    return v


class Recorder:
    """Replaces the lowlevel functions ops calls by wrappers that snapshot every tensor argument before and after the
    call and keep a copy of what it returns."""

    def __init__(self, monkeypatch):
        from internvideo_b200 import ops
        self.calls = []
        for name in RECORDED:
            fn = getattr(ops.ll, name)
            monkeypatch.setattr(ops.ll, name, self._wrap(name, fn, inspect.signature(fn)))

    def _wrap(self, name, fn, sig):
        def call(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            before = {k: v.clone() for k, v in bound.arguments.items() if torch.is_tensor(v)}
            ret = fn(*args, **kwargs)
            after = {k: v.clone() for k, v in bound.arguments.items() if torch.is_tensor(v)}
            self.calls.append(Call(name, before, after, _clone(ret)))
            return ret
        return call

    def take(self):
        """The calls recorded since the last take(), grouped by name in call order."""
        calls, self.calls = self.calls, []
        by = {nm: [c for c in calls if c.name == nm] for nm in RECORDED}
        return [c.name for c in calls], by


# ---------------------------------------------------------------- stage checks
class Stages:
    """The worst error of every checked output of every stage: name -> (value, limit, where)."""

    def __init__(self, cfg):
        self.cfg, self.res = cfg, {}

    def _rowinfo(self, m):
        return f"row {m} (clip {m // self.cfg.n}, token {m % self.cfg.n})"

    def elem(self, stage, fam, got, ref_scale, live=None):
        """Element-wise error of one output against (ref, scale), in units of the tolerance (gemm_ref.elem_errors).
        live: bool [M] rows to check (rows a DropPath plan may leave unwritten or zero are left out)."""
        ref, scale = ref_scale
        got = got.reshape(ref.shape)
        errs = elem_errors(got, ref, scale)
        if live is not None:
            errs = errs * live.to(errs.dtype).reshape(-1, *([1] * (errs.dim() - 1)))
        if errs.dim() == 2:
            e, where = gemm_worst(errs)
            m = int(errs.argmax()) // errs.shape[1]
            where = f"{self._rowinfo(m)}, {where}"
        else:
            i = int(errs.argmax())
            e, where = float(errs[i]), f"channel {i}"
        self.res[stage] = (e, LIMITS[fam], where)

    def attn(self, stage, fam, got, ref, live_clips):
        """Tile error (attn_ref.tile_errors) of a [M, H d] attention result over the live clips; a dropped clip's rows
        must be exactly 0."""
        c = self.cfg
        d = c.D // c.H
        worst_e, where = 0.0, "-"
        for b in range(c.B):
            rows = slice(b * c.n, (b + 1) * c.n)
            if not live_clips[b]:
                nz = int((got[rows] != 0).sum())
                if nz:
                    worst_e, where = math.inf, f"dropped clip {b}: {nz} nonzero elements"
                    break
                continue
            e, (_, h, band) = tile_worst(tile_errors(got[rows], ref[rows], 1, c.n, c.H, d))
            if e > worst_e:
                worst_e, where = e, f"clip {b}, head {h}, rows {64 * band}..{min(c.n, 64 * band + 64) - 1}"
        self.res[stage] = (worst_e, LIMITS[fam], where)

    def lse(self, stage, got, ref, live_clips):
        e = (got.double() - ref).abs()[live_clips]
        i = int(e.argmax())
        self.res[stage] = (float(e.reshape(-1)[i]), LIMITS["attn_lse"], f"flat index {i} of the live clips' [B, H, n]")

    def exact(self, stage, got, want):
        ok = torch.equal(got, want)
        self.res[stage] = (0.0 if ok else math.inf, 0.0, "bits" if ok else "differs")

    def failures(self):
        return [f"{s}: {e:.3g} > {lim:.3g} at {w}" for s, (e, lim, w) in self.res.items() if not e <= lim]


def _expected_calls(cfg, fused):
    pair = cfg.D <= 1536
    qkf = ["rmsnorm_pair_fwd"] if pair else ["norm_fwd", "norm_fwd"]
    qkb = ["rmsnorm_pair_bwd"] if pair else ["norm_bwd", "norm_bwd"]
    fwd = ["norm_fwd", "gemm", *(qkf if cfg.qk else []), "attn_fwd", "gemm", "norm_fwd", "gemm", "gemm"]
    bwd = ["layerscale_bwd", "gemm", "gemm", "colsum", "gemm", "gemm",
           *(["rmsnorm_bwd_layerscale"] if fused else ["norm_bwd", "layerscale_bwd"]), "gemm", "gemm", "attn_bwd",
           *(qkb if cfg.qk else []), "gemm", *(["colsum"] if cfg.qkv_bias else []), "gemm", "norm_bwd"]
    return fwd, bwd


def _run_calls(name, monkeypatch):
    """Runs block_forward(save=True) and block_backward on CONFIGS[name] with every library call recorded, and checks
    each stage.  Returns the Stages."""
    from internvideo_b200 import ops
    cfg = CONFIGS[name]
    blk = _block(cfg)
    x, dy, rs1, rs2, plans = _inputs(cfg)
    plan1, plan2 = plans or (None, None)
    spec = blk._spec(cfg.B, cfg.n, training=True)._replace(checkpoint=False)
    t = blk._param_tuple()
    t = ops.BlockParams(*(None if p is None else p.detach() for p in t))
    M, D, H, B, n = cfg.B * cfg.n, cfg.D, cfg.H, cfg.B, cfg.n
    d = D // H
    scale = d ** -0.5
    flags = spec.gelu_flags(True)
    fused = cfg.ls and D <= 1536 and M >= 1024

    rec = Recorder(monkeypatch)
    with torch.no_grad():
        x2, s = ops.block_forward(x, spec, t, rs1, rs2, save=True, plan1=plan1, plan2=plan2)
        fwd_names, F = rec.take()
        dx0, grads = ops.block_backward(x, s, spec, t, t, dy, rs1, rs2, plan1, plan2)
        bwd_names, Bw = rec.take()
    torch.cuda.synchronize()

    st = Stages(cfg)
    ones = torch.ones(M, dtype=torch.bool, device="cuda")
    # rows a plan may leave zero or unwritten in a branch's bf16 activations: the rows its factor drops
    live1 = (rs1 != 0) if plan1 is not None else ones
    live2 = (rs2 != 0) if plan2 is not None else ones
    # the clips the attention branch keeps: the forward skips the others only with a plan (its rows are then 0); their
    # gradient rows are 0 either way
    clips1 = [True] * B if rs1 is None else [bool(rs1[b * n] != 0) for b in range(B)]
    fwd_clips1 = clips1 if plan1 is not None else [True] * B
    z = lambda k: torch.zeros(k, dtype=torch.float64, device="cuda")  # noqa: E731  (an accumulator starting at 0)

    # ---- forward
    gemms, norms = list(F["gemm"]), list(F["norm_fwd"])
    c = norms.pop(0)
    n1, rstd1 = c.ret[0], c.ret[2]
    ref = rr.norm_fwd(x, t.n1w, eps=spec.eps1)
    st.elem("n1", "row_y", n1, ref["y"])
    st.elem("rstd1", "row_rstd", rstd1, ref["rstd"])

    c = gemms.pop(0)
    qkv = c.ret
    st.elem("qkv", "gemm_bf16", qkv, gemm_ref(n1, t.qkvw, bias=t.qkvb)[0], live1)

    q_in, k_in, v_in = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    rq = rk = None
    if cfg.qk:
        if D <= 1536:
            c = F["rmsnorm_pair_fwd"][0]
            qn, kn, rq, rk = c.after["out"][:, :D], c.after["out"][:, D:2 * D], c.ret[:, 0], c.ret[:, 1]
        else:
            cq, ck = norms.pop(0), norms.pop(0)
            qn, kn, rq, rk = cq.ret[0], ck.ret[0], cq.ret[2], ck.ret[2]
        for nm, got, r, src, w in (("qn", qn, rq, q_in, t.qnw), ("kn", kn, rk, k_in, t.knw)):
            ref = rr.norm_fwd(src, w)
            st.elem(nm, "row_y", got, ref["y"])
            st.elem("r" + nm[0], "row_rstd", r, ref["rstd"])
        q_in, k_in = qn, kn

    c = F["attn_fwd"][0]
    a, lse = c.ret
    o_ref, lse_ref = attn_ref_fwd(q_in, k_in, v_in, B, n, H, d, scale)
    st.attn("a", "attn_o", a, o_ref, fwd_clips1)
    st.lse("lse", lse, lse_ref, torch.tensor(fwd_clips1, device="cuda"))

    c = gemms.pop(0)
    x1 = c.ret
    refs = gemm_ref(a, t.projw, epi=EPI_RESID, bias=t.projb, gamma=t.g1, aux=x, rowscale=rs1,
                    out1=c.after.get("out1"))
    st.elem("x1", "gemm_resid", x1, refs[0])
    y1 = None
    if cfg.ls:
        y1 = c.after["out1"]
        st.elem("y1", "gemm_resid_y", y1, refs[1], live1)

    c = norms.pop(0)
    n2, rstd2 = c.ret[0], c.ret[2]
    ref = rr.norm_fwd(x1, t.n2w, eps=spec.eps2)
    st.elem("n2", "row_y", n2, ref["y"])
    st.elem("rstd2", "row_rstd", rstd2, ref["rstd"])

    c = gemms.pop(0)
    g, h = c.ret, c.after["out1"]
    refs = gemm_ref(n2, t.fc1w, epi=EPI_BIAS_GELU, flags=flags, bias=t.fc1b, out1=h)
    st.elem("g", "gemm_gelu", g, refs[0], live2)
    st.elem("h (GELU')", "gemm_gelu_d", h, refs[1], live2)

    c = gemms.pop(0)
    refs = gemm_ref(g, t.fc2w, epi=EPI_RESID, bias=t.fc2b, gamma=t.g2, aux=x1, rowscale=rs2, out1=c.after.get("out1"))
    st.elem("x2", "gemm_resid", c.ret, refs[0])
    st.exact("x2 returned", x2, c.ret)
    y2 = None
    if cfg.ls:
        y2 = c.after["out1"]
        st.elem("y2", "gemm_resid_y", y2, refs[1], live2)

    # ---- backward
    gemms, norms, lss = list(Bw["gemm"]), list(Bw["norm_bwd"]), list(Bw["layerscale_bwd"])
    cols = list(Bw["colsum"])
    c = lss.pop(0)
    dy2 = c.ret
    ref = rr.layerscale_bwd(dy, y2, t.g2, z(D) if cfg.ls else None, z(D), rowscale=rs2)
    st.elem("dy2", "row_dx16", dy2, ref["dy"])
    st.elem("fc2b sum", "row_pgrad", c.after["dcolsum"], ref["dcolsum"])
    if cfg.ls:
        st.elem("g2 sum", "row_pgrad", c.after["dgamma"], ref["dgamma"])

    c = gemms.pop(0)
    st.elem("dfc2w", "gemm_bf16", c.ret, gemm_ref(dy2, g, a_t=True, b_t=True)[0])
    c = gemms.pop(0)
    dh = c.ret
    st.elem("dh", "gemm_gelu_bwd", dh, gemm_ref(dy2, t.fc2w, b_t=True, epi=EPI_GELU_BWD, flags=flags, aux=h)[0])
    c = cols.pop(0)
    st.elem("fc1b sum", "row_pgrad", c.after["out"], rr.colsum(dh)["out"])
    c = gemms.pop(0)
    st.elem("dfc1w", "gemm_bf16", c.ret, gemm_ref(dh, n2, a_t=True, b_t=True)[0])
    c = gemms.pop(0)
    dn2 = c.ret
    st.elem("dn2", "gemm_bf16", dn2, gemm_ref(dh, t.fc1w, b_t=True)[0])

    if fused:
        c = Bw["rmsnorm_bwd_layerscale"][0]
        dx1, dy1 = c.ret
        ref = rr.rmsnorm_bwd_layerscale(dn2, x1, t.n2w, rstd2, dy, y1, t.g1, z(D), z(D), z(D), rowscale=rs1)
        st.elem("dx1 (fused)", "row_dx32", dx1, ref["dx"])
        st.elem("dy1 (fused)", "row_dx16", dy1, ref["dyb"])
        st.elem("n2w sum (fused)", "row_pgrad", c.after["dweight"], ref["dweight"])
        st.elem("g1 sum (fused)", "row_pgrad", c.after["dgamma"], ref["dgamma"])
        st.elem("projb sum (fused)", "row_pgrad", c.after["dcolsum"], ref["dcolsum"])
    else:
        c = norms.pop(0)
        dx1 = c.ret
        ref = rr.norm_bwd(dn2, x1, t.n2w, None, rstd2, dx_in=dy, dweight=z(D))
        st.elem("dx1", "row_dx32", dx1, ref["dx"])
        st.elem("n2w sum", "row_pgrad", c.after["dweight"], ref["dweight"])
        c = lss.pop(0)
        dy1 = c.ret
        ref = rr.layerscale_bwd(dx1, y1, t.g1, z(D) if cfg.ls else None, z(D), rowscale=rs1)
        st.elem("dy1", "row_dx16", dy1, ref["dy"])
        st.elem("projb sum", "row_pgrad", c.after["dcolsum"], ref["dcolsum"])
        if cfg.ls:
            st.elem("g1 sum", "row_pgrad", c.after["dgamma"], ref["dgamma"])

    c = gemms.pop(0)
    st.elem("dprojw", "gemm_bf16", c.ret, gemm_ref(dy1, a, a_t=True, b_t=True)[0])
    c = gemms.pop(0)
    da = c.ret
    st.elem("da", "gemm_bf16", da, gemm_ref(dy1, t.projw, b_t=True)[0])

    c = Bw["attn_bwd"][0]
    dq, dk, dv = c.after["dq"], c.after["dk"], c.after["dv"]
    for nm, got, r in zip(("dq", "dk", "dv"), (dq, dk, dv), attn_ref_bwd(q_in, k_in, v_in, da, B, n, H, d, scale)):
        st.attn(nm, "attn_" + nm, got, r, clips1)

    if cfg.qk:
        if D <= 1536:
            c = Bw["rmsnorm_pair_bwd"][0]
            dq_f, dk_f = c.after["dqk"][:, :D], c.after["dqk"][:, D:2 * D]
            dqw, dkw = c.after["dw0"], c.after["dw1"]
        else:
            cq, ck = norms.pop(0), norms.pop(0)
            dq_f, dk_f, dqw, dkw = cq.ret, ck.ret, cq.after["dweight"], ck.after["dweight"]
        for nm, got, gw, dgot, src, w, r in (("q", dq_f, dqw, dq, qkv[:, :D], t.qnw, rq),
                                             ("k", dk_f, dkw, dk, qkv[:, D:2 * D], t.knw, rk)):
            ref = rr.norm_bwd(dgot, src, w, None, r, dweight=z(D))
            st.elem(f"d{nm} (after the {nm}-norm backward)", "row_dx16", got, ref["dx"])
            st.elem(f"{nm}nw sum", "row_pgrad", gw, ref["dweight"])
        dq, dk = dq_f, dk_f
    dqkv = torch.cat([dq, dk, dv], 1)

    c = gemms.pop(0)
    st.elem("dqkvw", "gemm_bf16", c.ret, gemm_ref(dqkv, n1, a_t=True, b_t=True)[0])
    if cfg.qkv_bias:
        c = cols.pop(0)
        st.elem("qkvb sum", "row_pgrad", c.after["out"], rr.colsum(dqkv)["out"])
    c = gemms.pop(0)
    dn1 = c.ret
    st.elem("dn1", "gemm_bf16", dn1, gemm_ref(dqkv, t.qkvw, b_t=True)[0])
    c = norms.pop(0)
    ref = rr.norm_bwd(dn1, x, t.n1w, None, rstd1, dx_in=dx1, dweight=z(D))
    st.elem("dx0", "row_dx32", c.ret, ref["dx"])
    st.elem("n1w sum", "row_pgrad", c.after["dweight"], ref["dweight"])
    st.exact("dx0 returned", dx0, c.ret)

    # the call sequence: which of the host code's paths ran
    want_f, want_b = _expected_calls(cfg, fused)
    st.res["forward calls"] = (0.0 if fwd_names == want_f else math.inf, 0.0, f"{fwd_names} != {want_f}")
    st.res["backward calls"] = (0.0 if bwd_names == want_b else math.inf, 0.0, f"{bwd_names} != {want_b}")
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_rmsnorm_block_calls_match_float64(cuda_lib, monkeypatch, name):
    bad = _run_calls(name, monkeypatch).failures()
    assert not bad, "\n".join(bad)


# ---------------------------------------------------------------- end to end
def _train(blk, cfg, x, dy, rs1, rs2, plans):
    """forward_stream + backward: (y, dx, {name: grad})."""
    for p in blk.parameters():
        p.grad = None
    xs = x.clone().requires_grad_(True)
    y = blk.forward_stream(xs, cfg.B, cfg.n, rowscale=None if rs1 is None else (rs1, rs2), plans=plans)
    y.backward(dy)
    return y.detach(), xs.grad, {nm: p.grad.clone() for nm, p in blk.named_parameters()}


def _end_to_end(name):
    """Block.forward_stream through BlockFn against oracle.restate.block in float64.  Returns {check: (value, bound,
    where)}."""
    from oracle import restate as R
    cfg = CONFIGS[name]
    blk = _block(cfg)
    x, dy, rs1, rs2, plans = _inputs(cfg)
    y, dx, grads = _train(blk, cfg, x, dy, rs1, rs2, plans)

    B, n, D, H = cfg.B, cfg.n, cfg.D, cfg.H
    p = {"blocks.0." + k: v.detach().double().requires_grad_(True) for k, v in blk.named_parameters()}
    x64 = x.double().reshape(B, n, D).requires_grad_(True)
    dp = None if rs1 is None else (rs1.double().reshape(B, n)[:, 0], rs2.double().reshape(B, n)[:, 0])
    y64 = R.block(p, 0, x64, H, "tanh" if cfg.tanh else "none", drop_path=dp, qk_norm=cfg.qk)
    y64.backward(dy.double().reshape(B, n, D))

    res = {}
    rowinfo = lambda m: f"row {m} (clip {m // n}, token {m % n})"  # noqa: E731
    branch, branch64 = y - x, (y64 - x64).reshape(B * n, D).detach()
    dbr, dbr64 = dx - dy, x64.grad.reshape(B * n, D) - dy.double()
    res["branch"] = (rel(branch, branch64), 1e-2, "tensor")
    res["dx"] = (rel(dbr, dbr64), 1e-2, "tensor")
    e, m = worst_slice(slice_errors(branch, branch64, B * n))
    res["branch_row"] = (e, LOCAL["branch_row"], rowinfo(m))
    e, m = worst_slice(slice_errors(dbr, dbr64, B * n))
    res["dx_row"] = (e, LOCAL["dx_row"], rowinfo(m))
    for k, gr in grads.items():
        ref = p["blocks.0." + k].grad
        res["d " + k] = (rel(gr, ref), 3e-2, "tensor")
        if gr.dim() == 2:
            e, o = worst_slice(slice_errors(gr, ref, gr.shape[0]))
            res["d " + k + " per channel"] = (e, LOCAL[k], f"output channel {o}")
        elif k in ("attn.q_norm.weight", "attn.k_norm.weight"):
            e, hh = worst_slice(slice_errors(gr, ref, H))
            res["d " + k + " per head"] = (e, LOCAL[k], f"head {hh}")
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_rmsnorm_block_matches_float64(cuda_lib, name):
    res = _end_to_end(name)
    bad = [f"{k}: {e:.3g} > {b:.3g} at {w}" for k, (e, b, w) in res.items() if not e <= b]
    assert not bad, "\n".join(bad)


# ---------------------------------------------------------------- bit relations
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_rmsnorm_block_bit_relations(cuda_lib, name):
    """Checkpointed and saved blocks: the same output, input gradient and parameter gradients, bit for bit (the recompute
    runs block_forward(save=True) as the saved block did; the checkpointed forward's save=False writes the same x2).
    forward_infer (no grad, save=False, no plans) gives the training forward's output bits."""
    cfg = CONFIGS[name]
    blk = _block(cfg)
    x, dy, rs1, rs2, plans = _inputs(cfg)
    runs = {}
    for cp in (False, True):
        blk.with_cp = cp
        runs[cp] = _train(blk, cfg, x, dy, rs1, rs2, plans)
    (y0, dx0, g0), (y1, dx1, g1) = runs[False], runs[True]
    bad = [k for k, a, b in (("y", y0, y1), ("dx", dx0, dx1)) if not torch.equal(a, b)]
    bad += ["d " + k for k in g0 if not torch.equal(g0[k], g1[k])]
    yi = blk.forward_infer(x, cfg.B, cfg.n, (rs1, rs2))
    if not torch.equal(yi, y0):
        bad.append("forward_infer y")
    assert not bad, f"differ in bits: {bad}"
