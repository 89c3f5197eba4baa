"""DropPath skipping in per-token FP8 and in attention, on the H100.  Each planned call against the same call without a
plan: ivb_gemm_fp8_plan's live rows equal ivb_gemm_fp8's and its dead tiles hold the dead-tile table (ivb200.h);
ivb_attn_fwd_plan / ivb_attn_bwd_plan give the kept clips ivb_attn_fwd / ivb_attn_bwd's bits and the dropped clips
zeros; a training block and a model step give the same results with the skipping as without.  Equality is
torch.equal: the same values, where a zero may come out as +0 instead of -0."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import droppath_ref as ref
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import modules as M
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"

B = 32
DRAWS = {
    "none_dropped": np.ones(B, bool),
    "all_dropped": np.zeros(B, bool),
    "random": np.random.default_rng(3).random(B) >= 0.25,
    "alternating": np.arange(B) % 2 == 0,
}


def _rows(keep, n):
    return torch.from_numpy(ref.clip_rows(keep, n)).cuda()


def _m_plan(rs):
    return ops._branch_plans(ops.droppath_plan(rs[None].contiguous())[0], rs.numel(), ops.FP8_TOKEN)[0]


def _dead_rows(keep, n):
    order, live, _ = ref.plan(ref.clip_rows(keep, n))
    dead = torch.zeros(keep.size * n, dtype=torch.bool, device="cuda")
    for t in order[live:]:
        dead[128 * t:128 * t + 128] = True
    return dead


def _case(epi, Mr, N, K, g):
    """Per-token FP8 operands (row-scaled A, per-channel B) and the epilogue arguments of one GEMM."""
    a = torch.randn((Mr, K), generator=g, device="cuda").to(torch.bfloat16)
    w = (0.1 * torch.randn((N, K), generator=g, device="cuda")).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device="cuda").to(torch.bfloat16)
    ops_ = (*ll.fp8_quantize_rows(a), *ll.fp8_quantize_rows(w))
    if epi == "bf16":
        return ops_, dict(bias=bias), ["out0"]
    if epi == "bias_gelu_save":
        return ops_, dict(epi=ll.EPI_BIAS_GELU, bias=bias, flags=ll.FLAG_GELU_SAVE_GRAD, out1=True), ["out0", "out1"]
    if epi == "resid":
        gamma = (1e-2 * torch.randn(N, generator=g, device="cuda")).to(torch.bfloat16)
        aux = torch.randn((Mr, N), generator=g, device="cuda")
        return ops_, dict(epi=ll.EPI_RESID, bias=bias, gamma=gamma, aux=aux, out1=True), ["out0", "out1"]
    aux = torch.rand((Mr, N), generator=g, device="cuda").to(torch.bfloat16)
    return ops_, dict(epi=ll.EPI_GELU_BWD, flags=ll.FLAG_GELU_SAVE_GRAD, aux=aux), ["out0"]


def _check_m_plan(epi, n, N, K, flags, tile_n, draws, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Mr = B * n
    for draw in draws:
        keep = DRAWS[draw]
        rs = _rows(keep, n)
        (qa, sa, qb, sb), kw, outs = _case(epi, Mr, N, K, g)
        kw["flags"] = kw.get("flags", 0) | flags
        if kw.get("epi") == ll.EPI_RESID:
            kw["rowscale"] = rs
        res = []
        for plan, tn in ((None, tile_n), (_m_plan(rs), 128 if tile_n == 192 else tile_n)):
            o1 = torch.full((Mr, N), float("nan"), device="cuda").to(torch.bfloat16) if kw.get("out1") else None
            o0 = ll._gemm_fp8_plan(qa, sa, qb, sb, plan, tile_n=tn, **{**kw, "out1": o1})
            res.append({"out0": o0, "out1": o1})
        dead = _dead_rows(keep, n)
        for o in outs:
            full, planned = res[0][o], res[1][o]
            assert torch.equal(planned[~dead], full[~dead]), (draw, o)
            want = kw["aux"][dead] if (kw.get("epi") == ll.EPI_RESID and o == "out0") else torch.zeros_like(planned[dead])
            assert torch.equal(planned[dead], want), (draw, o)


# the eight block GEMMs of cfg-2 (n = 417: M = 13 344), each with the epilogue the block gives it
CFG2 = [("qkv", 4224, 1408, "bf16"), ("proj", 1408, 1408, "resid"), ("fc1", 6144, 1408, "bias_gelu_save"),
        ("fc2", 1408, 6144, "resid"), ("dh", 6144, 1408, "gelu_bwd_save"), ("dn2", 1408, 6144, "bf16"),
        ("da", 1408, 1408, "bf16"), ("dn1", 1408, 4224, "bf16")]


@pytest.mark.parametrize("name, N, K, epi", CFG2, ids=[c[0] for c in CFG2])
def test_fp8_m_plan_cfg2_shapes(cuda_lib, name, N, K, epi):
    """The library's default kernel at the step's shapes, with a random, an all-live and an all-dead draw."""
    _check_m_plan(epi, 417, N, K, 0, 0, ["random", "none_dropped", "all_dropped"], seed=1)


EPILOGUES = ["bf16", "resid", "bias_gelu_save", "gelu_bwd_save"]
# ping-pong; the cooperative kernel at the width the library picks, at 128, and forced to 192 without a plan (a plan
# runs it at 128)
FORMS = [(ll.FLAG_PINGPONG, 0), (ll.FLAG_1CTA, 0), (ll.FLAG_1CTA, 128), (ll.FLAG_1CTA, 192)]


@pytest.mark.parametrize("form", FORMS, ids=["pingpong", "coop", "coop128", "coop192"])
@pytest.mark.parametrize("epi", EPILOGUES)
def test_fp8_m_plan_forms_and_tails(cuda_lib, epi, form):
    """Both kernel forms at a row tail (32 clips of 65 rows: M = 2080, 32 rows into the last tile) and a column tail
    (N = 1416), with every draw."""
    _check_m_plan(epi, 65, 1416, 256, form[0], form[1], list(DRAWS), seed=7)


# ---- attention
@pytest.mark.parametrize("n", [417, 130])
@pytest.mark.parametrize("d", [64, 88, 128])
def test_attn_plan(cuda_lib, d, n):
    Bc, H = 6, 3
    D = H * d
    g = torch.Generator(device="cuda").manual_seed(d + n)
    qkv = torch.randn((Bc * n, 3 * D), generator=g, device="cuda").to(torch.bfloat16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    dout = torch.randn((Bc * n, D), generator=g, device="cuda").to(torch.bfloat16)
    scale = d ** -0.5
    for keep in (np.ones(Bc, bool), np.array([1, 0, 1, 1, 0, 0], bool), np.zeros(Bc, bool)):
        res = []
        for rs in (None, _rows(keep, n)):
            out, lse = ll.attn_fwd(q, k, v, Bc, n, H, d, scale, rowscale=rs)
            dqkv = torch.full((Bc * n, 3 * D), float("nan"), device="cuda").to(torch.bfloat16)
            ll.attn_bwd(q, k, v, out, dout, lse, Bc, n, H, d, scale, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:],
                        rowscale=rs)
            res.append((out.reshape(Bc, n, D), lse, dqkv.reshape(Bc, n, 3 * D)))
        kept = torch.from_numpy(keep).cuda()
        (o0, l0, g0), (o1, l1, g1) = res
        assert torch.equal(o1[kept], o0[kept]) and torch.equal(l1[kept], l0[kept]) and torch.equal(g1[kept], g0[kept])
        assert torch.all(o1[~kept] == 0) and torch.all(g1[~kept] == 0)
        assert torch.isfinite(l1[~kept]).all()


# ---- block and model
def _block_run(prec, checkpoint, plans_on, keep1, keep2, seed=3):
    """The block_cfg2 fixture's block (D = 1408, 16 heads of 88, n = 417, B = 2), trained on one step's draw."""
    cfg = json.loads(bytes(np.load(GOLD / "block_cfg2.npz")["cfg"]).decode())
    D, H, Bc, n = cfg["dim"], cfg["num_heads"], cfg["B"], cfg["n"]
    torch.manual_seed(seed)
    blk = M.Block(D, H, cfg["mlp_ratio"], init_values=1e-5, qk_normalization=True, use_fused_mlp=True,
                  drop_path=0.1, with_cp=checkpoint).bfloat16().cuda()
    if prec == "token":
        M.set_fp8(blk, True, scaling="token")
    x = torch.randn(Bc * n, D, device="cuda").requires_grad_(True)
    rs1, rs2 = _rows(keep1, n), _rows(keep2, n)
    plans = tuple(ops.droppath_plan(torch.stack([rs1, rs2]))) if plans_on else None
    y = blk.forward_stream(x, Bc, n, rowscale=(rs1, rs2), plans=plans)
    y.backward(torch.randn(y.shape, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda"))
    return y.detach(), x.grad.clone(), {nm: p.grad.clone() for nm, p in blk.named_parameters()}


@pytest.mark.parametrize("prec, checkpoint", [("token", False), ("token", True), ("bf16", False)])
@pytest.mark.parametrize("keep1, keep2", [((0, 1), (1, 0)), ((0, 0), (1, 1)), ((1, 1), (0, 1))])
def test_block_cfg2_planned_equals_unplanned(cuda_lib, prec, checkpoint, keep1, keep2):
    """A training block at the block_cfg2 size with DropPath factors that drop clips: x2, dx and every parameter
    gradient are the same with the plans (GEMM tiles, wgrad k-blocks, attention) as without."""
    keep1, keep2 = np.array(keep1, bool), np.array(keep2, bool)
    y0, dx0, g0 = _block_run(prec, checkpoint, False, keep1, keep2)
    y1, dx1, g1 = _block_run(prec, checkpoint, True, keep1, keep2)
    assert torch.equal(y1, y0)
    assert torch.equal(dx1, dx0)
    for nm in g0:
        assert torch.equal(g1[nm], g0[nm]), nm


def _dp_step(scaling, skip, graph):
    """One engine step of the pretrain_dp fixture (stochastic depth with a fully dropped sample) in FP8 `scaling`:
    (flat parameters, flat gradients) after it, eagerly or as the replay of a captured step."""
    from internvideo_b200.engine import GraphedStep, PretrainEngine
    z = np.load(GOLD / "pretrain_dp.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    x = torch.from_numpy(z["x"]).cuda().to(torch.bfloat16)
    mask = torch.from_numpy(z["mask"]).cuda()
    tg = [torch.from_numpy(z[k]).cuda() for k in ("tgt_clip", "tgt_final", "tgt_mae")]
    fac = torch.from_numpy(z["drop_path_factors"]).cuda()
    n_vis = int((~mask[0]).sum())           # read before capture: the step itself reads nothing back
    model = M.PretrainInternVideo2(use_flash_attn=True, use_fused_rmsnorm=True, use_fused_mlp=True, **cfg)
    model.load_state_dict(sd, strict=True)
    model = model.bfloat16().cuda().train()
    M.set_fp8(model, True, scaling=scaling)
    M.set_droppath_skip(model, skip)
    eng = PretrainEngine(model, clip_grad=3.0)

    def step(v, m):
        eng.zero_grad()
        ls = model.forward_loss(v, m, tg[0], tg[1], tg[2], n_visible=n_vis, drop_path_factors=fac)
        loss = ls[0] + ls[1] + ls[2]
        loss.backward()
        eng.step()
        return loss

    if graph:
        gs = GraphedStep(step, [x, mask], warmup=1)
        gs(x, mask)
    else:
        step(x, mask)
    torch.cuda.synchronize()
    return eng.flat_param.clone(), eng.flat_grad.clone()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pretrain_dp_step_fp8_token_skip_on_equals_off(cuda_lib, graph):
    p0, g0 = _dp_step("token", False, graph)
    p1, g1 = _dp_step("token", True, graph)
    assert torch.equal(g1, g0)
    assert torch.equal(p1, p0)


def test_fp8_tensor_mode_runs_planless(cuda_lib, monkeypatch):
    """Per-tensor FP8 gets no plan: no planned GEMM or attention call in its step, whatever the skip setting."""
    called = []
    for fn in ("_gemm_fp8_plan", "attn_fwd", "attn_bwd", "gemm"):
        orig = getattr(ll, fn)

        def spy(*a, _orig=orig, _fn=fn, **kw):
            planned = kw.get("m_plan") is not None or kw.get("k_plan") is not None
            planned |= _fn == "_gemm_fp8_plan" and a[4] is not None          # m_plan, the fifth argument
            if planned or (_fn.startswith("attn") and kw.get("rowscale") is not None):
                called.append(_fn)
            return _orig(*a, **kw)
        monkeypatch.setattr(ll, fn, spy)
    _dp_step("tensor", True, False)
    assert not called, called
    _dp_step("token", True, False)
    assert {"_gemm_fp8_plan", "attn_fwd", "attn_bwd", "gemm"} <= set(called)
