"""The FP8 training modes of modules.Block (modules.set_fp8) on the H100 (gpu).  Every test takes the mode as an input
from MODES, which holds set_fp8's own arguments.

- The block at the block_cfg2 size (D = 1408, 16 heads of 88, hidden 6144, B = 2 clips of n = 417 tokens) against the
  bf16 block, each mode by its own criterion; a checkpointed block, the no-grad forward and switching FP8 off give the
  bits they should; with DropPath factors that drop clips, the DropPath plans change no bit.
- A pretrain_dp step (stochastic depth with a fully dropped sample) gives the same results with DropPath skipping as
  without, eagerly and as the replay of a captured step; the per-tensor mode runs no plan.
- The pretrain_tiny model through engine.PretrainEngine: 100 steps on one fixed, seeded batch drop the loss at least
  90 % as far as bf16 does; the gradient sink (wgrad GEMMs accumulating straight into the engine's flat gradient) gives
  autograd's flat gradient to the tolerance the bf16 sink test uses; a batch with an Inf makes the step non-finite (the
  FP8 casts turn it into a NaN scale), so the engine skips it and the parameters stay unchanged; the step captured in
  engine.GraphedStep replays with the eager step's loss.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import droppath_ref as ref
from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import modules as M
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
MODES = {"tensor": dict(scaling="tensor"), "token": dict(scaling="token"),
         "token_wgrad": dict(scaling="token", wgrad=True)}

# Relative Frobenius errors against the bf16 block at block_cfg2.  Unit roundoff, round to nearest: u = 2^-4 for E4M3,
# 2^-3 for E5M2.  A GEMM whose two operands are each rounded with relative error at most u_a and u_b has a relative
# error of at most u_a + u_b per product, and its Frobenius relative error stays below that.
U_E4M3, U_E5M2 = 2.0 ** -4, 2.0 ** -3
# tensor: the output's branches come from E4M3 x E4M3 GEMMs: 2 u(E4M3) = 0.125; dx and every parameter gradient pass
# through E5M2 x E4M3 input-gradient GEMMs, and the weight gradients read activations of the FP8 forward:
# 2 (u(E5M2) + u(E4M3)) = 0.375.  The measured values are far below (DESIGN.md 4.1, FP8); the bounds catch a wrong
# scale, format or operand, which is off by factors, not by percent.
OUT_BOUND = 2 * U_E4M3
GRAD_BOUND = 2 * (U_E5M2 + U_E4M3)
# token: the derived bounds are output 2u = 0.125 (E4M3 x E4M3 GEMMs); dx and parameter gradients 4u = 0.25 (E4M3
# gradients x E4M3 weights, and weight gradients reading the FP8 forward's activations).  Each limit is the smaller of
# its derived bound and 1.5 times the value measured on an H100 80GB HBM3 (MEASURED; the computation is deterministic).
# Per-tensor FP8 on the same inputs measured y 0.0546, dx 0.0894, gradients up to 0.104.
MEASURED = {"y": 0.0546, "dx": 0.0623, "norm1.weight": 0.0849, "attn.qkv.weight": 0.0770, "attn.proj.weight": 0.0643,
            "attn.proj.bias": 0.0081, "attn.q_norm.weight": 0.0902, "attn.k_norm.weight": 0.0902, "ls1.gamma": 0.0708,
            "norm2.weight": 0.0602, "mlp.fc1.weight": 0.0489, "mlp.fc1.bias": 0.0490, "mlp.fc2.weight": 0.0390,
            "mlp.fc2.bias": 0.0, "ls2.gamma": 0.0547}
LIMITS = {k: min(2 * U_E4M3 if k == "y" else 4 * U_E4M3, 1.5 * v) for k, v in MEASURED.items()}
# token_wgrad: everything but the four weight gradients has the token mode's bits.  The weight gradients' errors were
# measured on an H100 80GB HBM3 (the computation is deterministic); each is held to 0.15 and to twice its measured
# value.
WEIGHTS = ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight")
WGRAD_MEASURED = {"attn.qkv.weight": 0.0850, "attn.proj.weight": 0.0744, "mlp.fc1.weight": 0.0617,
                  "mlp.fc2.weight": 0.0542}


def _rel(a, b):
    a = a.detach().double(); b = b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _assert_same(a, b):
    (y1, dx1, g1), (y0, dx0, g0) = a, b
    assert torch.equal(y1, y0) and torch.equal(dx1, dx0)
    for k in g0:
        assert torch.equal(g1[k], g0[k]), k


# ------------------------------------------------------------------------------------------------ the block
@pytest.fixture(scope="module")
def cfg2():
    """block_cfg2's configuration and state dict, and its x and dy as [B n, D] on the device."""
    from oracle.make_golden import block_cfg2_inputs
    cfg = json.loads(bytes(np.load(GOLD / "block_cfg2.npz")["cfg"]).decode())
    sd, x, dy = block_cfg2_inputs(cfg)
    D, B, n = cfg["dim"], cfg["B"], cfg["n"]
    return cfg, sd, x.reshape(B * n, D).cuda(), dy.reshape(B * n, D).cuda()


@pytest.fixture(scope="module")
def bf16_block(cfg2):
    """(y, dx, gradients) of the bf16 block."""
    return _run(_block(cfg2, None), cfg2)


def _block(cfg2, mode, with_cp=False):
    cfg, sd = cfg2[:2]
    blk = M.Block(cfg["dim"], cfg["num_heads"], cfg["mlp_ratio"], init_values=cfg["init_values"],
                  qk_normalization=True, with_cp=with_cp)
    blk.load_state_dict(sd, strict=True)
    blk = blk.bfloat16().cuda()
    if mode is not None:
        assert M.set_fp8(blk, True, **MODES[mode]) == 1
    return blk


def _run(blk, cfg2):
    cfg, _, x, dy = cfg2
    for p in blk.parameters():
        p.grad = None
    xs = x.clone().requires_grad_(True)
    y = blk.forward_stream(xs, cfg["B"], cfg["n"])
    y.backward(dy)
    return y.detach(), xs.grad, {k: p.grad.clone() for k, p in blk.named_parameters()}


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_block_against_bf16(cuda_lib, cfg2, bf16_block, mode):
    x, dy = cfg2[2:]
    y1, dx1, g1 = _run(_block(cfg2, mode), cfg2)
    y0, dx0, g0 = bf16_block
    r = {"y": _rel(y1 - x, y0 - x), "dx": _rel(dx1 - dy, dx0 - dy)}   # the branches' share: the residual is exact
    r.update({k: _rel(g1[k], g0[k]) for k in g0})
    print(f"{mode} FP8 vs bf16 relative errors:", {k: round(v, 4) for k, v in r.items()})
    if mode == "tensor":
        assert r["y"] <= OUT_BOUND, r
        bad = {k: v for k, v in r.items() if k != "y" and v > GRAD_BOUND}
        assert not bad, bad
        assert not torch.equal(y1, y0)     # not the bf16 bits: the FP8 path ran
    elif mode == "token":
        assert set(r) == set(LIMITS), sorted(r)
        bad = {k: (v, LIMITS[k]) for k, v in r.items() if v > LIMITS[k]}
        assert not bad, bad
        assert r["y"] > 0                  # not the bf16 bits: the FP8 path ran
    else:
        yt, dxt, gt = _run(_block(cfg2, "token"), cfg2)
        assert torch.equal(y1, yt) and torch.equal(dx1, dxt)
        for k in gt:
            if k not in WEIGHTS:
                assert torch.equal(g1[k], gt[k]), k
        for k in WEIGHTS:
            assert r[k] > 0 and not torch.equal(g1[k], gt[k]), k       # the FP8 weight gradient ran
            assert r[k] <= 0.15, (k, r[k])
            assert r[k] <= 2 * WGRAD_MEASURED[k], (k, r[k], WGRAD_MEASURED[k])


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_checkpointed_block_is_bit_identical(cuda_lib, cfg2, mode):
    _assert_same(_run(_block(cfg2, mode, with_cp=True), cfg2), _run(_block(cfg2, mode), cfg2))


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_no_grad_forward_matches_training_forward(cuda_lib, cfg2, mode):
    """The no-grad forward (frozen towers) runs the FP8 forward: the same bits as the training forward."""
    cfg, _, x, _ = cfg2
    blk = _block(cfg2, mode)
    y_train, _, _ = _run(blk, cfg2)
    with torch.no_grad():
        y_infer = blk.forward_stream(x.clone(), cfg["B"], cfg["n"])
    assert torch.equal(y_infer, y_train)


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_off_restores_bf16_bits_and_excludes_fp8_inference(cuda_lib, cfg2, bf16_block, mode):
    cfg, _, x, _ = cfg2
    blk = _block(cfg2, mode)
    _run(blk, cfg2)
    with pytest.raises(_lib.IvbError, match="switch that off first"):
        M.set_fp8_inference(blk)
    assert M.set_fp8(blk, False) == 1
    _assert_same(_run(blk, cfg2), bf16_block)
    M.set_fp8_inference(blk)
    M.set_fp8(blk, True, **MODES[mode])
    with pytest.raises(_lib.IvbError, match="both on"), torch.no_grad():
        blk.forward_stream(x.clone(), cfg["B"], cfg["n"])


def _dropped_block(cfg2, mode, checkpoint, plans_on, keep1, keep2, seed=3):
    """The block_cfg2 geometry (B = 2) with random weights, trained on one step's DropPath draw, with or without the
    DropPath plans."""
    cfg = cfg2[0]
    D, H, Bc, n = cfg["dim"], cfg["num_heads"], cfg["B"], cfg["n"]
    torch.manual_seed(seed)
    blk = M.Block(D, H, cfg["mlp_ratio"], init_values=1e-5, qk_normalization=True, use_fused_mlp=True,
                  drop_path=0.1, with_cp=checkpoint).bfloat16().cuda()
    if mode is not None:
        M.set_fp8(blk, True, **MODES[mode])
    x = torch.randn(Bc * n, D, device="cuda").requires_grad_(True)
    rs1, rs2 = (torch.from_numpy(ref.clip_rows(k, n)).cuda() for k in (keep1, keep2))
    plans = tuple(ops.droppath_plan(torch.stack([rs1, rs2]))) if plans_on else None
    y = blk.forward_stream(x, Bc, n, rowscale=(rs1, rs2), plans=plans)
    y.backward(torch.randn(y.shape, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda"))
    return y.detach(), x.grad.clone(), {nm: p.grad.clone() for nm, p in blk.named_parameters()}


@pytest.mark.parametrize("mode, checkpoint", [("token", False), ("token", True), ("token_wgrad", False),
                                              pytest.param(None, False, id="bf16-False")])
@pytest.mark.parametrize("keep1, keep2", [((0, 1), (1, 0)), ((0, 0), (1, 1)), ((1, 1), (0, 1))])
def test_block_cfg2_planned_equals_unplanned(cuda_lib, cfg2, mode, checkpoint, keep1, keep2):
    """With DropPath factors that drop clips: x2, dx and every parameter gradient are the same with the plans (GEMM
    tiles, wgrad k-blocks, attention) as without."""
    keep1, keep2 = np.array(keep1, bool), np.array(keep2, bool)
    _assert_same(_dropped_block(cfg2, mode, checkpoint, True, keep1, keep2),
                 _dropped_block(cfg2, mode, checkpoint, False, keep1, keep2))


# ------------------------------------------------------------------------------------------------ pretrain_dp
def _dp_step(mode, skip, graph):
    """One engine step of the pretrain_dp fixture (stochastic depth with a fully dropped sample) in FP8 `mode`:
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
    M.set_fp8(model, True, **MODES[mode])
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
@pytest.mark.parametrize("mode", ["token", "token_wgrad"])
def test_pretrain_dp_step_skip_on_equals_off(cuda_lib, mode, graph):
    p0, g0 = _dp_step(mode, False, graph)
    p1, g1 = _dp_step(mode, True, graph)
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


# ------------------------------------------------------------------------------------------------ pretrain_tiny
@pytest.fixture(scope="module")
def tiny():
    """pretrain_tiny's configuration, state dict, x, mask and targets (on the host)."""
    z = np.load(GOLD / "pretrain_tiny.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    return cfg, sd, *(torch.from_numpy(z[k]) for k in ("x", "mask", "tgt_clip", "tgt_final", "tgt_mae"))


@pytest.fixture(scope="module")
def bf16_losses(tiny):
    """The bf16 model's loss over 100 steps."""
    return _train(tiny, None)


def _setup(tiny, mode, direct=True, check_finite=False):
    from internvideo_b200.engine import PretrainEngine
    cfg, sd, x, mask, *tg = tiny
    model = M.PretrainInternVideo2(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False, **cfg)
    model.load_state_dict(sd, strict=True)
    model = model.bfloat16().cuda().train()
    if mode is not None:
        assert M.set_fp8(model, True, **MODES[mode]) > 0
    eng = PretrainEngine(model, lr=1e-3, clip_grad=0.0, direct_grads=direct, check_finite=check_finite)
    return model, eng, x.cuda().to(torch.bfloat16), mask.cuda(), [t.cuda() for t in tg]


def _loss(model, x, mask, tg, n_visible=None):
    lc, lf, lm = model.forward_loss(x, mask, tg[0], tg[1], tg[2], n_visible=n_visible)
    return lc + lf + lm


def _train(tiny, mode, steps=100):
    torch.manual_seed(0)
    model, eng, x, mask, tg = _setup(tiny, mode)
    losses = []
    for _ in range(steps):
        eng.zero_grad()
        loss = _loss(model, x, mask, tg)
        loss.backward()
        eng.step()
        losses.append(float(loss))
    return losses


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_loss_drops_like_bf16(cuda_lib, tiny, bf16_losses, mode):
    bf, f8 = bf16_losses, _train(tiny, mode)
    drop_bf, drop_f8 = bf[0] - bf[-1], f8[0] - f8[-1]
    print(f"loss bf16 {bf[0]:.4f} -> {bf[-1]:.4f}, {mode} fp8 {f8[0]:.4f} -> {f8[-1]:.4f}")
    assert drop_bf > 0
    assert drop_f8 >= 0.9 * drop_bf, (drop_f8, drop_bf)


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_gradient_sink_matches_autograd(cuda_lib, tiny, mode):
    flats = []
    for direct in (False, True):
        torch.manual_seed(0)
        model, eng, x, mask, tg = _setup(tiny, mode, direct=direct)
        eng.zero_grad()
        _loss(model, x, mask, tg).backward()
        flats.append(eng.flat_grad.float().clone())
    rel = float((flats[1] - flats[0]).norm() / flats[0].norm())
    assert float(flats[0].norm()) > 0 and rel < 2e-3, rel


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_step_with_inf_input_is_skipped(cuda_lib, tiny, mode):
    torch.manual_seed(0)
    model, eng, x, mask, tg = _setup(tiny, mode, check_finite=True)
    before = [p.detach().clone() for p in model.parameters()]
    x.fill_(float("inf"))
    eng.zero_grad()
    _loss(model, x, mask, tg).backward()
    eng.step()
    assert float(eng.skipped) == 1.0
    for p, b in zip(model.parameters(), before):
        assert torch.equal(p.detach(), b)


@pytest.mark.parametrize("mode", ["tensor", "token", "token_wgrad"])
def test_step_replays_in_a_cuda_graph(cuda_lib, tiny, mode):
    """The whole FP8 step (forward, backward, AdamW) captured in engine.GraphedStep replays with the eager step's loss.
    Both arms start from the same model and take one warm-up step first.  The loss sums per-block partials with
    atomics, so its last bits may differ between any two runs: 8 fp32 ulps are allowed."""
    from internvideo_b200.engine import GraphedStep
    arms = []
    for _ in range(2):
        torch.manual_seed(0)
        model, eng, x, mask, tg = _setup(tiny, mode)
        n_visible = int(mask.shape[1] - int(mask[0].sum()))    # given, so the captured step reads nothing to the host

        def step(v, model=model, eng=eng, mask=mask, tg=tg, n_visible=n_visible):
            eng.zero_grad()
            loss = _loss(model, v, mask, tg, n_visible)
            loss.backward()
            eng.step()
            return loss
        arms.append((step, x))
    step, x = arms[0]
    step(x)
    loss_eager = float(step(x))
    step, x = arms[1]
    graphed = GraphedStep(step, [x.clone()], warmup=1)
    loss_graph = float(graphed(x)[0])
    torch.cuda.synchronize()
    print(f"{mode} FP8 step: eager loss {loss_eager!r}, graph replay {loss_graph!r}")
    assert loss_eager == loss_eager and abs(loss_graph - loss_eager) <= 8 * 2.0 ** -23 * abs(loss_eager)
