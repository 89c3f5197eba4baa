"""The FP8 mode of modules.Block (modules.set_fp8) at the block_cfg2 size: D = 1408, 16 heads of 88, hidden 6144,
B = 2 clips of n = 417 tokens (gpu).

Bounds, from the formats' unit roundoff (round to nearest: u = 2^-4 for E4M3, 2^-3 for E5M2).  A GEMM whose two
operands are each rounded with relative error at most u_a and u_b has a relative error of at most u_a + u_b per
product, and its Frobenius relative error stays below that.  So, relative to the bf16 block:
  - the output: its branches come from E4M3 x E4M3 GEMMs: 2 u(E4M3) = 0.125;
  - dx and every parameter gradient: the input gradients pass through E5M2 x E4M3 GEMMs, and the weight gradients read
    activations of the FP8 forward: 2 (u(E5M2) + u(E4M3)) = 0.375.
The measured values are far below (DESIGN.md 4.1, FP8); the bounds catch a wrong scale, format or operand, which is
off by factors, not by percent.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
U_E4M3, U_E5M2 = 2.0 ** -4, 2.0 ** -3
OUT_BOUND = 2 * U_E4M3
GRAD_BOUND = 2 * (U_E5M2 + U_E4M3)


def _rel(a, b):
    a = a.detach().double(); b = b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _block(with_cp=False):
    from internvideo_b200 import modules as M
    from oracle.make_golden import block_cfg2_inputs
    z = np.load(GOLD / "block_cfg2.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd, x, dy = block_cfg2_inputs(cfg)
    D, H, B, n = cfg["dim"], cfg["num_heads"], cfg["B"], cfg["n"]
    blk = M.Block(D, H, cfg["mlp_ratio"], init_values=cfg["init_values"], qk_normalization=True, with_cp=with_cp)
    blk.load_state_dict(sd, strict=True)
    blk = blk.bfloat16().cuda()
    return blk, x.reshape(B * n, D).cuda(), dy.reshape(B * n, D).cuda(), B, n


def _run(blk, x, dy, B, n):
    for p in blk.parameters():
        p.grad = None
    xs = x.clone().requires_grad_(True)
    y = blk.forward_stream(xs, B, n)
    y.backward(dy)
    return y.detach(), xs.grad, {k: p.grad.clone() for k, p in blk.named_parameters()}


def test_fp8_block_within_roundoff_bounds_of_bf16(cuda_lib):
    from internvideo_b200.modules import set_fp8
    blk, x, dy, B, n = _block()
    y0, dx0, g0 = _run(blk, x, dy, B, n)
    assert set_fp8(blk, True) == 1
    y1, dx1, g1 = _run(blk, x, dy, B, n)
    r = {"y": _rel(y1 - x, y0 - x), "dx": _rel(dx1 - dy, dx0 - dy)}   # the branches' share: the residual is exact
    r.update({k: _rel(g1[k], g0[k]) for k in g0})
    print("fp8 vs bf16 relative errors:", {k: round(v, 4) for k, v in r.items()})
    assert r["y"] <= OUT_BOUND, r
    bad = {k: v for k, v in r.items() if k != "y" and v > GRAD_BOUND}
    assert not bad, bad
    # not the bf16 bits: the FP8 path ran
    assert not torch.equal(y1, y0)


def test_checkpointed_fp8_block_is_bit_identical(cuda_lib):
    from internvideo_b200.modules import set_fp8
    res = []
    for with_cp in (False, True):
        blk, x, dy, B, n = _block(with_cp)
        set_fp8(blk, True)
        res.append(_run(blk, x, dy, B, n))
    (y0, dx0, g0), (y1, dx1, g1) = res
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_set_fp8_off_restores_bf16_bits(cuda_lib):
    from internvideo_b200.modules import set_fp8
    blk, x, dy, B, n = _block()
    y0, dx0, g0 = _run(blk, x, dy, B, n)
    set_fp8(blk, True)
    _run(blk, x, dy, B, n)
    assert set_fp8(blk, False) == 1
    y1, dx1, g1 = _run(blk, x, dy, B, n)
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_no_grad_forward_uses_fp8_and_matches_training_forward(cuda_lib):
    """Block.forward_infer (frozen towers) runs the FP8 forward: the same bits as the training forward."""
    from internvideo_b200.modules import set_fp8
    blk, x, dy, B, n = _block()
    set_fp8(blk, True)
    y_train, _, _ = _run(blk, x, dy, B, n)
    with torch.no_grad():
        y_infer = blk.forward_stream(x.clone(), B, n)
    assert torch.equal(y_infer, y_train)
