"""Training with the FP8 block mode through engine.PretrainEngine (gpu), on the pretrain_tiny model.

- 100 steps on one fixed, seeded batch with FP8 on and off: the FP8 run's loss drop is at least 90 % of the bf16 run's.
- The gradient sink (wgrad GEMMs accumulating straight into the engine's flat gradient) and autograd accumulation
  give the same flat gradient in FP8 mode, to the tolerance the bf16 sink test uses.
- A batch with an Inf makes the step non-finite: the FP8 casts turn it into a NaN scale, the engine skips the step and
  the parameters stay unchanged.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


def _setup(fp8, direct=True, check_finite=False):
    from internvideo_b200.engine import PretrainEngine
    from internvideo_b200.modules import PretrainInternVideo2, set_fp8
    z = np.load(GOLD / "pretrain_tiny.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    model = PretrainInternVideo2(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False, **cfg)
    model.load_state_dict(sd, strict=True)
    model = model.bfloat16().cuda().train()
    assert set_fp8(model, fp8) > 0
    eng = PretrainEngine(model, lr=1e-3, clip_grad=0.0, direct_grads=direct, check_finite=check_finite)
    x = torch.from_numpy(z["x"]).cuda().to(torch.bfloat16)
    mask = torch.from_numpy(z["mask"]).cuda()
    tg = [torch.from_numpy(z[k]).cuda() for k in ("tgt_clip", "tgt_final", "tgt_mae")]
    return model, eng, x, mask, tg


def _loss(model, x, mask, tg):
    lc, lf, lm = model.forward_loss(x, mask, tg[0], tg[1], tg[2])
    return lc + lf + lm


def _train(fp8, steps=100):
    torch.manual_seed(0)
    model, eng, x, mask, tg = _setup(fp8)
    losses = []
    for _ in range(steps):
        eng.zero_grad()
        loss = _loss(model, x, mask, tg)
        loss.backward()
        eng.step()
        losses.append(float(loss))
    return losses


def test_fp8_training_loss_drops_like_bf16(cuda_lib):
    bf = _train(False)
    f8 = _train(True)
    drop_bf, drop_f8 = bf[0] - bf[-1], f8[0] - f8[-1]
    print(f"loss bf16 {bf[0]:.4f} -> {bf[-1]:.4f}, fp8 {f8[0]:.4f} -> {f8[-1]:.4f}")
    assert drop_bf > 0
    assert drop_f8 >= 0.9 * drop_bf, (drop_f8, drop_bf)


def test_fp8_gradient_sink_matches_autograd(cuda_lib):
    flats = []
    for direct in (False, True):
        torch.manual_seed(0)
        model, eng, x, mask, tg = _setup(True, direct=direct)
        eng.zero_grad()
        _loss(model, x, mask, tg).backward()
        flats.append(eng.flat_grad.float().clone())
    rel = float((flats[1] - flats[0]).norm() / flats[0].norm())
    assert float(flats[0].norm()) > 0 and rel < 2e-3, rel


def test_fp8_step_with_inf_input_is_skipped(cuda_lib):
    torch.manual_seed(0)
    model, eng, x, mask, tg = _setup(True, check_finite=True)
    before = [p.detach().clone() for p in model.parameters()]
    x = x.clone()
    x.fill_(float("inf"))
    eng.zero_grad()
    _loss(model, x, mask, tg).backward()
    eng.step()
    assert float(eng.skipped) == 1.0
    for p, b in zip(model.parameters(), before):
        assert torch.equal(p.detach(), b)
