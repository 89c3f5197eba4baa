"""FP8 inference of the frozen teachers (modules.set_fp8_inference) on the H100 (gpu).

Bounds.  Every GEMM of a switched block reads two E4M3 operands, each rounded with relative error at most
u = 2^-4 per element (per-row and per-channel power-of-two scales keep every element in E4M3's normal range unless it is
below 2^-6 of its row's amax), so each product, and the Frobenius norm of each branch, errs by at most 2u = 0.125
relative to the bf16 block (the bound tests/test_fp8_modes_gpu.py uses).

For the whole teachers: a tap is t = z / |z| of a token's fp32 stream z.  For unit t_bf16,
    |t_fp8 - t_bf16| <= 2 |z_fp8 - z_bf16| / |z_bf16|,
and z is the embedding plus the sum of the blocks' branches, each within 2u of its bf16 value: the per-token bound is
2 * 2u = 0.25 under the assumption that the branches do not cancel in z (then |z| is close to the sum of the parts'
norms); it is not a bound without that assumption.  The student's loss term is 2 - 2<s, t> with unit s, so
|t_fp8 - t_bf16| bounds the change of every loss term.  The pooled feature and the attention map are held to the
branch bound 2u.  Those bounds are far above what the teachers.npz configuration gives on an H100 (taps 0.0145 CLIP /
0.0055 MAE, pooled 0.0061, attention map 0.0022; DESIGN.md 4.1, Frozen towers), so each quantity is also held to about
twice its measured value: the kernels are deterministic and the fixture fixed, so only a change of the FP8 path's
numerics moves these numbers, and a doubling of its error fails.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
U_E4M3 = 2.0 ** -4
BRANCH_BOUND = 2 * U_E4M3
TAP_BOUND = 2 * BRANCH_BOUND
MEASURED_LIMITS = {"clip taps": 0.03, "mae taps": 0.012, "pooled": 0.013, "attn": 0.005}   # about 2x the H100 values


def _rel(a, b):
    a = a.detach().double(); b = b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _ivl_block():
    from internvideo_b200.modules import Block
    torch.manual_seed(0)
    blk = Block(3200, 25, 4, init_values=0.1, qk_normalization=True, use_fused_mlp=True)
    with torch.no_grad():
        for nm, p in blk.named_parameters():
            if "norm" in nm:
                p.copy_(1 + 0.1 * torch.randn_like(p))
    return blk.bfloat16().cuda().eval()


def _mae_block():
    from internvideo_b200.modules import LayerNormB, VideoMAEBlock
    torch.manual_seed(1)
    blk = VideoMAEBlock(1408, 16, 48 / 11, qkv_bias=True, norm_layer=lambda d: LayerNormB(d, eps=1e-6))
    assert blk.mlp.fc1.out_features == 6144
    with torch.no_grad():
        blk.attn.q_bias.normal_(0, 0.02); blk.attn.v_bias.normal_(0, 0.02)
        blk.norm1.bias.normal_(0, 0.1); blk.norm2.bias.normal_(0, 0.1)
    return blk.bfloat16().cuda().eval()


def test_internvl_block_full_width(cuda_lib):
    from internvideo_b200.modules import set_fp8, set_fp8_inference
    blk = _ivl_block()
    B, n = 4, 257
    x = torch.randn((B * n, 3200), device="cuda")
    y0 = blk.forward_infer(x, B, n)
    assert set_fp8_inference(blk) == 1
    y1 = blk.forward_infer(x, B, n)
    again = blk.forward_infer(x, B, n)
    set_fp8_inference(blk, False)
    assert torch.equal(blk.forward_infer(x, B, n), y0)
    set_fp8(blk)
    yt = blk.forward_infer(x, B, n)
    set_fp8(blk, False)
    r, rt = _rel(y1 - x, y0 - x), _rel(yt - x, y0 - x)
    print(f"InternVL block (D 3200, n 257): branch rel. error per-token FP8 {r:.4f}, per-tensor set_fp8 {rt:.4f}")
    assert torch.equal(y1, again)
    assert r <= BRANCH_BOUND


def test_shared_videomae_block_full_width(cuda_lib):
    """The VideoMAE-g teacher's block (modules.VideoMAEBlock, head-axis attention) at full width under FP8 inference."""
    from internvideo_b200.modules import set_fp8_inference
    blk = _mae_block()
    B, n = 2, 2048
    x = torch.randn((B * n, 1408), device="cuda")
    y0 = blk.forward_infer(x, B, n, head_axis=True)
    assert set_fp8_inference(blk) == 1
    y1 = blk.forward_infer(x, B, n, head_axis=True)
    r = _rel(y1 - x, y0 - x)
    print(f"VideoMAE-g block (D 1408, n 2048, head-axis attention): branch rel. error {r:.4f}")
    assert torch.equal(y1, blk.forward_infer(x, B, n, head_axis=True))
    assert r <= BRANCH_BOUND
    set_fp8_inference(blk, False)
    assert torch.equal(blk.forward_infer(x, B, n, head_axis=True), y0)


def _teachers():
    from functools import partial
    from internvideo_b200.teachers import InternVL_CLIP, VisionTransformer
    z = np.load(GOLD / "teachers.npz")
    ccfg, mcfg = json.loads(bytes(z["clip_cfg"]).decode()), json.loads(bytes(z["mae_cfg"]).decode())
    c = InternVL_CLIP(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False, **ccfg)
    c.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("wc/")}, strict=True)
    m = VisionTransformer(norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), **mcfg)
    m.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("wm/")}, strict=True)
    cv = torch.from_numpy(z["clip_video"]).cuda().to(torch.bfloat16)
    mv = torch.from_numpy(z["mae_video"]).cuda().to(torch.bfloat16)
    return z, c.bfloat16().cuda().eval(), m.bfloat16().cuda().eval(), cv, mv


def _tap_err(a, b):
    return float((a.double() - b.double()).norm(dim=-1).max())


def test_teachers_fp8_against_bf16(cuda_lib):
    from internvideo_b200.modules import set_fp8_inference
    from internvideo_b200.teachers import attention_guided_mask, select_targets
    z, clip_t, mae_t, cv, mv = _teachers()
    zc0, x0, a0 = clip_t(cv)
    zm0 = mae_t(mv)
    assert set_fp8_inference(clip_t) == len(clip_t.blocks) and set_fp8_inference(mae_t) == len(mae_t.blocks)
    zc1, x1, a1 = clip_t(cv)
    zm1 = mae_t(mv)
    e = {"clip taps": _tap_err(zc1, zc0), "mae taps": _tap_err(zm1, zm0), "pooled": _rel(x1, x0), "attn": _rel(a1, a0)}
    print("teachers.npz, FP8 inference against bf16: " + ", ".join(f"{k} {v:.4f}" for k, v in e.items()))
    assert e["clip taps"] <= TAP_BOUND and e["mae taps"] <= TAP_BOUND
    assert e["pooled"] <= BRANCH_BOUND and e["attn"] <= BRANCH_BOUND
    assert all(e[k] <= lim for k, lim in MEASURED_LIMITS.items()), e
    imp = torch.from_numpy(z["importance"]).cuda()
    m0 = attention_guided_mask(a0, 2, 0.75, importance=imp)
    m1 = attention_guided_mask(a1, 2, 0.75, importance=imp)
    assert torch.equal(m0, m1)
    n = int((~m0[0]).sum())
    mae_small = torch.from_numpy(z["norm_mae_small"]).cuda()    # the fixture's MAE taps at the CLIP clip's geometry
    i0 = select_targets(zc0, x0, mae_small, m0, n)
    i1 = select_targets(zc1, x1, mae_small, m1, n)
    # the same tokens are selected: each CLIP target row is the FP8 tap of the token the bf16 run selected
    assert int(i0[3]) == int(i1[3]) == 0 and torch.equal(i0[2], i1[2])
    assert _tap_err(i1[0], i0[0]) <= TAP_BOUND
    # switching off restores the bf16 bits
    set_fp8_inference(clip_t, False); set_fp8_inference(mae_t, False)
    zc2, x2, a2 = clip_t(cv)
    assert torch.equal(zc2, zc0) and torch.equal(x2, x0) and torch.equal(a2, a0) and torch.equal(mae_t(mv), zm0)


def test_in_place_weight_change_is_picked_up(cuda_lib):
    from internvideo_b200.modules import set_fp8_inference
    _, clip_t, mae_t, cv, mv = _teachers()
    set_fp8_inference(clip_t); set_fp8_inference(mae_t)
    zc0, _, _ = clip_t(cv)
    zm0 = mae_t(mv)
    with torch.no_grad():
        clip_t.blocks[0].mlp.fc1.weight.mul_(0.5)
        mae_t.blocks[-1].attn.proj.weight.add_(0.01)
    zc1, _, _ = clip_t(cv)
    zm1 = mae_t(mv)
    assert not torch.equal(zc1, zc0) and not torch.equal(zm1, zm0)
    set_fp8_inference(clip_t, False); set_fp8_inference(mae_t, False)
    set_fp8_inference(clip_t); set_fp8_inference(mae_t)          # freshly quantised copies
    zc2, _, _ = clip_t(cv)
    assert torch.equal(zc1, zc2) and torch.equal(mae_t(mv), zm1)


def test_exclusion_rules_and_grad_refusal(cuda_lib):
    from internvideo_b200 import _lib
    from internvideo_b200.modules import set_fp8, set_fp8_inference
    blk = _ivl_block()
    B, n = 1, 257
    x = torch.randn((B * n, 3200), device="cuda")
    set_fp8(blk)
    with pytest.raises(_lib.IvbError, match="set_fp8"):
        set_fp8_inference(blk)
    set_fp8(blk, False)
    set_fp8_inference(blk)
    set_fp8(blk)
    with pytest.raises(_lib.IvbError, match="both on"):
        blk.forward_infer(x, B, n)
    set_fp8(blk, False)
    with pytest.raises(_lib.IvbError, match="no gradient"):
        blk.forward_stream(x.clone().requires_grad_(True), B, n)
    with torch.no_grad():
        assert torch.equal(blk.forward_stream(x, B, n), blk.forward_infer(x, B, n))


def _recipe_geometry_step(clip_t, mae_t, seed):
    """A DistillationStep at the recipe's token geometry (16 frames of 224^2, patch 14: VideoMAE 2048 tokens, the CLIP
    teacher and the student on every second frame, 8 x 257 tokens) with narrow towers, seeded."""
    from internvideo_b200.engine import PretrainEngine
    from internvideo_b200.modules import PretrainInternVideo2
    from internvideo_b200.teachers import DistillationStep
    torch.manual_seed(seed)
    student = PretrainInternVideo2(img_size=224, patch_size=14, num_frames=8, embed_dim=128, depth=2, num_heads=2,
                                   mlp_ratio=4, clip_embed_dim=64, clip_teacher_embed_dim=128, clip_teacher_final_dim=64,
                                   mae_teacher_embed_dim=64, clip_return_layer=2, mae_return_layer=2,
                                   attn_pool_num_heads=2, init_values=0.1, drop_path_rate=0.0, use_flash_attn=False,
                                   use_fused_rmsnorm=False, use_fused_mlp=False)
    student = student.bfloat16().cuda().train()
    engine = PretrainEngine(student, lr=1e-3, clip_grad=3.0, check_finite=True)
    return DistillationStep(student, engine, clip_t, mae_t, mask_ratio=0.8, td_ratio=2)


def test_distillation_step_with_fp8_teachers(cuda_lib):
    """DistillationStep with both teachers switched, unchanged: targets() gives the same bits on two calls, and the
    whole step (teachers, mask, targets, student forward + backward, AdamW) captured in engine.GraphedStep replays with
    the loss of the eager step to within its last bits.  The two arms start from identical students and take the same
    steps: one warm-up step, then the eager step or the first replay.  The loss is a sum of per-block partials added
    with atomics, so it may differ in its last bits between any two runs (DESIGN.md 10): 8 fp32 ulps are allowed."""
    from functools import partial
    from internvideo_b200.engine import GraphedStep
    from internvideo_b200.modules import set_fp8_inference
    from internvideo_b200.teachers import InternVL_CLIP, VisionTransformer
    torch.manual_seed(3)
    with torch.device("cuda"):     # as bench.py --with-teachers builds them (the MAE position table on the device)
        clip_t = InternVL_CLIP(img_size=224, patch_size=14, embed_dim=128, depth=2, num_heads=2, mlp_ratio=4,
                               attn_pool_num_heads=2, clip_embed_dim=64, clip_return_layer=2, init_values=0.1,
                               use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False)
        mae_t = VisionTransformer(img_size=224, patch_size=14, embed_dim=64, depth=2, num_heads=2, mlp_ratio=4,
                                  qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), all_frames=16,
                                  tubelet_size=2, mae_return_layer=2, mae_return_interval=1)
    clip_t = clip_t.bfloat16().cuda().eval(); mae_t = mae_t.bfloat16().cuda().eval()
    assert set_fp8_inference(clip_t) == 2 and set_fp8_inference(mae_t) == 2
    g = torch.Generator(device="cuda").manual_seed(5)
    video = torch.randn((1, 3, 16, 224, 224), device="cuda", generator=g).to(torch.bfloat16)
    imp = torch.stack([torch.randperm(256, device="cuda", generator=g) for _ in range(8)])   # the injected draw

    eager = _recipe_geometry_step(clip_t, mae_t, seed=11)
    t0, t1 = eager.targets(video, imp), eager.targets(video, imp)
    for a, b in zip(t0, t1):
        assert torch.equal(a, b) if torch.is_tensor(a) else a == b
    eager(video, imp)                                       # the warm-up step of the graphed arm
    loss_eager = float(eager(video, imp))

    graphed_step = _recipe_geometry_step(clip_t, mae_t, seed=11)
    graphed = GraphedStep(lambda v: graphed_step(v, imp), [video.clone()], warmup=1)
    loss_graph = float(graphed(video)[0])
    torch.cuda.synchronize()
    print(f"DistillationStep with FP8 teachers: eager loss {loss_eager!r}, graph replay {loss_graph!r}")
    assert loss_eager == loss_eager and abs(loss_graph - loss_eager) <= 8 * 2.0 ** -23 * abs(loss_eager)
