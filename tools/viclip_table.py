"""ViCLIP-L/14 on the H100, in one call that also prints the card name and power limit:
  1. the recipe's training step on one GPU (exp/exp_pretrain_ViCLIP: 8 frames at 224^2, masking_prob 0.9, so n = 206
     tokens per clip; the text tower frozen with 32-token captions; checkpoint_num 24; DropPath 0.1): forward, VTC loss
     and backward, ms per step over CUDA events, the library's ViCLIP against the staged unmodified reference modules
     (oracle/_ref/, filled by oracle/viclip.stage at build time) under bf16 autocast on the same card, the two arms
     alternated in windows;
  2. the fc1 GEMM of that step (M = B * 206, N = 4096, K = 1024, saving the GELU derivative as training does) with the
     erf GELU epilogue against the QuickGELU one, and the dh GEMM (EPI_GELU_BWD from the saved derivative), ms per
     launch, alternated.

    python tools/viclip_table.py [--batch 32] [--steps 5] [--rounds 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import card, timed  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402
from internvideo_b200 import viclip  # noqa: E402
from internvideo_b200.contrastive import VTC_VTM_Loss  # noqa: E402

bf = torch.bfloat16
T, RES, P, MASK_P, CTX = 8, 224, 14, 0.9, 32


def recipe_config():
    return {"max_txt_l": CTX, "inputs": {"image_res": RES, "video_input": {"num_frames": T}},
            "model": {"vision_encoder": {"name": "vit_l14", "pretrained": False, "d_model": 1024, "kernel_size": 1,
                                         "center": True, "drop_path_rate": 0.1, "masking_prob": MASK_P,
                                         "checkpoint_num": 24},
                      "text_encoder": {"name": "vit_l14", "pretrained": False, "d_model": 768, "vocab_size": 49408},
                      "embed_dim": 768, "temp": 1 / 100.0, "temp_min": 1 / 100.0, "freeze_text": True}}


def _init_empty(model):
    """Draw the parameters the constructors leave uninitialised (checkpoint-loaded in practice)."""
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith(("proj", "text_projection", "text_encoder.positional_embedding")):
                p.normal_(0, p.shape[0] ** -0.5 * 0.1)


def _inputs(B):
    g = torch.Generator(device="cuda").manual_seed(0)
    video = torch.randn(B, T, 3, RES, RES, device="cuda", generator=g).to(bf)
    ids = torch.randint(1, 49406, (B, CTX), device="cuda", generator=g)
    ids[:, -1] = 49407                                    # the EOT, the largest id
    return video, ids, torch.arange(B, device="cuda")


def ours(B):
    torch.manual_seed(0)
    model = viclip.ViCLIP(recipe_config())
    _init_empty(model)
    model = model.bfloat16().cuda().train()
    video, ids, idx = _inputs(B)

    def step():
        model.zero_grad(set_to_none=True)
        model(video, None, ids, idx)["loss_vtc"].backward()
    return step


def reference(B):
    """The unmodified reference towers (clip_joint_l14's and clip_text_l14's modules, built without their downloads)
    with InternVideo2's VTC loss, which is ViCLIP's statement for statement, all_gather off (one GPU).  The recipe
    trains under autocast (fp16=True) with fp32 parameters; the text tower's fp32 LayerNorm refuses bf16 parameters, so
    the reference runs as the recipe does, under bf16 autocast."""
    from oracle import ref_shim
    from oracle import viclip as ov
    if not ov.available():
        return None
    vision_mod, text_mod = ov.import_viclip()
    crit, _ = ref_shim.import_criterions()
    torch.manual_seed(0)
    vis = vision_mod.VisionTransformer(input_resolution=RES, patch_size=P, width=1024, layers=24, heads=16,
                                       output_dim=768, kernel_size=1, num_frames=T, drop_path=0.1, checkpoint_num=24)
    txt = text_mod.CLIP_TEXT(768, CTX, 49408, 768, 12, 12, 0)
    for m in (vis, txt):
        _init_empty(m)
    txt.requires_grad_(False)
    vis, txt = vis.cuda().train(), txt.cuda().train()
    temp = torch.nn.Parameter(torch.tensor(0.01, device="cuda"))
    loss = crit.VTC_VTM_Loss(False)
    video, ids, idx = _inputs(B)

    def step():
        vis.zero_grad(set_to_none=True)
        with torch.no_grad():
            temp.clamp_(min=0.01)
        with torch.autocast("cuda", dtype=bf):
            v = vis(video.permute(0, 2, 1, 3, 4).contiguous(), masking_prob=MASK_P)
            t = txt(ids)
            out = loss.vtc_loss(v, t, idx, temp, all_gather=False)
        out.backward()
    return step


def step_table(B, steps, rounds):
    L = (RES // P) ** 2 * T
    n = L - int(MASK_P * L) + 1
    print(f"\n1. ViCLIP-L/14 training step, {B} clips x {T} frames at {RES}^2 (n = {n} after masking), frozen text "
          f"{B} x {CTX} tokens, checkpoint_num 24, DropPath 0.1 (ms per step; {rounds} alternated windows of {steps} "
          "steps)")
    arms = {"ivb200": ours(B)}
    ref = reference(B)
    if ref is not None:
        arms["reference (bf16)"] = ref
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, steps))
    for k, v in res.items():
        print(f"  {k:18s} min {min(v):8.1f}  max {max(v):8.1f}   ({', '.join(f'{x:.1f}' for x in v)})")
    if ref is not None:
        print(f"  ivb200 / reference (best windows): {min(res['ivb200']) / min(res['reference (bf16)']):.3f}")
    else:
        print("  reference not staged (oracle/_ref/): its arm is not measured")


def gemm_table(B, iters, rounds):
    L = (RES // P) ** 2 * T
    n = L - int(MASK_P * L) + 1
    M, D, Hd = B * n, 1024, 4096
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(M, D, device="cuda", generator=g)).to(bf)
    w1 = (torch.randn(Hd, D, device="cuda", generator=g) * 0.02).to(bf)
    b1 = (torch.randn(Hd, device="cuda", generator=g) * 0.1).to(bf)
    w2 = (torch.randn(D, Hd, device="cuda", generator=g) * 0.02).to(bf)
    dy = (torch.randn(M, D, device="cuda", generator=g)).to(bf)
    h = torch.empty(M, Hd, device="cuda", dtype=bf)
    gd = torch.empty(M, Hd, device="cuda", dtype=bf)
    ll.gemm(x, w1, epi=ll.EPI_BIAS_GELU, flags=ll.FLAG_GELU_QUICK | ll.FLAG_GELU_SAVE_GRAD, bias=b1, out1=gd)
    forms = {"erf": 0, "QuickGELU": ll.FLAG_GELU_QUICK}
    res = {(f, k): [] for f in forms for k in ("fc1", "dh")}
    for _ in range(rounds):
        for f, fl in forms.items():
            res[f, "fc1"].append(timed(lambda: ll.gemm(x, w1, epi=ll.EPI_BIAS_GELU, flags=fl | ll.FLAG_GELU_SAVE_GRAD,
                                                       bias=b1, out1=h), iters))
            res[f, "dh"].append(timed(lambda: ll.gemm(dy, w2, b_t=True, epi=ll.EPI_GELU_BWD,
                                                      flags=fl | ll.FLAG_GELU_SAVE_GRAD, aux=gd), iters))
    print(f"\n2. GEMMs of the step, {M} x {Hd} x {D} (fc1, out1 = GELU') and {M} x {Hd} x {D} (dh from the saved GELU'), "
          f"ms per launch, min-max of {rounds} alternated windows of {iters}")
    for f in forms:
        print(f"  {f:10s} fc1 {min(res[f, 'fc1']):.4f}-{max(res[f, 'fc1']):.4f}   "
              f"dh {min(res[f, 'dh']):.4f}-{max(res[f, 'dh']):.4f}")
    flop = 2.0 * M * Hd * D
    print(f"  fc1 QuickGELU: {flop / min(res['QuickGELU', 'fc1']) / 1e9:.0f} TFLOP/s (best window)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/viclip_table.py measures on the GPU"
    print(f"GPU: {card()} (name, power limit, max SM clock)")
    step_table(a.batch, a.steps, a.rounds)
    gemm_table(a.batch, a.iters, a.rounds)


if __name__ == "__main__":
    main()
