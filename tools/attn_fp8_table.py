"""FP8 attention for inference (modules.set_fp8_inference(model, attention=True)) on the H100, in one call.

Prints, with the card name and power limit read by the same call:
  1. the attention forward, bf16 (ivb_attn_fwd) against FP8 (ivb_attn_fp8_pack + ivb_attn_fwd_fp8, the pack also timed
     alone), at (n, d, H, B) = (1025, 64, 16, 128) (cfg-3 L tower), (2049, 88, 16, 32) (unmasked 1B stage-2 tower),
     (417, 88, 16, 32) (the 1B tower at the stage-1 student's 417 tokens) and (257, 128, 25, 256) (InternVL teacher),
     in ms per call, with q, k, v the column slots of one [B*n, 3*H*d] buffer as the blocks pass them.
  2. the frozen cfg-3 L tower forward (B = 128, 4 frames) and the unmasked 1B stage-2 tower forward (B = 32, 8 frames)
     under set_fp8_inference, attention off and on, alternated three times (ms per forward).

    python tools/attn_fp8_table.py [--no-towers] [--iters 20]
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

SHAPES = [(1025, 64, 16, 128), (2049, 88, 16, 32), (417, 88, 16, 32), (257, 128, 25, 256)]


def attn_table(iters):
    print("\n1. attention forward (ms per call; TFLOP/s of 4 n^2 d H B)")
    print(f"  {'n':>5s} {'d':>4s} {'H':>3s} {'B':>4s}  {'bf16':>7s}  {'pack':>7s}  {'fp8 fwd':>7s}  {'pack+fwd':>8s}  "
          f"{'TF bf16':>7s}  {'TF fp8':>6s}  {'speed-up':>8s}")
    for n, d, H, B in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(n)
        qkv = torch.randn((B * n, 3 * H * d), device="cuda", generator=g).to(torch.bfloat16)
        D = H * d
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        out = torch.empty((B * n, D), device="cuda", dtype=torch.bfloat16)
        packed = ll._attn_fp8_pack(q, k, v, B, n, H, d)
        s = d ** -0.5
        t_bf = timed(lambda: ll.attn_fwd(q, k, v, B, n, H, d, s, out=out, want_lse=False), iters)
        t_pk = timed(lambda: ll._attn_fp8_pack(q, k, v, B, n, H, d), iters)
        t_f8 = timed(lambda: ll._attn_fwd_fp8(*packed, B, n, H, d, s, out=out), iters)
        t_all = timed(lambda: ll._attn_fwd_fp8(*ll._attn_fp8_pack(q, k, v, B, n, H, d), B, n, H, d, s, out=out), iters)
        fl = 4.0 * n * n * d * H * B
        print(f"  {n:5d} {d:4d} {H:3d} {B:4d}  {t_bf:7.3f}  {t_pk:7.3f}  {t_f8:7.3f}  {t_all:8.3f}  "
              f"{fl / t_bf / 1e9:7.0f}  {fl / t_f8 / 1e9:6.0f}  {t_bf / t_all:7.2f}x")
        del qkv, out, packed


def tower_table():
    from internvideo_b200.clip_modules import InternVideo2
    from internvideo_b200.modules import set_fp8_inference
    from internvideo_b200.stage2 import PretrainInternVideo2
    print("\n2. frozen tower forwards under set_fp8_inference (ms per forward), attention off / on, alternated")
    torch.manual_seed(0)
    kw = dict(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False, drop_path_rate=0.0)
    towers = [
        ("cfg-3 L tower, B 128, n 1025", 128, 4,
         lambda: InternVideo2(embed_dim=1024, num_heads=16, mlp_ratio=4, depth=24, num_frames=4, attn_pool_num_heads=16,
                              clip_embed_dim=768, **kw), lambda m, x: m(x)),
        ("1B stage-2 tower unmasked, B 32, n 2049", 32, 8,
         lambda: PretrainInternVideo2(embed_dim=1408, num_heads=16, mlp_ratio=48 / 11, depth=40, num_frames=8,
                                      clip_embed_dim=768, clip_teacher_embed_dim=3200, clip_teacher_final_dim=768,
                                      **kw), lambda m, x: m(x, x_vis_only=True)),
    ]
    for label, B, T, make, fwd in towers:
        with torch.device("cuda"):
            model = make()
        model = model.bfloat16().cuda().eval()
        x = torch.randn((B, 3, T, 224, 224), device="cuda").to(torch.bfloat16)
        set_fp8_inference(model)
        res = {False: [], True: []}
        with torch.no_grad():
            outs = {}
            for att in (False, True):
                set_fp8_inference(model, True, attention=att)
                outs[att] = fwd(model, x).float()
            rel = float((outs[True] - outs[False]).norm() / outs[False].norm())
            for _ in range(3):
                for att in (False, True):
                    set_fp8_inference(model, True, attention=att)
                    res[att].append(timed(lambda: fwd(model, x), 3))
        print(f"  {label}: attention bf16 " + " / ".join(f"{t:.1f}" for t in res[False]) + " ms, FP8 "
              + " / ".join(f"{t:.1f}" for t in res[True]) + f" ms; output rel. difference {rel:.4f}")
        del model, x, outs
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-towers", action="store_true")
    args = ap.parse_args()
    ll.device_check()
    print("card:", card())
    attn_table(args.iters)
    if not args.no_towers:
        tower_table()
    print("card:", card())


if __name__ == "__main__":
    main()
