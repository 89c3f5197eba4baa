"""FP8 weight gradients (modules.set_fp8(model, scaling="token", wgrad=True)) on the H100, in one call.

Prints, with the card name and power limit read by the same call:
  1. the four weight-gradient GEMMs of a block at the cfg-2 shapes (D = 1408, hidden 6144, 13 344 tokens: B = 32 clips
     of 417) and at the cfg-4 (6B) block shapes (D = 3200, hidden 12 800, 6 664 tokens: 8 clips of 833): the bf16
     wgrad (ivb_gemm_bf16, both operands MN-major), the FP8 GEMM (ivb_gemm_fp8_wgrad), the two transposing casts that
     feed it (ivb_fp8_quantize_blocks_t of dy and of the activation) and FP8 GEMM + casts, in ms per call.
  2. the cfg-2 training step (B = 32, drop-path 0.25, one CUDA graph), per-token FP8 with FP8 weight gradients and
     without, alternated three times.

    python tools/fp8_wgrad_table.py [--no-step] [--iters 30]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import card, step_table, timed  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402


def shapes(D, Hd):
    """(name, dy width = output channels, activation width = input channels) of the four weight gradients."""
    return [("qkv", 3 * D, D), ("proj", D, D), ("fc1", Hd, D), ("fc2", D, Hd)]


def gemm_table(label, T, D, Hd, iters):
    print(f"\n1. {label}: weight gradients over {T} tokens (ms per call)")
    print(f"  {'wgrad':5s} {'M':>6s} {'N':>6s}  {'bf16':>7s}  {'fp8 gemm':>8s}  {'casts':>7s}  {'fp8+casts':>9s}  "
          f"{'TF bf16':>7s}  {'TF fp8':>6s}")
    g = torch.Generator(device="cuda").manual_seed(0)
    tot = [0.0, 0.0, 0.0]
    for name, Mo, N in shapes(D, Hd):
        dy = torch.randn((T, Mo), device="cuda", generator=g).to(torch.bfloat16)
        act = torch.randn((T, N), device="cuda", generator=g).to(torch.bfloat16)
        (qa, sa), (qb, sb) = ll._fp8_quantize_blocks_t(dy), ll._fp8_quantize_blocks_t(act)
        t_bf = timed(lambda: ll.gemm(dy, act, a_t=True, b_t=True), iters)
        t_f8 = timed(lambda: ll._gemm_fp8_wgrad(qa, sa, qb, sb), iters)
        t_c = timed(lambda: (ll._fp8_quantize_blocks_t(dy), ll._fp8_quantize_blocks_t(act)), iters)
        fl = 2.0 * Mo * N * T
        for i, t in enumerate((t_bf, t_f8, t_c)):
            tot[i] += t
        print(f"  {name:5s} {Mo:6d} {N:6d}  {t_bf:7.3f}  {t_f8:8.3f}  {t_c:7.3f}  {t_f8 + t_c:9.3f}  "
              f"{fl / t_bf / 1e9:7.0f}  {fl / t_f8 / 1e9:6.0f}")
    print(f"  block: bf16 {tot[0]:.3f}, fp8 gemm {tot[1]:.3f}, casts {tot[2]:.3f}, fp8 + casts {tot[1] + tot[2]:.3f} ms"
          f" ({tot[0] - tot[1] - tot[2]:+.3f} ms saved per block)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    ll.device_check()
    print("card:", card())
    gemm_table("cfg-2 (D 1408, hidden 6144)", 32 * 417, 1408, 6144, args.iters)
    gemm_table("cfg-4 block (D 3200, hidden 12800)", 8 * 833, 3200, 12800, args.iters)
    if not args.no_step:
        step_table(modes=("token", "token_wgrad"))
    print("card:", card())


if __name__ == "__main__":
    main()
