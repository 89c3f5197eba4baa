"""Stochastic depth on the H100: what skipping the dropped clips saves, in one call.

Prints, with the card name and power limit:
  1. the eight forward and input-gradient GEMMs of a cfg-2 block (B = 32 clips of n = 417 tokens, M = 13 344), in bf16
     and in per-token FP8, without a plan and with the M plan of a draw that drops 0, 1/8, 1/4 or 1/2 of the clips (the
     dropped clips spread over the batch): ms per launch, the library's default kernel;
  2. attention forward and backward (16 heads of 88) at the same draws, plain against planned (ivb_attn_*_plan);
  3. the cfg-2 training step (B = 32, one CUDA graph, drop-path rate 0.25) in bf16 and per-token FP8, with the skipping
     on and off (modules.set_droppath_skip), alternated three times each.

    python tools/droppath_table.py [--no-step] [--iters 50]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import GEMMS, card, step_table, timed  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402
from internvideo_b200 import ops  # noqa: E402

B, N_TOK, H, HD = 32, 417, 16, 88
M = B * N_TOK
FRACTIONS = [(0, "0"), (8, "1/8"), (4, "1/4"), (2, "1/2")]   # every k-th clip dropped


def draw(k):
    """Per-row DropPath factors [M] of a draw that drops every k-th clip (k = 0: none)."""
    keep = torch.ones(B, device="cuda") if k == 0 else (torch.arange(B, device="cuda") % k != 0).float()
    return (keep / 0.75).repeat_interleave(N_TOK).contiguous()


def m_plan(rs):
    return ops._branch_plans(ops.droppath_plan(rs[None])[0], M, ops.BF16)[0]


def gemm_table(iters):
    print(f"\n1. block GEMMs at M = {M} (ms per launch: no plan, then the plan of each dropped fraction)")
    head = "  ".join(f"{'drop ' + f:>8s}" for _, f in FRACTIONS)
    print(f"  {'gemm':6s} {'prec':5s} {'N':>5s} {'K':>5s}  {'no plan':>8s}  {head}")
    plans = [m_plan(draw(k)) for k, _ in FRACTIONS]
    tot = {prec: [0.0] * (1 + len(plans)) for prec in ("bf16", "token")}
    for name, N, K, _, bt in GEMMS:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = torch.randn((M, K), generator=g, device="cuda").to(torch.bfloat16)
        w = (torch.randn((N, K) if not bt else (K, N), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        ra, rsa = ll.fp8_quantize_rows(a)
        rb, rsb = ll.fp8_quantize_rows(w, transposed=bt)
        calls = {"bf16": lambda plan: ll.gemm(a, w, b_t=bt, m_plan=plan),
                 "token": lambda plan: ll._gemm_fp8_plan(ra, rsa, rb, rsb, plan)}
        for prec, fn in calls.items():
            ts = [timed(lambda: fn(None), iters)] + [timed(lambda: fn(p), iters) for p in plans]
            tot[prec] = [x + t for x, t in zip(tot[prec], ts)]
            print(f"  {name:6s} {prec:5s} {N:5d} {K:5d}  {ts[0]:8.3f}  " + "  ".join(f"{t:8.3f}" for t in ts[1:]))
    for prec, ts in tot.items():
        print(f"  sum of the eight, {prec:5s}: {ts[0]:8.3f}  " + "  ".join(f"{t:8.3f}" for t in ts[1:]))


def attn_table(iters):
    print(f"\n2. attention, B = {B}, n = {N_TOK}, {H} heads of {HD} (ms per call: plain, then planned per fraction)")
    D = H * HD
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn((M, 3 * D), generator=g, device="cuda").to(torch.bfloat16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    dout = torch.randn((M, D), generator=g, device="cuda").to(torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    out, lse = ll.attn_fwd(q, k, v, B, N_TOK, H, HD, HD ** -0.5)
    fwd = lambda rs: ll.attn_fwd(q, k, v, B, N_TOK, H, HD, HD ** -0.5, out=out, rowscale=rs)  # noqa: E731
    bwd = lambda rs: ll.attn_bwd(q, k, v, out, dout, lse, B, N_TOK, H, HD, HD ** -0.5,  # noqa: E731
                                 dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:], rowscale=rs)
    rss = [draw(kk) for kk, _ in FRACTIONS]
    head = "  ".join(f"{'drop ' + f:>8s}" for _, f in FRACTIONS)
    print(f"  {'pass':8s}  {'plain':>8s}  {head}")
    for name, fn in (("forward", fwd), ("backward", bwd)):
        ts = [timed(lambda: fn(None), iters)] + [timed(lambda: fn(rs), iters) for rs in rss]
        print(f"  {name:8s}  {ts[0]:8.3f}  " + "  ".join(f"{t:8.3f}" for t in ts[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    ll.device_check()
    print("card:", card())
    gemm_table(args.iters)
    attn_table(args.iters)
    if not args.no_step:
        step_table(modes=("off", "token"), skips=(True, False))
    print("card:", card())


if __name__ == "__main__":
    main()
