"""Per-token FP8 training of the ViT block (modules.set_fp8(model, scaling="token")) on the H100, in one call.

Prints, with the card name and power limit:
  1. the cast calls of one cfg-2 block (M = 13 344 tokens), per-tensor (ivb_fp8_quantize) against per-token: time and
     achieved GB/s of the algorithmic bytes.  Per-tensor: bf16 read twice (amax, cast) plus the FP8 write, a weight also
     its transposed copy.  Per-token: n1 and n2 come out of the norm kernel, so their cast is the E4M3 write and the
     time the fused norm takes over the bf16 norm (ivb_norm_fwd_fp8_train against ivb_norm_fwd); a, g and the four
     gradients read bf16 once and write E4M3 (ivb_fp8_quantize_rows); a weight is cast by rows (read, write) and by
     columns into its transposed copy (ivb_fp8_quantize_cols_t: read twice, write).
  2. the eight forward and input-gradient GEMMs at the cfg-2 shapes: bf16, per-tensor FP8 and per-token FP8 (row and
     column scale vectors), the library's default kernel, plain bf16 epilogue; and the per-token accumulation-error
     ratio (tests/test_fp8_rowwise_gpu.py::rowwise_accumulation_ratio, limit 0.25 as in tests/test_gemm_fp8_gpu.py).
  3. the cfg-2 training step (B = 32, one CUDA graph) in bf16, per-tensor FP8 and per-token FP8, alternated three times.

    python tools/fp8_token_table.py [--no-step] [--iters 50]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import GEMMS, HBM, M, card, step_table, timed  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402

D, HID = 1408, 6144
WEIGHTS = [("Wqkv", 3 * D, D), ("Wproj", D, D), ("Wfc1", HID, D), ("Wfc2", D, HID)]
ACTS = [("a", D), ("g", HID)]
GRADS = [("dy2", D), ("dh", HID), ("dy1", D), ("dqkv", 3 * D)]


def _row(name, ms, nb):
    print(f"  {name:12s} {ms:7.3f} ms  {nb / 1e9:6.3f} GB  {nb / ms / 1e6:7.0f} GB/s  {nb / ms * 1e3 / HBM:5.1%}")
    return ms, nb


def _total(label, rows):
    ms, nb = sum(r[0] for r in rows), sum(r[1] for r in rows)
    print(f"  {label}: {ms:.3f} ms for {nb / 1e9:.3f} GB ({nb / ms / 1e6:.0f} GB/s; at 3.35 TB/s {nb / HBM * 1e3:.3f} ms)")


def cast_table(iters):
    print("\n1. casts of one cfg-2 block, M = 13344 (ms per call; algorithmic GB; GB/s; share of 3.35 TB/s)")
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda r, c: torch.randn((r, c), device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
    x = torch.randn((M, D), device="cuda", generator=g)
    nw = torch.ones(D, device="cuda", dtype=torch.bfloat16)
    print(" per-tensor (ivb_fp8_quantize)")
    rows = []
    for name, C, fmt in ([("n1", D, ll.FP8_E4M3), ("n2", D, ll.FP8_E4M3)] + [(n, c, ll.FP8_E4M3) for n, c in ACTS]
                         + [(n, c, ll.FP8_E5M2) for n, c in GRADS]):
        t = rnd(M, C)
        rows.append(_row(name, timed(lambda: ll.fp8_quantize(t, fmt), iters), M * C * 5))
    for name, N, K in WEIGHTS:
        w = rnd(N, K)
        rows.append(_row(name + " +T", timed(lambda: ll.fp8_quantize(w, ll.FP8_E4M3, transpose=True), iters), N * K * 6))
    _total("per-tensor total", rows)
    print(" per-token")
    rows = []
    t_bf = timed(lambda: ll.norm_fwd(x, nw), iters)
    t_f8 = timed(lambda: ll.norm_fwd_fp8(x, nw, save=True), iters)
    print(f"  (norm: ivb_norm_fwd {t_bf:.3f} ms, ivb_norm_fwd_fp8_train {t_f8:.3f} ms)")
    for name in ("n1", "n2"):
        rows.append(_row(name + " (fused)", t_f8 - t_bf, M * D))
    for name, C in ACTS + GRADS:
        t = rnd(M, C)
        rows.append(_row(name, timed(lambda: ll.fp8_quantize_rows(t), iters), M * C * 3))
    for name, N, K in WEIGHTS:
        w = rnd(N, K)
        rows.append(_row(name + " rows", timed(lambda: ll.fp8_quantize_rows(w), iters), N * K * 3))
        rows.append(_row(name + " cols^T", timed(lambda: ll.fp8_quantize_rows(w, transposed=True), iters), N * K * 5))
    _total("per-token total", rows)


def gemm_table(iters):
    from test_fp8_rowwise_gpu import rowwise_accumulation_ratio
    print("\n2. GEMMs at M = 13344 (ms per launch; TFLOP/s; per-token accumulation ratio, limit 0.25)")
    print(f"  {'gemm':6s} {'N':>5s} {'K':>5s}  {'bf16':>7s}  {'tensor':>7s}  {'token':>7s}  {'TF token':>8s}  {'ratio':>6s}")
    tot = [0.0, 0.0, 0.0]
    for name, N, K, fmt, bt in GEMMS:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = torch.randn((M, K), generator=g, device="cuda").to(torch.bfloat16)
        w = (torch.randn((N, K) if not bt else (K, N), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        qa, _, sa, _ = ll.fp8_quantize(a, ll.FP8_E5M2 if fmt == torch.float8_e5m2 else ll.FP8_E4M3)
        qw, qwt, sw, _ = ll.fp8_quantize(w, ll.FP8_E4M3, transpose=True)
        ra, rsa = ll.fp8_quantize_rows(a)
        rb, rsb = ll.fp8_quantize_rows(w, transposed=bt)
        t_bf = timed(lambda: ll.gemm(a, w, b_t=bt), iters)
        t_te = timed(lambda: ll.gemm_fp8(qa, sa, qwt if bt else qw, sw), iters)
        t_to = timed(lambda: ll.gemm_fp8(ra, rsa, rb, rsb), iters)
        ratio = rowwise_accumulation_ratio(M, N, K)
        for i, t in enumerate((t_bf, t_te, t_to)):
            tot[i] += t
        print(f"  {name:6s} {N:5d} {K:5d}  {t_bf:7.3f}  {t_te:7.3f}  {t_to:7.3f}  {2.0 * M * N * K / t_to / 1e9:8.0f}"
              f"  {ratio:6.4f}")
    print(f"  sum of the eight: bf16 {tot[0]:.3f}, per-tensor {tot[1]:.3f}, per-token {tot[2]:.3f} ms per block")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    ll.device_check()
    print("card:", card())
    cast_table(args.iters)
    gemm_table(args.iters)
    if not args.no_step:
        step_table(modes=("off", "tensor", "token"))
    print("card:", card())


if __name__ == "__main__":
    main()
