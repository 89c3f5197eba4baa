"""Every GEMM shape of the cfg-2 (InternVideo2-1B, B=32, n=417) step — forward (NT), dgrad (NN) and wgrad (TT) — on
libivb200's default kernel (what the step launches) against cuBLAS via torch.matmul on the same operands.
usage: python tools/gemm_table.py > gemm_vs_cublas.md      (device-timed, 20 launches after 3 warm-ups)"""
import json, os, sys
sys.path.insert(0, ".")
import torch
from internvideo_b200 import lowlevel as ll

bf = torch.bfloat16


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


peak = None
try:
    peak = json.load(open("MEASURED_PEAKS.json")).get("bf16_tflops_sustained")
except Exception:
    pass
M = 13344          # 32 clips x 417 visible tokens
layers = [("qkv", 1408, 4224), ("proj", 1408, 1408), ("fc1", 1408, 6144), ("fc2", 6144, 1408), ("clip head", 1408, 3200)]
print(f"# libivb200 wgmma GEMM (default single-CTA kernel) vs cuBLAS, cfg-2 shapes, {torch.cuda.get_device_name()}\n")
print(f"M = {M} tokens; TF/s = 2MNK / device time (CUDA events, 20 launches, same operands for both); "
      f"sustained bf16 peak of this pool {peak} TF/s (MEASURED_PEAKS.json).\n")
print("| GEMM | role | M x N x K | cuBLAS TF/s | ivb200 TF/s | ivb/cuBLAS | ivb / peak |")
print("|---|---|---|---|---|---|---|")
tot_c = tot_i = 0.0
for name, din, dout in layers:
    x = torch.randn(M, din, device="cuda").to(bf)
    w = (torch.randn(dout, din, device="cuda") * 0.02).to(bf)
    dy = torch.randn(M, dout, device="cuda").to(bf)
    y = torch.empty(M, dout, device="cuda", dtype=bf)
    dx = torch.empty(M, din, device="cuda", dtype=bf)
    dw = torch.empty(dout, din, device="cuda", dtype=bf)
    cases = [
        ("fwd  y = x W^T", (M, dout, din), lambda: torch.matmul(x, w.t(), out=y), lambda: ll.gemm(x, w, out0=y)),
        ("dgrad dx = dy W", (M, din, dout), lambda: torch.matmul(dy, w, out=dx), lambda: ll.gemm(dy, w, b_t=True, out0=dx)),
        ("wgrad dW = dy^T x", (dout, din, M), lambda: torch.matmul(dy.t(), x, out=dw),
         lambda: ll.gemm(dy, x, a_t=True, b_t=True, out0=dw)),
    ]
    for role, (m, n, k), f_c, f_i in cases:
        fl = 2.0 * m * n * k
        tc, ti = timeit(f_c), timeit(f_i)
        tot_c += tc; tot_i += ti
        a, b = fl / tc / 1e9, fl / ti / 1e9
        pk = f"{b / peak:.2f}" if peak else "n/a"
        print(f"| {name} | {role} | {m} x {n} x {k} | {a:.0f} | {b:.0f} | {b / a:.2f} | {pk} |", flush=True)
print(f"\nSum of the 15 launches: cuBLAS {tot_c:.3f} ms, ivb200 {tot_i:.3f} ms ({tot_c / tot_i:.3f}x).")
