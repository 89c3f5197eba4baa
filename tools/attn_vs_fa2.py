"""Attention forward AND backward vs flash_attn (FA2, the kernel the reference calls: flash_attention_class.py:47-50) on the
same GPU, at the BASELINE shapes: cfg-2 (1B, n=417, d=88, B=32), cfg-3 (L, n=1025, d=64), cfg-4 (6B, n=833, d=128) and the
cfg-5 sequence-length sweep 1568 -> 12544 tokens (d=88).  CUDA events, 3 warm-ups, L2 flushed between iterations.
Prints a markdown table (TFLOP/s of the algorithmic 4 n^2 D fwd / 10 n^2 D bwd; fraction of the sustained bf16 peak).
  python tools/attn_vs_fa2.py > attention_vs_fa2.md"""
import json
import sys
from pathlib import Path

sys.path.insert(0, ".")
import torch
from internvideo_b200 import lowlevel as ll

bf = torch.bfloat16
ROOT = Path(__file__).resolve().parent.parent
pk = ROOT / "MEASURED_PEAKS.json"
PEAK = json.loads(pk.read_text()).get("bf16_tflops_sustained", 989.0) if pk.exists() else 989.0   # H100 SXM data sheet, dense BF16
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()                           # > 50 MB L2
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


SHAPES = [("cfg-2 1B", 32, 417, 16, 88), ("cfg-3 L", 16, 1025, 16, 64), ("cfg-3 L (B=128)", 128, 1025, 16, 64),
          ("cfg-4 6B", 8, 833, 25, 128), ("cfg-5", 8, 1568, 16, 88), ("cfg-5", 4, 3136, 16, 88), ("cfg-5", 2, 6272, 16, 88),
          ("cfg-5", 1, 12544, 16, 88), ("cfg-5 d=64", 1, 12544, 16, 64), ("cfg-5 d=128", 1, 12544, 16, 128)]
try:
    from flash_attn import flash_attn_func
    import flash_attn
    fav = flash_attn.__version__
except Exception as e:  # noqa: BLE001
    flash_attn_func, fav = None, f"n/a ({type(e).__name__})"
print(f"# attention fwd / bwd: ivb200 (wgmma) vs flash_attn {fav} — {torch.cuda.get_device_name()}, sustained bf16 peak {PEAK} TFLOP/s\n")
print("| shape | B | n | H x d | ivb fwd us | TF/s | frac | FA2 fwd TF/s | ivb/FA2 | ivb bwd us | TF/s | frac | FA2 bwd TF/s | ivb/FA2 |")
print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
for tag, B, n, H, d in SHAPES:
    D = H * d
    qkv = (torch.randn(B * n, 3 * D, device="cuda") * 0.5).to(bf)
    dout = torch.randn(B * n, D, device="cuda").to(bf)
    dqkv = torch.empty_like(qkv)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    out, lse = ll.attn_fwd(q, k, v, B, n, H, d, d ** -0.5)
    tf = timeit(lambda: ll.attn_fwd(q, k, v, B, n, H, d, d ** -0.5, out=out))
    tb = timeit(lambda: ll.attn_bwd(q, k, v, out, dout, lse, B, n, H, d, d ** -0.5, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:]))
    ff, fb = 4.0 * B * H * n * n * d, 10.0 * B * H * n * n * d
    row = f"| {tag} | {B} | {n} | {H}x{d} | {tf*1e3:.0f} | {ff/tf/1e9:.0f} | {ff/tf/1e9/PEAK:.3f} |"
    fa_f = fa_b = None
    if flash_attn_func is not None:
        try:
            q4 = qkv.view(B, n, 3, H, d)
            qq, kk, vv = (q4[:, :, i].detach().requires_grad_(True) for i in range(3))
            fa_f = timeit(lambda: flash_attn_func(qq, kk, vv))
            o = flash_attn_func(qq, kk, vv)
            do4 = dout.view(B, n, H, d)
            fa_b = timeit(lambda: torch.autograd.grad(o, (qq, kk, vv), do4, retain_graph=True))
        except Exception as e:  # noqa: BLE001
            print(f"<!-- FA2 failed at {tag}: {type(e).__name__}: {e} -->")
    row += f" {ff/fa_f/1e9:.0f} | {fa_f/tf:.2f}x |" if fa_f else " n/a | n/a |"
    row += f" {tb*1e3:.0f} | {fb/tb/1e9:.0f} | {fb/tb/1e9/PEAK:.3f} |"
    row += f" {fb/fa_b/1e9:.0f} | {fa_b/tb:.2f}x |" if fa_b else " n/a | n/a |"
    print(row, flush=True)
    del qkv, dout, dqkv, out, lse
