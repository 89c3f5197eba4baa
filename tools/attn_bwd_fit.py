"""Fit attention-backward time to  CTAs/SMs * (F + ntile * I): F = per-CTA fixed cost (prologue + epilogue),
I = cost per streamed 64-token tile.  B*H = 512 heads of d=88 (cfg-2 head shape), n swept."""
import sys
sys.path.insert(0, ".")
import torch
from internvideo_b200 import lowlevel as ll

bf = torch.bfloat16
SMS = torch.cuda.get_device_properties(0).multi_processor_count
B, H, d = 32, 16, 88
D = H * d
res = []
for n in (128, 256, 384, 417, 512, 768, 1024, 2048):
    qkv = torch.randn(B * n, 3 * D, device="cuda").to(bf)
    dout = torch.randn(B * n, D, device="cuda").to(bf)
    dqkv = torch.empty_like(qkv)
    out, lse = ll.attn_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B, n, H, d, d ** -0.5)
    f = lambda: ll.attn_bwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], out, dout, lse, B, n, H, d, d ** -0.5,
                            dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])
    for _ in range(3): f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): f()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 10 * 1e3
    rt, nt = (n + 127) // 128, (n + 63) // 64
    ctas = 2 * B * H * rt          # two passes (dK/dV and dQ)
    fl = 2.5 * 4 * n * n * d * B * H
    print(f"n={n:5d} row_tiles={rt:3d} tiles={nt:3d}  {us:9.1f} us   per-CTA-slot {us * SMS / ctas:7.2f} us   {fl / us / 1e6:7.1f} TFLOP/s", flush=True)
    res.append((nt, us * SMS / ctas))
import numpy as np
A = np.array([[1.0, nt] for nt, _ in res]); y = np.array([t for _, t in res])
(F, I), *_ = np.linalg.lstsq(A, y, rcond=None)
print(f"fit: per-CTA fixed {F:.2f} us + {I:.3f} us per streamed tile (both passes averaged)")
