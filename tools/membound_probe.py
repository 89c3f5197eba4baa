"""Per-call time of the memory-bound entry points at cfg-2 shapes (M = 32*417 rows, D = 1408, decoder width 3200,
a 64 M-parameter AdamW slice), timed with CUDA events over many back-to-back calls, with the achieved HBM rate.

Bytes are the algorithmic traffic computed from the shapes (every input read once, every output written once, O(D)
vectors ignored); a call includes its colred_finish launch where it has one.  Most inputs are larger than the 50 MB
L2.  The card name and power limit are printed with the numbers, since both are part of them.

    python tools/membound_probe.py [--lib path/to/libivb200.so] [--iters 200]
"""
import argparse
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch

from internvideo_b200 import _lib
from internvideo_b200 import lowlevel as ll

ap = argparse.ArgumentParser()
ap.add_argument("--lib", help="libivb200.so to time (default: the one in this tree)")
ap.add_argument("--iters", type=int, default=200)
args = ap.parse_args()
if args.lib:
    _lib.LIB_PATH = Path(args.lib).resolve()
assert torch.cuda.is_available(), "membound_probe needs a GPU"


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


bf, f32 = torch.bfloat16, torch.float32
M, D, C = 32 * 417, 1408, 3200
dev = "cuda"
torch.manual_seed(0)
x = torch.randn(M, D, device=dev); w = torch.ones(D, device=dev, dtype=bf); bias = torch.zeros(D, device=dev, dtype=bf)
dy = torch.randn(M, D, device=dev).to(bf); dxin = torch.randn(M, D, device=dev)
_, _, rstd = ll.norm_fwd(x, w)
_, lmean, lrstd = ll.norm_fwd(x, w, bias, eps=1e-5, layernorm=True)
dw = torch.zeros(D, device=dev); db = torch.zeros(D, device=dev)
qkv = torch.randn(M, 3 * D, device=dev).to(bf); qn = torch.empty(M, 2 * D, device=dev, dtype=bf)
_, _, rq = ll.norm_fwd(qkv[:, :D], w, out=qn[:, :D])
rpair = ll.rmsnorm_pair_fwd(qkv, D, w, w, qn)
dq = torch.randn(M, 3 * D, device=dev).to(bf)
ybr = torch.randn(M, D, device=dev).to(bf); g = torch.ones(D, device=dev, dtype=bf)
dg = torch.zeros(D, device=dev); dcs = torch.zeros(D, device=dev); rs = torch.ones(M, device=dev)
dh = torch.randn(M, 6144, device=dev).to(bf); dbh = torch.zeros(6144, device=dev)
z = torch.randn(M, C, device=dev).to(bf); tgt = torch.randn(M, C, device=dev).to(bf)
lw = torch.ones(C, device=dev, dtype=bf); lb = torch.zeros(C, device=dev, dtype=bf)
ls = torch.zeros(1, device=dev)
_, stats = ll.ln_l2_fwd(z, lw, lb, 1e-5, want_out=False, target=tgt, loss_sum=ls)
dwl = torch.zeros(C, device=dev); dbl = torch.zeros(C, device=dev); gd = torch.ones(1, device=dev)
B, n = 32, 417
src = torch.randn(B, n, D, device=dev); table = torch.randn(2049, D, device=dev).to(bf)
mask = torch.ones(B, 2049, dtype=torch.bool, device=dev); mask[:, :n] = False
idx, _ = ll.visible_indices(mask, n)
gout = torch.empty(B * n, D, device=dev, dtype=bf); tg = torch.zeros(2049, D, device=dev)
video = torch.randn(B, 3, 8, 224, 224, device=dev).to(bf)
N = 64 << 20
master = torch.randn(N, device=dev); m1 = torch.zeros(N, device=dev); m2 = torch.zeros(N, device=dev)
gr = torch.randn(N, device=dev).to(bf); pb = torch.empty(N, device=dev, dtype=bf)
MD, MC = M * D, M * C

# name, call, bytes per call
CASES = [
    ("rmsnorm fwd (fp32 stream)", lambda: ll.norm_fwd(x, w), MD * (4 + 2)),
    ("rmsnorm bwd (+dx_in, dweight)", lambda: ll.norm_bwd(dy, x, w, None, rstd, dx_in=dxin, dweight=dw), MD * (2 + 4 + 4 + 4)),
    ("layernorm fwd (fp32 x)", lambda: ll.norm_fwd(x, w, bias, eps=1e-5, layernorm=True), MD * (4 + 2)),
    ("layernorm bwd (dweight, dbias)",
     lambda: ll.norm_bwd(dy, x, w, lmean, lrstd, layernorm=True, dweight=dw, dbias=db), MD * (2 + 4 + 4)),
    ("q-norm fwd (strided bf16)", lambda: ll.norm_fwd(qkv[:, :D], w, out=qn[:, :D]), MD * (2 + 2)),
    ("q-norm bwd (in place)",
     lambda: ll.norm_bwd(dq[:, :D], qkv[:, :D], w, None, rq, dx_out=dq[:, :D], dweight=dw), MD * (2 + 2 + 2)),
    ("q+k-norm pair fwd", lambda: ll.rmsnorm_pair_fwd(qkv, D, w, w, qn), 2 * MD * (2 + 2)),
    ("q+k-norm pair bwd", lambda: ll.rmsnorm_pair_bwd(dq, qkv, D, w, w, rpair, dw, db), 2 * MD * (2 + 2 + 2)),
    ("rmsnorm bwd + layerscale bwd (fused)",
     lambda: ll.rmsnorm_bwd_layerscale(dy, x, w, rstd, dxin, ybr, g, dw, dg, dcs, rowscale=rs), MD * (2 + 4 + 4 + 2 + 4 + 2)),
    ("layerscale bwd", lambda: ll.layerscale_bwd(dxin, ybr, g, dg, dcs, rowscale=rs), MD * (4 + 2 + 2)),
    ("colsum bf16 (N = 6144)", lambda: ll.colsum(dh, out=dbh), M * 6144 * 2),
    ("decoder LN->L2->loss fwd", lambda: ll.ln_l2_fwd(z, lw, lb, 1e-5, want_out=False, target=tgt, loss_sum=ls), MC * (2 + 2)),
    ("decoder LN->L2->loss bwd", lambda: ll.ln_l2_bwd(z, lw, lb, stats, tgt, -2.0 / M, gd, dwl, dbl), MC * (2 + 2 + 2)),
    ("pos-embed gather-add", lambda: ll.gather_add(src, n * D, table, idx, n, 0, B, n, D, gout, n * D), MD * (4 + 2 + 2)),
    ("pos-embed gradient scatter", lambda: ll.scatter_add(src, n * D, idx, n, 0, B, n, D, tg), MD * (4 + 4 + 4)),
    ("visible-patch im2col", lambda: ll.im2col_visible(video, idx, 1, n - 1, 1, 14, 592), B * (n - 1) * 588 * 2 * 2),
    ("AdamW, 64 M params", lambda: ll.adamw_step(master, m1, m2, gr, pb, 1e-4, 0.9, 0.98, 1e-6, 0.05, 1), N * 28),
]

print(f"# {torch.cuda.get_device_name()}, power limit {power_limit()}, library {_lib.LIB_PATH}")
print(f"# {'entry point':40s} {'ms/call':>9s} {'GB/s':>8s}")
for name, call, nbytes in CASES:
    for _ in range(5):
        call()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.iters):
        call()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.iters
    print(f"  {name:40s} {ms:9.4f} {nbytes / ms / 1e6:8.0f}")
