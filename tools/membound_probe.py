"""One launch each of the memory-bound kernels at cfg-2 shapes (M = 32*417 rows, D = 1408, decoder width 3200,
1.07 B-parameter AdamW slice), for an `ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum` pass
(bytes over duration gives the achieved GB/s).  Inputs exceed the 50 MB L2
or the L2 is flushed before each launch."""
import sys
sys.path.insert(0, ".")
import torch
from internvideo_b200 import lowlevel as ll

bf, f32 = torch.bfloat16, torch.float32
M, D, C = 32 * 417, 1408, 3200
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def fl():
    flush.zero_()


x = torch.randn(M, D, device="cuda"); w = torch.ones(D, device="cuda", dtype=bf)
dy = torch.randn(M, D, device="cuda").to(bf); dxin = torch.randn(M, D, device="cuda")
for rep in range(2):
    fl(); y, _, rstd = ll.norm_fwd(x, w)                                                    # rms fwd (fp32 stream -> bf16)
    dw = torch.zeros(D, device="cuda", dtype=f32)
    fl(); ll.norm_bwd(dy, x, w, None, rstd, dx_in=dxin, dweight=dw)                          # rms bwd (+ residual grad in)
    qkv = torch.randn(M, 3 * D, device="cuda").to(bf); qn = torch.empty(M, D, device="cuda", dtype=bf)
    fl(); _, _, rq = ll.norm_fwd(qkv[:, :D], w, out=qn)                                      # q-norm fwd (strided bf16)
    dq = torch.randn(M, 3 * D, device="cuda").to(bf)
    fl(); ll.norm_bwd(dq[:, :D], qkv[:, :D], w, None, rq, dx_out=dq[:, :D], dweight=dw)      # q-norm bwd in place
    ybr = torch.randn(M, D, device="cuda").to(bf); g = torch.ones(D, device="cuda", dtype=bf)
    dg = torch.zeros(D, device="cuda", dtype=f32); dcs = torch.zeros(D, device="cuda", dtype=f32)
    rs = torch.ones(M, device="cuda")
    fl(); ll.layerscale_bwd(dxin, ybr, g, dg, dcs, rowscale=rs)                               # LayerScale bwd
    dh = torch.randn(M, 6144, device="cuda").to(bf); db = torch.zeros(6144, device="cuda", dtype=f32)
    fl(); ll.colsum(dh, out=db)                                                              # bias-gradient column sum
    z = torch.randn(M, C, device="cuda").to(bf); tgt = torch.randn(M, C, device="cuda").to(bf)
    lw = torch.ones(C, device="cuda", dtype=bf); lb = torch.zeros(C, device="cuda", dtype=bf)
    ls = torch.zeros(1, device="cuda")
    fl(); _, stats = ll.ln_l2_fwd(z, lw, lb, 1e-5, want_out=False, target=tgt, loss_sum=ls)  # decoder LN->L2->loss fwd
    dwl = torch.zeros(C, device="cuda"); dbl = torch.zeros(C, device="cuda"); gd = torch.ones(1, device="cuda")
    fl(); ll.ln_l2_bwd(z, lw, lb, stats, tgt, -2.0 / M, gd, dwl, dbl)                        # ... bwd
    B, n = 32, 417
    src = torch.randn(B, n, D, device="cuda"); table = torch.randn(2049, D, device="cuda").to(bf)
    mask = torch.ones(B, 2049, dtype=torch.bool, device="cuda"); mask[:, :n] = False
    idx, _ = ll.visible_indices(mask, n)
    out = torch.empty(B * n, D, device="cuda", dtype=bf)
    fl(); ll.gather_add(src, n * D, table, idx, n, 0, B, n, D, out, n * D)                    # decoder pos-embed gather-add
    tg = torch.zeros(2049, D, device="cuda")
    fl(); ll.scatter_add(src, n * D, idx, n, 0, B, n, D, tg)                                  # pos-embed gradient scatter
    video = torch.randn(B, 3, 8, 224, 224, device="cuda").to(bf)
    fl(); ll.im2col_visible(video, idx, 1, n - 1, 1, 14, 592)                                 # visible-patch im2col
    N = 64 << 20
    master = torch.randn(N, device="cuda"); m1 = torch.zeros(N, device="cuda"); m2 = torch.zeros(N, device="cuda")
    gr = torch.randn(N, device="cuda").to(bf); pb = torch.empty(N, device="cuda", dtype=bf)
    fl(); ll.adamw_step(master, m1, m2, gr, pb, 1e-4, 0.9, 0.98, 1e-6, 0.05, 1)               # AdamW, 64 M params
torch.cuda.synchronize()
print("done")
