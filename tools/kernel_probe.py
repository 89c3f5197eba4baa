"""Tiny driver for ncu captures: one launch each of the dominant kernels at cfg-2 shapes."""
import sys
sys.path.insert(0, ".")
import torch
from internvideo_b200 import lowlevel as ll

which = sys.argv[1] if len(sys.argv) > 1 else "all"
bf = torch.bfloat16
M = 13344
if which in ("gemm", "all"):
    a = torch.randn(M, 1408, device="cuda").to(bf); w = (torch.randn(6144, 1408, device="cuda") * 0.02).to(bf)
    b = torch.zeros(6144, device="cuda", dtype=bf)
    h = torch.empty(M, 6144, device="cuda", dtype=bf); g = torch.empty(M, 6144, device="cuda", dtype=bf)
    for _ in range(3):
        ll.gemm(a, w, epi=ll.EPI_BIAS_GELU, bias=b, out0=g, out1=h)          # fc1 + GELU (fwd)
    dy = torch.randn(M, 1408, device="cuda").to(bf)
    for _ in range(3):
        ll.gemm(dy, g, a_t=True, b_t=True)                                      # wgrad fc2
if which == "gelu":
    a = torch.randn(M, 1408, device="cuda").to(bf); w = (torch.randn(6144, 1408, device="cuda") * 0.02).to(bf)
    b = torch.zeros(6144, device="cuda", dtype=bf)
    h = torch.empty(M, 6144, device="cuda", dtype=bf); g = torch.empty(M, 6144, device="cuda", dtype=bf)
    dy = torch.randn(M, 1408, device="cuda").to(bf); w2 = (torch.randn(1408, 6144, device="cuda") * 0.02).to(bf)
    dh = torch.empty(M, 6144, device="cuda", dtype=bf)
    for _ in range(2):
        ll.gemm(a, w, epi=ll.EPI_BIAS_GELU, flags=ll.FLAG_GELU_SAVE_GRAD, bias=b, out0=g, out1=h)   # fc1 + erf-GELU, saves gelu'
        ll.gemm(dy, w2, b_t=True, epi=ll.EPI_GELU_BWD, flags=ll.FLAG_GELU_SAVE_GRAD, aux=h, out0=dh)  # dgrad * saved gelu'
        ll.gemm(a, w, out0=g)                                                                    # same shape, plain store
if which in ("attn", "all"):
    B, n, H, d = 32, 417, 16, 88
    D = H * d
    qkv = torch.randn(B * n, 3 * D, device="cuda").to(bf)
    dout = torch.randn(B * n, D, device="cuda").to(bf)
    dqkv = torch.empty_like(qkv)
    for _ in range(3):
        out, lse = ll.attn_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B, n, H, d, d ** -0.5)
        ll.attn_bwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], out, dout, lse, B, n, H, d, d ** -0.5,
                    dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])
torch.cuda.synchronize()
print("done")
if which == "norm":
    x = torch.randn(M, 1408, device="cuda"); w = torch.ones(1408, device="cuda", dtype=bf)
    dy = torch.randn(M, 1408, device="cuda").to(bf); dxin = torch.randn(M, 1408, device="cuda")
    ybr = torch.randn(M, 1408, device="cuda").to(bf)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(2):
        flush.zero_()
        y, _, rstd = ll.norm_fwd(x, w)
        dw = torch.zeros(1408, device="cuda")
        flush.zero_()
        ll.norm_bwd(dy, x, w, None, rstd, dx_in=dxin, dweight=dw)
        dg = torch.zeros(1408, device="cuda"); dcs = torch.zeros(1408, device="cuda")
        flush.zero_()
        ll.layerscale_bwd(dxin, ybr, w, dg, dcs)
    torch.cuda.synchronize()
    print("done")
