"""InternVideo-Next-L/14 on the H100, in one call that also prints the card name and power limit:
  1. the encoder at 16 x 224^2 (n = 4 + 16 * 256 = 4 100 tokens): the forward with projected=True under no_grad, and
     forward + backward (a fixed-weight sum of the patch tokens), ms per call and per clip over CUDA events; the
     library's encoder against the staged unmodified reference module (oracle/_ref/, filled by
     oracle/internvideo_next.stage at build time) on its naive path under bf16 autocast, the two arms alternated in
     windows.  The reference's attention materialises the n x n scores of every head, so it runs at a smaller batch;
  2. the front end alone, ms per launch: the pre-norm im2col against the plain im2col at the same shape, and the two
     launches the backward adds for norm_before: the dgrad GEMM of the im2col rows and the weight-gradient kernel.

    python tools/next_table.py [--batch 4] [--ref-batch 1] [--steps 3] [--rounds 3] [--iters 50]
"""
import argparse
import contextlib
import io
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import card, timed  # noqa: E402
from internvideo_b200 import internvideo_next as nx  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402

bf = torch.bfloat16
T, RES, P = 16, 224, 14
N = T * (RES // P) ** 2


def _video(B):
    g = torch.Generator(device="cuda").manual_seed(0)
    return torch.randn(B, 3, T, RES, RES, device="cuda", generator=g).to(bf)


def _arms(model, B, autocast):
    x = _video(B)
    ctx = (lambda: torch.autocast("cuda", dtype=bf)) if autocast else contextlib.nullcontext
    x = x.float() if autocast else x

    def fwd():
        with torch.no_grad(), ctx():
            model(x, projected=True)

    def fwd_bwd():
        model.zero_grad(set_to_none=True)
        with ctx():
            out = model(x)
        out.float().sum().backward()
    return fwd, fwd_bwd


def ours(B):
    torch.manual_seed(0)
    m = nx.internvideo_next_large_patch14_224(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False)
    return _arms(m.to(bf).cuda().train(), B, False)


def reference(B):
    from oracle import internvideo_next as on
    if not on.available():
        return None
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = on.build("internvideo_next_large_patch14_224")
    return _arms(m.cuda().train(), B, True)


def encoder_table(B, ref_B, steps, rounds):
    print(f"\n1. InternVideo-Next-L/14 at {T} x {RES}^2, n = {4 + N} tokens, DropPath 0.25 (ms per call; per clip in "
          f"brackets; {rounds} alternated windows of {steps} calls)")
    arms = {f"ivb200 B={B}": (ours(B), B)}
    ref = reference(ref_B)
    if ref is not None:
        arms[f"reference bf16 autocast B={ref_B}"] = (ref, ref_B)
    for i, what in enumerate(("forward, projected=True, no_grad", "forward + backward")):
        res = {k: [] for k in arms}
        for _ in range(rounds):
            for k, (fns, _) in arms.items():
                res[k].append(timed(fns[i], steps))
        print(f"  {what}")
        for k, v in res.items():
            b = arms[k][1]
            print(f"    {k:32s} min {min(v):9.1f} ({min(v) / b:8.1f} per clip)  max {max(v):9.1f}")
        if ref is not None:
            ko, kr = list(arms)
            print(f"    ivb200 / reference per clip (best windows): "
                  f"{(min(res[ko]) / arms[ko][1]) / (min(res[kr]) / arms[kr][1]):.3f}")
    if ref is None:
        print("  reference not staged (oracle/_ref/): its arm is not measured")
    del arms
    torch.cuda.empty_cache()


def front_table(B, iters, rounds):
    K, Kpad, D = 588, 592, 1024
    x = _video(B)
    idx = torch.arange(0, N + 1, device="cuda", dtype=torch.int32).repeat(B, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(1)
    w = (1 + 0.1 * torch.randn(K, device="cuda", generator=g)).to(bf)
    wp = (0.02 * torch.randn(D, Kpad, device="cuda", generator=g)).to(bf)
    demb = torch.randn(B * N, D, device="cuda", generator=g).to(bf)
    _, r = ll._im2col_prenorm(x, idx, 1, N, 1, P, Kpad, w)
    dcols = ll.gemm(demb, wp, b_t=True)
    forms = {
        "im2col_visible": lambda: ll.im2col_visible(x, idx, 1, N, 1, P, Kpad),
        "im2col_prenorm": lambda: ll._im2col_prenorm(x, idx, 1, N, 1, P, Kpad, w),
        "dgrad GEMM (dcols)": lambda: ll.gemm(demb, wp, b_t=True),
        "prenorm_wgrad": lambda: ll._prenorm_wgrad(x, idx, 1, N, 1, P, Kpad, r, dcols),
    }
    res = {k: [] for k in forms}
    for _ in range(rounds):
        for k, fn in forms.items():
            res[k].append(timed(fn, iters))
    M = B * N
    print(f"\n2. front end, {B} clips x {N} patches (M = {M}, K = {K}), ms per launch, min-max of {rounds} alternated "
          f"windows of {iters}")
    video_bytes, cols_bytes = x.numel() * 2, M * Kpad * 2
    for k, v in res.items():
        extra = ""
        if k.startswith("im2col"):
            extra = f"   {(video_bytes + cols_bytes) / min(v) / 1e6:.0f} GB/s of video read + rows written"
        print(f"  {k:20s} {min(v):.4f}-{max(v):.4f}{extra}")
    print(f"  the pre-norm front end adds {min(res['im2col_prenorm']) - min(res['im2col_visible']):.4f} ms forward and "
          f"{min(res['dgrad GEMM (dcols)']) + min(res['prenorm_wgrad']):.4f} ms backward")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--ref-batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/next_table.py measures on the GPU"
    print(f"GPU: {card()} (name, power limit, max SM clock)")
    encoder_table(a.batch, a.ref_batch, a.steps, a.rounds)
    front_table(a.batch, a.iters, a.rounds)


if __name__ == "__main__":
    main()
