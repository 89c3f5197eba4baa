"""Every GEMM of the cfg-2 (InternVideo2-1B, B=32, n=417) training step as the step launches it: same shapes, operand
layouts, epilogues and flags, one row per launch of one block (forward qkv / proj / fc1 / fc2; backward dh, dn2, da,
dn1 and the four ACCUM wgrads) and of the CLIP (x6) and MAE (x4) decoder heads.

Columns (device time per launch, CUDA events, 50 launches after 3 warm-ups, same operands for every column):
  coop      the cooperative single-CTA kernel (IVB_FLAG_1CTA) with the real epilogue, its own BN choice
  pingpong  the ping-pong kernel (IVB_FLAG_PINGPONG) with the real epilogue
  default   what ivb_gemm_bf16 picks by itself (what the step runs)
  plain     the cooperative kernel with a plain EPI_BF16 epilogue (no bias, no out1, no aux) at its own BN
  plain128  the same at tile_n = 128
  pp plain  the ping-pong kernel with a plain EPI_BF16 epilogue: what the ping-pong kernel costs with its epilogue hidden
  cuBLAS    torch.matmul on the same operands (bf16 out)
coop - plain is a lower bound on the exposed epilogue time; plain128 - plain is the mainloop cost of the 128-wide tile;
pingpong - pp plain is the epilogue time the ping-pong kernel leaves exposed.
A second table runs fwd fc1 on the ping-pong kernel with its epilogue taken apart (bias only; tanh-GELU without and with
the pre-activation output; with GELU'(h) saved; the erf forms), which separates the cost of the stores, of the MUFU work
and of the epilogue's code length.
Per-step totals weight each row by its launches per step (x40 blocks, x6 / x4 heads).  With a library that has no
ping-pong kernel the pingpong column is left out.
usage: python tools/gemm_table.py > gemm_table.md"""
import subprocess
import sys

sys.path.insert(0, ".")
import torch
from internvideo_b200 import lowlevel as ll
from internvideo_b200._lib import IvbError

bf, f32 = torch.bfloat16, torch.float32
M, Mm, D, HD, DEPTH, CLIP_K, MAE_K = 13344, 13312, 1408, 6144, 40, 6, 4   # Mm = 32 x 416 MAE decoder rows
GELU_TRAIN = ll.FLAG_GELU_TANH | ll.FLAG_GELU_SAVE_GRAD


def timeit(fn, iters=50, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def rnd(*shape, scale=1.0, dtype=bf):
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


def has_pingpong():
    """A library with the ping-pong kernel refuses IVB_FLAG_PINGPONG together with IVB_FLAG_1CTA."""
    a = rnd(128, 64)
    try:
        ll.gemm(a, a, flags=ll.FLAG_PINGPONG | ll.FLAG_1CTA)
    except IvbError:
        return True
    return False


def cases():
    """(name, launches per step, operands a, b, a_t, b_t, real-epilogue kwargs)."""
    x, a_in, n2 = rnd(M, D), rnd(M, D), rnd(M, D)
    g = rnd(M, HD)
    qkvw, projw, fc1w, fc2w = rnd(3 * D, D, scale=0.02), rnd(D, D, scale=0.02), rnd(HD, D, scale=0.02), rnd(D, HD, scale=0.02)
    qkvb, projb, fc1b, fc2b, gam = rnd(3 * D, scale=0.1), rnd(D, scale=0.1), rnd(HD, scale=0.1), rnd(D, scale=0.1), rnd(D, scale=0.1)
    resid = torch.randn(M, D, device="cuda")
    rs = (torch.rand(M, device="cuda") > 0.25).float() / 0.75
    y = torch.empty(M, D, device="cuda", dtype=bf)
    h = torch.empty(M, HD, device="cuda", dtype=bf)
    dy, dhh, dqkv = rnd(M, D), rnd(M, HD), rnd(M, 3 * D)
    gw = {k: torch.zeros(s, device="cuda", dtype=bf) for k, s in
          (("qkv", (3 * D, D)), ("proj", (D, D)), ("fc1", (HD, D)), ("fc2", (D, HD)))}
    cw, cb, xc = rnd(3200, D, scale=0.02), rnd(3200, scale=0.1), rnd(M, D)
    dyc = rnd(M, 3200)
    mw0, mb0, mw1, mb1, xm = rnd(D, D, scale=0.02), rnd(D, scale=0.1), rnd(D, D, scale=0.02), rnd(D, scale=0.1), rnd(Mm, D)
    hm = torch.empty(Mm, D, device="cuda", dtype=bf)
    dym = rnd(Mm, D)
    resid_out = torch.empty(M, D, device="cuda", dtype=f32)
    B = DEPTH
    return [
        ("fwd qkv", B, x, qkvw, False, False, dict(bias=qkvb)),
        ("fwd proj", B, a_in, projw, False, False,
         dict(epi=ll.EPI_RESID, bias=projb, gamma=gam, aux=resid, out1=y, rowscale=rs, out0=resid_out)),
        ("fwd fc1", B, n2, fc1w, False, False, dict(epi=ll.EPI_BIAS_GELU, flags=GELU_TRAIN, bias=fc1b, out1=h)),
        ("fwd fc2", B, g, fc2w, False, False,
         dict(epi=ll.EPI_RESID, bias=fc2b, gamma=gam, aux=resid, out1=y, rowscale=rs, out0=resid_out)),
        ("bwd dh", B, dy, fc2w, False, True, dict(epi=ll.EPI_GELU_BWD, flags=GELU_TRAIN, aux=h)),
        ("bwd dn2", B, dhh, fc1w, False, True, dict()),
        ("bwd da", B, dy, projw, False, True, dict()),
        ("bwd dn1", B, dqkv, qkvw, False, True, dict()),
        ("wgrad fc2", B, dy, g, True, True, dict(flags=ll.FLAG_ACCUM, out0=gw["fc2"])),
        ("wgrad fc1", B, dhh, n2, True, True, dict(flags=ll.FLAG_ACCUM, out0=gw["fc1"])),
        ("wgrad proj", B, dy, a_in, True, True, dict(flags=ll.FLAG_ACCUM, out0=gw["proj"])),
        ("wgrad qkv", B, dqkv, x, True, True, dict(flags=ll.FLAG_ACCUM, out0=gw["qkv"])),
        ("clip head fwd", CLIP_K, xc, cw, False, False, dict(bias=cb)),
        ("clip head dgrad", CLIP_K, dyc, cw, False, True, dict()),
        ("clip head wgrad", CLIP_K, dyc, xc, True, True, dict()),
        ("mae fc0 fwd", MAE_K, xm, mw0, False, False, dict(epi=ll.EPI_BIAS_GELU, bias=mb0, out1=hm)),
        ("mae fc1 fwd", MAE_K, hm, mw1, False, False, dict(bias=mb1)),
        ("mae dgrad", 2 * MAE_K, dym, mw1, False, True, dict()),
        ("mae wgrad", 2 * MAE_K, dym, xm, True, True, dict()),
    ]


def shape(a, b, a_t, b_t):
    m, k = (a.shape[1], a.shape[0]) if a_t else a.shape
    n = b.shape[1] if b_t else b.shape[0]
    return m, n, k


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    pp = has_pingpong()
    cols = ["coop"] + (["pingpong"] if pp else []) + ["default", "plain", "plain128"] + (["pp plain"] if pp else []) \
        + ["cuBLAS"]
    print(f"# libivb200 GEMMs of the cfg-2 step, one launch each (ms, CUDA events)\n\nGPU: {card} "
          f"(name, power limit, max SM clock)\n")
    print("| GEMM | per step | M x N x K | " + " | ".join(cols) + " | coop-plain | plain128-plain |"
          + (" pingpong-pp plain | pingpong/coop |" if pp else ""))
    print("|---|---|---|" + "---|" * (len(cols) + 2 + 2 * pp))
    tot = dict.fromkeys(cols, 0.0)
    tot_epi = tot_pen = 0.0
    tflop = 0.0
    for name, per_step, a, b, a_t, b_t, kw in cases():
        m, n, k = shape(a, b, a_t, b_t)
        kw = dict(kw)
        flags = kw.pop("flags", 0)
        ta = a.t() if a_t else a
        tb = b if b_t else b.t()
        cout = torch.empty(m, n, device="cuda", dtype=bf)
        fns = {
            "coop": lambda: ll.gemm(a, b, a_t=a_t, b_t=b_t, flags=flags | ll.FLAG_1CTA, **kw),
            "pingpong": lambda: ll.gemm(a, b, a_t=a_t, b_t=b_t, flags=flags | ll.FLAG_PINGPONG, **kw),
            "default": lambda: ll.gemm(a, b, a_t=a_t, b_t=b_t, flags=flags, **kw),
            "plain": lambda: ll.gemm(a, b, a_t=a_t, b_t=b_t, flags=ll.FLAG_1CTA),
            "plain128": lambda: ll.gemm(a, b, a_t=a_t, b_t=b_t, flags=ll.FLAG_1CTA, tile_n=128),
            "pp plain": lambda: ll.gemm(a, b, a_t=a_t, b_t=b_t, flags=ll.FLAG_PINGPONG),
            "cuBLAS": lambda: torch.matmul(ta, tb, out=cout),
        }
        t = {c: timeit(fns[c]) for c in cols}
        for c in cols:
            tot[c] += per_step * t[c]
        tot_epi += per_step * (t["coop"] - t["plain"])
        tot_pen += per_step * (t["plain128"] - t["plain"])
        tflop += per_step * 2.0 * m * n * k / 1e12
        row = f"| {name} | {per_step} | {m} x {n} x {k} | " + " | ".join(f"{t[c]:.3f}" for c in cols)
        row += f" | {t['coop'] - t['plain']:+.3f} | {t['plain128'] - t['plain']:+.3f} |"
        if pp:
            row += f" {t['pingpong'] - t['pp plain']:+.3f} | {t['pingpong'] / t['coop']:.3f} |"
        print(row, flush=True)
    print("\nPer step (ms, each row x its launches per step; TFLOP/s = the step's GEMM flops / that time):\n")
    print("| | " + " | ".join(cols) + " |\n|---|" + "---|" * len(cols))
    print("| ms | " + " | ".join(f"{tot[c]:.1f}" for c in cols) + " |")
    print("| TFLOP/s | " + " | ".join(f"{tflop / tot[c] * 1e3:.0f}" for c in cols) + " |")
    print(f"\nExposed epilogue (coop - plain): {tot_epi:.1f} ms/step; 128-wide tile penalty (plain128 - plain): "
          f"{tot_pen:.1f} ms/step.")
    if pp:
        fc1_ablation()


def fc1_ablation():
    """fwd fc1 on the ping-pong kernel, one epilogue ingredient at a time (same operands, ms per launch)."""
    n2, fc1w, fc1b = rnd(M, D), rnd(HD, D, scale=0.02), rnd(HD, scale=0.1)
    h = torch.empty(M, HD, device="cuda", dtype=bf)
    PP, TANH, SAVE, GELU = ll.FLAG_PINGPONG, ll.FLAG_GELU_TANH, ll.FLAG_GELU_SAVE_GRAD, ll.EPI_BIAS_GELU
    rows = [
        ("plain EPI_BF16", dict()),
        ("bias", dict(bias=fc1b)),
        ("bias + GELU tanh", dict(epi=GELU, flags=TANH, bias=fc1b)),
        ("bias + GELU tanh, out1 = h", dict(epi=GELU, flags=TANH, bias=fc1b, out1=h)),
        ("bias + GELU tanh, out1 = GELU'(h) (the step's fc1)", dict(epi=GELU, flags=TANH | SAVE, bias=fc1b, out1=h)),
        ("bias + GELU erf", dict(epi=GELU, bias=fc1b)),
        ("bias + GELU erf, out1 = h", dict(epi=GELU, bias=fc1b, out1=h)),
        ("bias + GELU erf, out1 = GELU'(h)", dict(epi=GELU, flags=SAVE, bias=fc1b, out1=h)),
    ]
    print(f"\nfwd fc1 {M} x {HD} x {D} on the ping-pong kernel, epilogue taken apart (ms per launch):\n")
    print("| epilogue | ms | - plain |\n|---|---|---|")
    base = None
    for name, kw in rows:
        kw = dict(kw)
        flags = kw.pop("flags", 0) | PP
        t = timeit(lambda: ll.gemm(n2, fc1w, flags=flags, **kw))
        base = t if base is None else base
        print(f"| {name} | {t:.3f} | {t - base:+.3f} |", flush=True)


if __name__ == "__main__":
    main()
