"""FP8 inference of the frozen teachers on the H100 (modules.set_fp8_inference): where the time goes, in one call.

Prints, with the card name and power limit:
  1. the teachers' eight forward GEMMs at B = 32 (InternVL-6B: M = 32 x 8 x 257 = 65 792; VideoMAEv2-g: M = 32 x 2048 =
     65 536), each with the fused epilogue the teacher's block gives it: ms per launch and TFLOP/s of bf16, of
     per-tensor FP8 (scalar scales) and of vector-scale FP8 (per-token activation scales, per-channel weight scales) on
     the library's default kernel (named), and of vector-scale FP8 forced onto each kernel form;
  2. the activation casts of one block of each teacher: per-tensor (norm_fwd to bf16, then fp8_quantize of n1 and n2;
     fp8_quantize of a and g) against per-token (norm_fwd_fp8 of n1 and n2; fp8_quantize_rows of a and g): ms and
     achieved GB/s of the algorithmic bytes against the data-sheet 3.35 TB/s;
  3. each whole teacher forward at B = 32, built as `bench.py --with-teachers` builds them (random init), in the modes
     bf16, set_fp8 (InternVL only) and set_fp8_inference, alternated three times.

    python tools/teacher_fp8_table.py [--iters 20] [--no-teachers]
"""
import argparse
import os
import subprocess
import sys
import time
from functools import partial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from internvideo_b200 import lowlevel as ll  # noqa: E402

HBM = 3.35e12
IVL_M, MAE_M = 32 * 8 * 257, 32 * 2048
GEMMS = [  # (teacher, name, M, N, K)
    ("ivl", "qkv", IVL_M, 9600, 3200), ("ivl", "proj", IVL_M, 3200, 3200), ("ivl", "fc1", IVL_M, 12800, 3200),
    ("ivl", "fc2", IVL_M, 3200, 12800), ("mae", "qkv", MAE_M, 4224, 1408), ("mae", "proj", MAE_M, 1408, 1408),
    ("mae", "fc1", MAE_M, 6144, 1408), ("mae", "fc2", MAE_M, 1408, 6144),
]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _epilogue(t, name, M, N):
    """The fused epilogue the teacher's block gives this GEMM (ops.block_forward, RMSNorm or LayerNorm form): InternVL
    qkv without bias, proj and fc2 into the residual stream with LayerScale gamma, fc1 with tanh GELU; VideoMAE-g qkv
    with the q/v bias, proj and fc2 into the stream without gamma (init_values 0), fc1 with erf GELU."""
    bias = (torch.randn(N, device="cuda") * 0.02).to(torch.bfloat16)
    gamma = torch.full((N,), 0.1, device="cuda", dtype=torch.bfloat16) if t == "ivl" else None
    if name == "qkv":
        return dict(epi=ll.EPI_BF16, bias=bias if t == "mae" else None)
    if name == "fc1":
        return dict(epi=ll.EPI_BIAS_GELU, bias=bias, flags=ll.FLAG_GELU_TANH if t == "ivl" else 0)
    return dict(epi=ll.EPI_RESID, bias=bias, gamma=gamma, aux=torch.randn((M, N), device="cuda"))


def gemm_table(iters):
    print("\n1. forward GEMMs at B = 32 with the teachers' fused epilogues (ms per launch; TFLOP/s for the defaults)")
    print("   kernel: the one the library selects by default (pp = ping-pong, coop = cooperative); the last two columns")
    print("   force each form for the per-token GEMM")
    print(f"{'gemm':9s} {'M':>6s} {'N':>6s} {'K':>6s} {'kernel':>6s}  {'bf16':>13s}  {'fp8 tensor':>13s}  "
          f"{'fp8 token':>13s}  {'token pp':>8s}  {'token coop':>10s}")
    tot = {}
    for t, name, M, N, K in GEMMS:
        a = torch.randn((M, K), device="cuda").to(torch.bfloat16)
        b = (torch.randn((N, K), device="cuda") * 0.02).to(torch.bfloat16)
        qa, _, sa, _ = ll.fp8_quantize(a, ll.FP8_E4M3)
        qb, _, sb, _ = ll.fp8_quantize(b, ll.FP8_E4M3)
        ra, va = ll.fp8_quantize_rows(a)
        rb, vb = ll.fp8_quantize_rows(b)
        kw = _epilogue(t, name, M, N)
        flags = kw.pop("flags", 0)
        out = torch.empty((M, N), device="cuda", dtype=torch.float32 if kw["epi"] == ll.EPI_RESID else torch.bfloat16)
        ms = [timed(lambda: ll.gemm(a, b, out0=out, flags=flags, **kw), iters),
              timed(lambda: ll.gemm_fp8(qa, sa, qb, sb, out0=out, flags=flags, **kw), iters),
              timed(lambda: ll.gemm_fp8(ra, va, rb, vb, out0=out, flags=flags, **kw), iters)]
        forced = [timed(lambda: ll.gemm_fp8(ra, va, rb, vb, out0=out, flags=flags | ll.FLAG_PINGPONG, **kw), iters),
                  timed(lambda: ll.gemm_fp8(ra, va, rb, vb, out0=out, flags=flags | ll.FLAG_1CTA, **kw), iters)]
        fl = 2.0 * M * N * K
        for i, m in enumerate(ms):
            tot[(t, i)] = tot.get((t, i), 0.0) + m
        print(f"{t + ' ' + name:9s} {M:6d} {N:6d} {K:6d} {default_kernel(M, N, K):>6s}  " +
              "  ".join(f"{m:6.3f} {fl / m / 1e9:6.0f}" for m in ms) + f"  {forced[0]:8.3f}  {forced[1]:10.3f}")
        del a, b, qa, qb, ra, rb, out, kw
    for t in ("ivl", "mae"):
        print(f"{t} block total: bf16 {tot[(t, 0)]:.3f} ms, fp8 tensor {tot[(t, 1)]:.3f} ms, "
              f"fp8 token {tot[(t, 2)]:.3f} ms")


def default_kernel(M, N, K):
    """The FP8 kernel ivb_gemm_fp8 selects without a forcing flag: ping-pong where it has more 128 x 128 tiles than the
    card has SMs, unless K >= 8192 and its cooperative tile choice is 256 wide (ivb_gemm.cu, use_pingpong; the FP8
    cooperative kernel then runs at BN 192 or 128)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = ((M + 127) // 128) * ((N + 127) // 128)
    if tiles <= sms:
        return "coop"
    best, best_bn, num_m = 1e30, 256, (M + 127) // 128
    for bn in (256, 192, 176, 128):
        waves = (num_m * ((N + bn - 1) // bn) + sms - 1) // sms
        cost = waves * bn * (1.0 if bn >= 176 else 1.15)
        if cost < best - 1e-9:
            best, best_bn = cost, bn
    return "coop" if K >= 8192 and best_bn == 256 else "pp"


def cast_table(iters):
    print("\n2. activation casts of one block at B = 32 (ms; GB/s of the algorithmic bytes, % of 3.35 TB/s)")
    for t, M, D, Hd, ln in (("ivl", IVL_M, 3200, 12800, False), ("mae", MAE_M, 1408, 6144, True)):
        x = torch.randn((M, D), device="cuda")
        w = torch.ones(D, device="cuda", dtype=torch.bfloat16)
        bias = torch.zeros(D, device="cuda", dtype=torch.bfloat16) if ln else None
        a = torch.randn((M, D), device="cuda").to(torch.bfloat16)
        g = torch.randn((M, Hd), device="cuda").to(torch.bfloat16)
        rows = [  # (what, per-tensor fn, its bytes, per-token fn, its bytes)
            ("n1/n2", lambda: ll.fp8_quantize(ll.norm_fwd(x, w, bias, layernorm=ln, want_stats=False)[0]),
             M * D * (4 + 2 + 2 * 2 + 1), lambda: ll.norm_fwd_fp8(x, w, bias, layernorm=ln), M * D * (4 + 1)),
            ("a", lambda: ll.fp8_quantize(a), M * D * 5, lambda: ll.fp8_quantize_rows(a), M * D * 3),
            ("g", lambda: ll.fp8_quantize(g), M * Hd * 5, lambda: ll.fp8_quantize_rows(g), M * Hd * 3),
        ]
        per_t = per_r = 0.0
        for what, ft, bt, fr, br in rows:
            mt, mr = timed(ft, iters), timed(fr, iters)
            k = 2 if what == "n1/n2" else 1
            per_t += k * mt; per_r += k * mr
            print(f"{t} {what:6s} per-tensor {mt:6.3f} ms {bt / mt / 1e6:6.0f} GB/s ({bt / mt / 1e9 / HBM * 1e12:4.0%})"
                  f"   per-token {mr:6.3f} ms {br / mr / 1e6:6.0f} GB/s ({br / mr / 1e9 / HBM * 1e12:4.0%})")
        print(f"{t} block (n1, a, n2, g): per-tensor {per_t:.3f} ms, per-token {per_r:.3f} ms "
              "(per-tensor includes the bf16 norm the FP8 path does not need)")
        del x, a, g


def teachers_table(reps):
    from internvideo_b200.modules import set_fp8, set_fp8_inference
    from internvideo_b200.teachers import InternVL_CLIP, VisionTransformer
    print("\n3. whole teacher forwards at B = 32 (ms; modes alternated)")
    B, T = 32, 8
    torch.manual_seed(0)
    with torch.device("cuda"):
        clip_t = InternVL_CLIP(img_size=224, layerscale_no_force_fp32=False, clip_return_layer=6, clip_return_interval=1)
        mae_t = VisionTransformer(img_size=224, patch_size=14, embed_dim=1408, depth=40, num_heads=16, mlp_ratio=48 / 11,
                                  qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), all_frames=2 * T,
                                  tubelet_size=2, mae_return_layer=4, mae_return_interval=1)
    clip_t = clip_t.bfloat16().cuda().eval(); mae_t = mae_t.bfloat16().cuda().eval()
    video = torch.randn((B, 3, 2 * T, 224, 224), device="cuda").to(torch.bfloat16)
    clip_video = video[:, :, ::2]

    def run(model, v):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = model(v)
        torch.cuda.synchronize()
        del out
        return (time.perf_counter() - t0) * 1e3

    modes = {"ivl": ["bf16", "set_fp8", "fp8_inference"], "mae": ["bf16", "fp8_inference"]}
    res = {(t, m): [] for t in modes for m in modes[t]}
    for t, model, v in (("ivl", clip_t, clip_video), ("mae", mae_t, video)):
        for rep in range(reps + 1):          # the first round warms every mode up and is not reported
            for mode in modes[t]:
                set_fp8_inference(model, False); set_fp8(model, False)
                if mode == "set_fp8":
                    set_fp8(model, True)
                elif mode == "fp8_inference":
                    set_fp8_inference(model, True)
                ms = run(model, v)
                if rep > 0:
                    res[(t, mode)].append(ms)
        set_fp8_inference(model, False); set_fp8(model, False)
    for (t, mode), v in res.items():
        print(f"{t} {mode:14s} " + " / ".join(f"{m:8.1f}" for m in v) + " ms")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-teachers", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("teacher_fp8_table.py measures on the GPU: no CUDA device")
    print("card (name, power limit, max SM clock):", card())
    with torch.no_grad():
        gemm_table(args.iters)
        cast_table(args.iters)
        torch.cuda.empty_cache()
        if not args.no_teachers:
            teachers_table(args.reps)


if __name__ == "__main__":
    main()
