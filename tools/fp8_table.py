"""FP8 mode of the ViT block on the H100: where its time goes, in one call.

Prints, with the card name and power limit:
  1. the eight forward / input-gradient GEMMs of a cfg-2 block (M = 13 344 tokens): per-launch time of the bf16
     default, of the FP8 ping-pong kernel (accumulation in the tensor core), of the FP8 cooperative kernel (each k-block
     promoted to fp32) and of the FP8 default, and the accumulation-error ratio of the two FP8 forms
     (tests/test_gemm_fp8_gpu.py::accumulation_ratio, limit 0.25);
  2. the quantise calls of one block (ivb_fp8_quantize): time and achieved GB/s of the algorithmic bytes (bf16 read
     twice, for amax and for the cast, plus the fp8 write; a weight also writes its transposed copy) against the
     data-sheet 3.35 TB/s;
  3. the cfg-2 training step (B = 32, one CUDA graph) with FP8 off and on, alternated three times each.

    python tools/fp8_table.py [--no-step] [--iters 50]
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from internvideo_b200 import lowlevel as ll  # noqa: E402

M = 13344
HBM = 3.35e12
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
GEMMS = [  # name, N, K, A format (forward: E4M3 activations; dgrad: E5M2 gradients), bf16 layout of B
    ("qkv", 4224, 1408, E4, False), ("proj", 1408, 1408, E4, False), ("fc1", 6144, 1408, E4, False),
    ("fc2", 1408, 6144, E4, False), ("dh", 6144, 1408, E5, True), ("dn2", 1408, 6144, E5, True),
    ("da", 1408, 1408, E5, True), ("dn1", 1408, 4224, E5, True),
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


def gemm_table(iters):
    from test_gemm_fp8_gpu import accumulation_ratio
    print("\n1. GEMMs at M = 13344 (ms per launch; TFLOP/s; accumulation ratio, limit 0.25)")
    print(f"{'gemm':6s} {'N':>5s} {'K':>5s}  {'bf16':>7s}  {'fp8 pp':>7s}  {'fp8 coop':>8s}  {'fp8 dflt':>8s}"
          f"  {'TF bf16':>7s} {'TF fp8':>7s}  {'ratio pp':>8s} {'ratio coop':>10s}")
    tot = [0.0, 0.0]
    for name, N, K, fmt, bt in GEMMS:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = torch.randn((M, K), generator=g, device="cuda").to(torch.bfloat16)
        w = (torch.randn((N, K) if not bt else (K, N), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        qa, _, sa, _ = ll.fp8_quantize(a, ll.FP8_E5M2 if fmt == E5 else ll.FP8_E4M3)
        qw, qwt, sw, _ = ll.fp8_quantize(w, ll.FP8_E4M3, transpose=True)
        qb = qwt if bt else qw
        t_bf = timed(lambda: ll.gemm(a, w, b_t=bt), iters)
        t_pp = timed(lambda: ll.gemm_fp8(qa, sa, qb, sw, flags=ll.FLAG_PINGPONG), iters)
        t_co = timed(lambda: ll.gemm_fp8(qa, sa, qb, sw, flags=ll.FLAG_1CTA), iters)
        t_df = timed(lambda: ll.gemm_fp8(qa, sa, qb, sw), iters)
        r_pp = accumulation_ratio(N, K, fmt, flags=ll.FLAG_PINGPONG)
        r_co = accumulation_ratio(N, K, fmt, flags=ll.FLAG_1CTA)
        fl = 2.0 * M * N * K
        tot[0] += t_bf; tot[1] += t_df
        print(f"{name:6s} {N:5d} {K:5d}  {t_bf:7.3f}  {t_pp:7.3f}  {t_co:8.3f}  {t_df:8.3f}"
              f"  {fl / t_bf / 1e9:7.0f} {fl / t_df / 1e9:7.0f}  {r_pp:8.4f} {r_co:10.4f}")
    print(f"sum of the eight: bf16 {tot[0]:.3f} ms, fp8 default {tot[1]:.3f} ms per block")


def quant_table(iters):
    print("\n2. quantise calls of one block (ms; GB/s of the algorithmic bytes; share of 3.35 TB/s)")
    rows = [("n1", M, 1408, ll.FP8_E4M3, False), ("a", M, 1408, ll.FP8_E4M3, False), ("n2", M, 1408, ll.FP8_E4M3, False),
            ("g", M, 6144, ll.FP8_E4M3, False), ("dy2", M, 1408, ll.FP8_E5M2, False),
            ("dh", M, 6144, ll.FP8_E5M2, False), ("dy1", M, 1408, ll.FP8_E5M2, False),
            ("dqkv", M, 4224, ll.FP8_E5M2, False), ("Wqkv", 4224, 1408, ll.FP8_E4M3, True),
            ("Wproj", 1408, 1408, ll.FP8_E4M3, True), ("Wfc1", 6144, 1408, ll.FP8_E4M3, True),
            ("Wfc2", 1408, 6144, ll.FP8_E4M3, True)]
    tot_ms = tot_b = 0.0
    for name, R, C, fmt, tr in rows:
        x = torch.randn((R, C), device="cuda").to(torch.bfloat16)
        ms = timed(lambda: ll.fp8_quantize(x, fmt, transpose=tr), iters)
        nb = R * C * (2 + 2 + 1 + (1 if tr else 0))
        tot_ms += ms; tot_b += nb
        print(f"{name:6s} [{R:5d} x {C:5d}]{' +T' if tr else '   '}  {ms:7.3f} ms  {nb / ms / 1e6:7.0f} GB/s  "
              f"{nb / ms * 1e3 / HBM:5.1%}")
    print(f"total {tot_ms:.3f} ms for {tot_b / 1e9:.3f} GB ({tot_b / tot_ms / 1e6:.0f} GB/s; at 3.35 TB/s: "
          f"{tot_b / HBM * 1e3:.3f} ms)")


def step_table(reps=3, steps=10, modes=("off", "tensor"), skips=(True,)):
    """modes: "off" (bf16), a set_fp8 scaling or "token_wgrad" (scaling="token", wgrad=True); skips: the set_droppath_skip settings.  Each (mode, skip) pair is
    captured and timed once per repetition, in turn."""
    import bench
    from internvideo_b200.engine import GraphedStep, PretrainEngine
    from internvideo_b200.modules import PretrainInternVideo2, set_droppath_skip, set_fp8
    print("\n3. cfg-2 step, B = 32, one CUDA graph per step (alternated)")
    cfg = dict(bench.CFGS["1B"])
    B = cfg.pop("batch")
    T, L, keep = cfg["num_frames"], 256, 52
    n = 1 + T * keep
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = PretrainInternVideo2(drop_path_rate=0.25, clip_teacher_embed_dim=3200, clip_teacher_final_dim=768,
                                     mae_teacher_embed_dim=1408, init_values=1e-5, attn_pool_num_heads=16,
                                     clip_embed_dim=768, use_flash_attn=True, use_fused_rmsnorm=True,
                                     use_fused_mlp=True, **cfg)
    model = model.bfloat16().cuda().train()
    engine = PretrainEngine(model, clip_grad=3.0, check_finite=True)
    g = torch.Generator().manual_seed(1234)
    K, Km = cfg["clip_return_layer"], cfg["mae_return_layer"]
    video = torch.randn(B, 3, T, 224, 224, generator=g).to(torch.bfloat16).cuda()
    mask = bench.make_mask(B, T, L, keep, 1234).cuda()
    gd = torch.Generator(device="cuda").manual_seed(99)
    nrm = torch.nn.functional.normalize
    tc = nrm(torch.randn(K, B * n, 3200, device="cuda", generator=gd), dim=-1).to(torch.bfloat16)
    tf = nrm(torch.randn(B, 768, device="cuda", generator=gd), dim=-1).to(torch.bfloat16)
    tm = nrm(torch.randn(Km, B * (n - 1), 1408, device="cuda", generator=gd), dim=-1).to(torch.bfloat16)

    def step(v, m):
        engine.zero_grad()
        lc, lf, lm = model.forward_loss(v, m, tc, tf, tm, n_visible=n)
        loss = lc + lf + lm
        loss.backward()
        engine.step()
        return loss

    runs = [(fp8, skip) for fp8 in modes for skip in skips]
    label = {r: f"fp8={r[0]:6s}" + (f" skip={'on ' if r[1] else 'off'}" if len(skips) > 1 else "") for r in runs}
    res = {r: [] for r in runs}
    for _ in range(reps):
        for fp8, skip in runs:
            wgrad = fp8 == "token_wgrad"     # per-token FP8 with FP8 weight gradients
            set_fp8(model, fp8 != "off", scaling="tensor" if fp8 == "off" else "token" if wgrad else fp8, wgrad=wgrad)
            set_droppath_skip(model, skip)
            gs = GraphedStep(step, [video, mask], warmup=1)
            gs(video, mask)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                loss = gs(video, mask)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / steps
            res[(fp8, skip)].append(ms)
            print(f"  {label[(fp8, skip)]}  {ms:8.2f} ms/step  {B / ms * 1e3:7.2f} clips/s  loss {float(loss):.4f}")
            del gs
            torch.cuda.empty_cache()
    for r in runs:
        best = min(res[r])
        print(f"{label[r]}: best {best:.2f} ms/step = {B / best * 1e3:.2f} clips/s "
              f"(all: {', '.join(f'{x:.2f}' for x in res[r])})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    ll.device_check()
    print("card:", card())
    gemm_table(args.iters)
    quant_table(args.iters)
    if not args.no_step:
        step_table()


if __name__ == "__main__":
    main()
