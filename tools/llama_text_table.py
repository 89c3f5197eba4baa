"""Timings of InternVideo2-CLIP's LLaMA-7B text tower on one GPU, in one call that prints the card's name and power
limit: the text forward at 256 x 32 and 128 x 32 tokens (the 1B and 6B recipes' per-GPU batches) against transformers'
LlamaModel in bf16 with the same weights (alternated over three windows), the SwiGLU GEMM against the plain N = 2I GEMM
plus a separate silu * up, the RoPE kernel's bandwidth, and the InternVideo2_CLIP-1B recipe step (frozen 1B vision at
8 x 224^2, frozen text, projector trained) split into vision and text.  Weights are random, built on the device.

    python tools/llama_text_table.py [--out results.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from internvideo_b200 import lowlevel as ll  # noqa: E402
from internvideo_b200.llama_modules import LLAMA_7B, LLaMA, rope_tables  # noqa: E402

bf = torch.bfloat16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def build_7b():
    with torch.device("meta"):
        model = LLaMA(use_lora=False, config=LLAMA_7B).bfloat16()
    model = model.to_empty(device="cuda").requires_grad_(False)
    g = torch.Generator(device="cuda").manual_seed(0)
    for k, p in model.named_parameters():
        if k.endswith("norm.weight"):
            p.fill_(1.0)
        else:
            p.copy_(torch.randn(p.shape, generator=g, device="cuda") * 0.02)
    return model


def hf_twin(model):
    """transformers' LlamaModel on the port's own parameter tensors (assign=True: no copy)."""
    from transformers import LlamaConfig, LlamaModel
    cfg = LlamaConfig(**{k: v for k, v in LLAMA_7B.items() if k not in ("architectures", "model_type")})
    with torch.device("meta"):
        hf = LlamaModel(cfg)
    sd = {k[len("transformer."):]: v for k, v in model.state_dict().items() if k.startswith("transformer.")}
    hf.load_state_dict(sd, strict=True, assign=True)
    hf.rotary_emb = hf.rotary_emb.__class__(cfg, device="cuda")
    return hf.eval().requires_grad_(False)


def ids_for(B, L, V=LLAMA_7B["vocab_size"], seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(3, V, (B, L), generator=g, device="cuda")
    lengths = torch.randint(L // 2, L + 1, (B,), generator=g, device="cuda")
    return ids * (torch.arange(L, device="cuda")[None] < lengths[:, None])


def text_table(model, hf, res):
    proj = model.text_projection

    def ref(ids):       # internvideo2_clip_text.py:45-52 through HF
        m = ids > 0
        x = hf(input_ids=ids, attention_mask=m).last_hidden_state
        return x[torch.arange(x.shape[0], device=ids.device), m.sum(1) - 1] @ proj
    for B in (256, 128):
        ids = ids_for(B, 32)
        with torch.no_grad():
            a, b = model(ids), ref(ids)
            ours, theirs = [], []
            for _ in range(3):
                ours.append(timed(lambda: model(ids), 5))
                theirs.append(timed(lambda: ref(ids), 5))
        rel = float((a.float() - b.float()).norm() / b.float().norm())
        flops = 2.0 * B * 32 * (sum(p.numel() for n, p in model.named_parameters() if "layers" in n))
        res[f"text_{B}x32"] = dict(ivb_ms=min(ours), hf_ms=min(theirs), ratio_hf_over_ivb=min(theirs) / min(ours),
                                   ivb_windows=ours, hf_windows=theirs, rel_diff_vs_hf=rel,
                                   layer_gemm_tflops=flops / min(ours) / 1e9)
        print(f"text {B}x32: ivb {min(ours):.1f} ms, HF {min(theirs):.1f} ms (x{min(theirs) / min(ours):.2f}), "
              f"rel diff {rel:.2e}", flush=True)


def swiglu_table(res, M=8192, D=4096, I=11008):
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn((M, D), generator=g, device="cuda").to(bf)
    w = (torch.randn((2 * I, D), generator=g, device="cuda") * 0.02).to(bf)
    fused = lambda: ll.gemm(x, w, epi=ll.EPI_SWIGLU)  # noqa: E731

    def split():
        h = ll.gemm(x, w)
        return torch.nn.functional.silu(h[:, :I]) * h[:, I:]
    fused(), split()
    tf, ts = timed(fused, 20), timed(split, 20)
    tp = timed(lambda: ll.gemm(x, w), 20)
    fl = 2.0 * M * 2 * I * D
    res["swiglu_8192"] = dict(fused_ms=tf, plain_gemm_ms=tp, gemm_plus_silu_mul_ms=ts, fused_tflops=fl / tf / 1e9)
    print(f"SwiGLU M=8192: fused {tf:.3f} ms ({fl / tf / 1e9:.0f} TFLOP/s), plain GEMM {tp:.3f}, "
          f"GEMM + silu*mul {ts:.3f}", flush=True)


def rope_table(res, B=256, L=32, H=32, d=128):
    qkv = torch.randn((B * L, 3 * H * d), device="cuda").to(bf)
    cos, sin = rope_tables(L, d, 10000.0, "cuda")
    f = lambda: ll._rope_qk(qkv[:, :H * d], qkv[:, H * d:2 * H * d], B, L, H, d, cos, sin)  # noqa: E731
    f()
    t = timed(f, 50)
    gb = 2 * 2 * B * L * H * d * 2 / t / 1e6      # q and k read and written
    res["rope_256x32"] = dict(ms=t, gbps=gb)
    print(f"RoPE 256x32: {t * 1e3:.1f} us, {gb:.0f} GB/s", flush=True)


def recipe_table(text, res, B=128):
    from internvideo_b200.clip_modules import InternVideo2_CLIP
    ve = dict(in_chans=3, patch_size=14, img_size=224, qkv_bias=False, drop_path_rate=0.0, head_drop_path_rate=0.0,
              embed_dim=1408, num_heads=16, mlp_ratio=48 / 11, init_values=0.1, qk_normalization=True, depth=40,
              use_flash_attn=True, use_fused_rmsnorm=True, use_fused_mlp=True, fused_mlp_heuristic=1,
              attn_pool_num_heads=16, clip_embed_dim=768, layerscale_no_force_fp32=True, num_frames=8, tubelet_size=1,
              sep_pos_embed=False, use_checkpoint=False, checkpoint_num=0)
    cfg = dict(model=dict(vision_encoder=ve, temp=0.01, temp_min=0.01, freeze_vision=True,
                          open_vision_clip_projector=True, freeze_text=True, open_text_projection=False))
    with torch.device("cuda"):
        model = InternVideo2_CLIP(cfg, text_encoder=text)
    model.bfloat16()
    image = torch.randn((B, 8, 3, 224, 224), device="cuda").to(bf)
    ids, idx = ids_for(B, 32), torch.arange(B, device="cuda")

    def step():
        model(image, ids, idx)["loss_vtc"].backward()
    step()
    t = timed(step, 3)
    with torch.no_grad():
        tv = timed(lambda: model.encode_vision(image), 3)
        tt = timed(lambda: model.encode_text(ids), 3)
    res[f"clip1b_step_{B}"] = dict(step_ms=t, vision_fwd_ms=tv, text_fwd_ms=tt)
    print(f"InternVideo2_CLIP-1B step, batch {B}: {t:.0f} ms (vision forward {tv:.0f} ms, text forward {tt:.0f} ms)",
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="", help="also write the results as JSON to this file")
    args = ap.parse_args()
    res = {"card": card()}
    print(res["card"], flush=True)
    model = build_7b()
    with torch.no_grad():
        model(ids_for(2, 32))          # joins gate and up before the twin takes the tensors
    text_table(model, hf_twin(model), res)
    torch.cuda.empty_cache()
    swiglu_table(res)
    rope_table(res)
    torch.cuda.empty_cache()
    recipe_table(model, res)
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
