"""GPU-side anchors for the headline number (BASELINE.md §4 comparators, reported, not the reference arm): the UNMODIFIED
reference PretrainInternVideo2-1B on the same GPU, bf16, training step (fwd + bwd + torch fused AdamW):
  reference-naive : the reference's pure-PyTorch path (use_flash_attn = use_fused_* = False)
  reference-flash : the reference's FlashAttention class (FA2) with its all-or-nothing fused flags on; FA2's
                    DropoutAddRMSNorm / FusedMLP extensions are not installed in this image, so they are provided by
                    the reference's OWN RMSNorm / Mlp wrapped to the fused calling convention (SURVEY §8c).
Needs the reference sources: /root/reference, or the copies oracle/stage_ref.py staged under oracle/_ref/.
  python tools/ref_gpu_compare.py [--batch 8] > reference_gpu_comparators.log"""
import argparse
import sys
import time

sys.path.insert(0, ".")
import torch
import torch.nn as nn

import bench
from oracle import ref_shim

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--steps", type=int, default=4)
a = ap.parse_args()
assert ref_shim.available(), "reference sources not found (run oracle/stage_ref.py where /root/reference is mounted)"
mod = ref_shim.import_single_modality()
cfg = dict(bench.CFGS["1B"]); cfg.pop("batch")
T, keep = cfg["num_frames"], 52
n = 1 + T * keep


class FusedNormAdapter(mod.RMSNorm):
    """DropoutAddRMSNorm(prenorm=True) calling convention on the reference's own RMSNorm: (x, residual) -> (norm(x+res), x+res)."""

    def __init__(self, hidden_size, eps=1e-6, prenorm=True, **_):
        super().__init__(hidden_size, eps=eps)

    def forward(self, x, residual=None):
        res = x if residual is None else x + residual
        return super().forward(res), res


class FusedMLPAdapter(mod.Mlp):
    """flash_attn FusedMLP(in, hidden, heuristic): Linear - tanh-GELU - Linear."""

    def __init__(self, in_features, hidden_features, heuristic=None, **_):
        super().__init__(in_features, hidden_features, act_layer=lambda: nn.GELU(approximate="tanh"))


def build(flash):
    torch.manual_seed(0)
    kw = dict(drop_path_rate=0.25, init_values=1e-5, clip_teacher_embed_dim=3200, clip_teacher_final_dim=768,
              mae_teacher_embed_dim=1408, attn_pool_num_heads=16, clip_embed_dim=768, **cfg)
    if flash:
        mod.DropoutAddRMSNorm, mod.FusedMLP = FusedNormAdapter, FusedMLPAdapter
    import contextlib, io
    with contextlib.redirect_stdout(io.StringIO()), torch.device("cuda"):
        m = mod.PretrainInternVideo2(use_flash_attn=flash, use_fused_rmsnorm=flash, use_fused_mlp=flash, **kw)
    return m.bfloat16().cuda().train()


def run(flash, B):
    model = build(flash)
    opt = torch.optim.AdamW(model.parameters(), lr=1.5e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.05, fused=True)
    g = torch.Generator(device="cuda").manual_seed(1)
    video = torch.randn(B, 3, T, 224, 224, device="cuda", generator=g).to(torch.bfloat16)
    mask = bench.make_mask(B, T, 256, keep, 1).cuda()
    nrm = torch.nn.functional.normalize
    tg = [nrm(torch.randn(6, B, n, 3200, device="cuda", generator=g), dim=-1).to(torch.bfloat16),
          nrm(torch.randn(B, 768, device="cuda", generator=g), dim=-1).to(torch.bfloat16),
          nrm(torch.randn(4, B, n - 1, 1408, device="cuda", generator=g), dim=-1).to(torch.bfloat16)]

    def step():
        opt.zero_grad(set_to_none=True)
        out = model(video, mask)
        loss = sum((2 - 2 * (o * t).sum(-1)).mean() for o, t in zip(out, tg))
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 3.0)
        opt.step()
        return loss

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss = step()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    mem = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"reference-{'flash (FA2 ' + __import__('flash_attn').__version__ + ')' if flash else 'naive'}: B={B} "
          f"{ms:.1f} ms/step -> {B / ms * 1e3:.1f} clips/s (loss {float(loss):.4f}, peak mem {mem:.1f} GiB)", flush=True)
    del model, opt
    torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()


print(f"# reference GPU comparators on {torch.cuda.get_device_name()} (cfg-2: InternVideo2-1B, 8f 224^2, n={n}, bf16, fwd+bwd+clip+fused AdamW, eager)")
for flash in (False, True):
    for B in sorted({a.batch, 32}):
        try:
            run(flash, B)
        except Exception as e:  # noqa: BLE001
            print(f"reference-{'flash' if flash else 'naive'}: B={B} failed: {type(e).__name__}: {str(e)[:200]}", flush=True)
            torch.cuda.empty_cache()
