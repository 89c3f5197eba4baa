"""FP8 for the LayerNorm towers on the H100, in one call that prints the card name and power limit first and last:
  1. the InternVideo1 VideoMAE pre-training step (videomae_v1.pretrain_mae_base_patch16_224 and
     pretrain_mae_large_patch16_224; B = 32 clips of 16 frames, mask ratio 0.9: 157 visible tokens per clip in the
     encoder, 1568 in the decoder; forward, backward and AdamW captured in one CUDA graph): bf16 against per-token FP8
     (modules.set_fp8(model, scaling="token"));
  2. the MobileCLIP-B text tower, forward + backward at the cfg-3 per-GPU batch (128 captions x 77 tokens): bf16
     against per-token FP8;
  3. the stage-2 BERT-large text encoder forward (its 19 text layers) at 1024 captions x 40 tokens: bf16 against FP8
     inference (modules.set_fp8_inference).
Each pair of modes is timed in three windows, alternating; the table shows every window and the fastest.

    python tools/ln_fp8_table.py [--steps 10] [--iters 20]
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import card, timed  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402
from internvideo_b200.modules import set_fp8, set_fp8_inference  # noqa: E402

REPS = 3


def _report(name, res, unit="ms"):
    for mode, ts in res.items():
        print(f"  {name} {mode:6s}: best {min(ts):8.3f} {unit}  (windows: {', '.join(f'{t:.3f}' for t in ts)})")
    (m0, t0), (m1, t1) = res.items()
    print(f"  {name}: {m1} / {m0} = {min(t1) / min(t0):.3f}")


def iv1_table(steps):
    from internvideo_b200 import videomae_v1 as v1
    from internvideo_b200.engine import GraphedStep, PretrainEngine
    B, T, N = 32, 16, 1568
    n_masked = int(0.9 * N)
    print(f"\n1. InternVideo1 VideoMAE step, B = {B} x {T} frames, {N - n_masked} visible of {N} tokens, one CUDA graph "
          "(ms/step)")
    g = torch.Generator().manual_seed(0)
    video = torch.randn(B, 3, T, 224, 224, generator=g).to(torch.bfloat16).cuda()
    mask = torch.zeros(B, N, dtype=torch.bool)
    for b in range(B):
        mask[b, torch.randperm(N, generator=g)[:n_masked]] = True
    mask = mask.cuda()
    for name in ("pretrain_mae_base_patch16_224", "pretrain_mae_large_patch16_224"):
        torch.manual_seed(0)
        model = getattr(v1, name)().bfloat16().cuda().train()
        eng = PretrainEngine(model, lr=1.5e-4, betas=(0.9, 0.95), weight_decay=0.05, clip_grad=0.0)

        def step(v):
            eng.zero_grad()
            loss = v1.pretrain_loss(model, v, mask, n_masked=n_masked)
            loss.backward()
            eng.step()
            return loss
        res = {"bf16": [], "fp8": []}
        for _ in range(REPS):
            for mode in res:
                set_fp8(model, mode == "fp8", scaling="token")
                gs = GraphedStep(step, [video], warmup=1)
                gs(video)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(steps):
                    loss = gs(video)
                torch.cuda.synchronize()
                res[mode].append((time.perf_counter() - t0) * 1e3 / steps)
                print(f"  {name} {mode}: {res[mode][-1]:.2f} ms/step, loss {float(loss):.4f}")
                del gs
                torch.cuda.empty_cache()
        _report(name, res)
        del model, eng
        torch.cuda.empty_cache()


def text_table(iters):
    from internvideo_b200.text_modules import MOBILECLIP_B, MOBILECLIP_B_PROJECTION_DIM, TextTransformer
    print("\n2. MobileCLIP-B text tower, 128 captions x 77 tokens, forward + backward (ms per call)")
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1, 49406, (128, 77), generator=g)
    for b in range(128):
        e = 5 + b % 60
        ids[b, 0], ids[b, e], ids[b, e + 1:] = 49406, 49407, 0
    ids = ids.cuda()
    torch.manual_seed(0)
    tower = TextTransformer(MOBILECLIP_B, MOBILECLIP_B_PROJECTION_DIM)
    with torch.no_grad():
        tower.projection_layer.normal_(0, 512 ** -0.5)
    tower = tower.bfloat16().cuda()

    def step():
        tower.zero_grad(set_to_none=True)
        tower(ids).float().sum().backward()
    res = {"bf16": [], "fp8": []}
    for _ in range(REPS):
        for mode in res:
            set_fp8(tower, mode == "fp8", scaling="token")
            res[mode].append(timed(step, iters))
    _report("text tower", res)


def bert_table(iters):
    from internvideo_b200.bert_modules import BERT_LARGE, BertModel
    from bert_text_table import _captions
    print("\n3. BERT-large text encoder (19 layers), 1024 captions x 40 tokens, no-grad forward (ms per call)")
    ids, mask = _captions()
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = BertModel(BERT_LARGE)
    model = model.bfloat16().eval().requires_grad_(False)
    run = lambda: model(ids, attention_mask=mask, mode="text")  # noqa: E731
    base = run().last_hidden_state[:, 0].float()
    res = {"bf16": [], "fp8": []}
    for _ in range(REPS):
        for mode in res:
            set_fp8_inference(model, mode == "fp8")
            res[mode].append(timed(run, iters))
    set_fp8_inference(model)
    got = run().last_hidden_state[:, 0].float()
    print(f"  pooled rows, FP8 against bf16: {float((got - base).norm() / base.norm()):.2e} relative")
    _report("BERT text", res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    ll.device_check()
    print("card:", card())
    iv1_table(a.steps)
    text_table(a.iters)
    bert_table(a.iters)
    print("card:", card())


if __name__ == "__main__":
    main()
