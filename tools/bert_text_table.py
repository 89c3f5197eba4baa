"""The stage-2 BERT-large text encoder on the H100, in one call that also prints the card name and power limit:
  1. the key-length attention forward (ivb_attn_fwd_keylen) against ivb_attn_fwd at n = 40 (1024 captions, BERT-large's
     16 heads of 64; one key tile, nothing to skip) and at n = 417 (32 clips, 16 heads of 64; key lengths drawn
     uniformly from [1, n], so about half the key tiles are skipped), ms per call;
  2. the text encoder forward (bert_modules.BertModel, mode="text": the 19 text layers of BERT-large) at 1024 captions
     x 40 tokens with lengths drawn from [5, 40], no-grad, ms per call;
  3. where the staged reference is present (oracle/_ref/, which the build fills through oracle/bert_text.stage), the
     reference xbert.BertModel on the same GPU in bf16 with the same weights and captions, alternated with 2.

Every arm is timed in three windows, alternating with the arm it is compared with; the table shows the fastest and
slowest of the three.

    python tools/bert_text_table.py [--iters 10]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from fp8_table import card, timed  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402
from internvideo_b200.bert_modules import BERT_LARGE, BertModel  # noqa: E402

B_TEXT, L_TEXT = 1024, 40


def _span(ts):
    return f"{min(ts):.3f}-{max(ts):.3f}"


def attn_table(iters):
    print("\n1. key-length attention vs ivb_attn_fwd (ms per call: fastest-slowest of 3 alternated windows)")
    print(f"  {'n':>5s} {'d':>3s} {'H':>3s} {'B':>5s} {'mean kv_len':>11s}  {'attn_fwd':>11s} {'keylen':>11s}")
    for n, d, H, B in ((40, 64, 16, 1024), (417, 64, 16, 32)):
        g = torch.Generator(device="cuda").manual_seed(n)
        D = H * d
        qkv = torch.randn((B * n, 3 * D), device="cuda", generator=g).to(torch.bfloat16)
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        kv = torch.randint(1, n + 1, (B,), device="cuda", generator=g, dtype=torch.int32) if n > 64 else \
            torch.randint(5, n + 1, (B,), device="cuda", generator=g, dtype=torch.int32)
        out = torch.empty((B * n, D), device="cuda", dtype=torch.bfloat16)
        s = d ** -0.5
        calls = iters * (20 if n < 256 else 10)
        plain, keylen = [], []
        for _ in range(3):
            plain.append(timed(lambda: ll.attn_fwd(q, k, v, B, n, H, d, s, out=out, want_lse=False), calls))
            keylen.append(timed(lambda: ll.attn_fwd(q, k, v, B, n, H, d, s, out=out, want_lse=False, kv_len=kv),
                                calls))
        print(f"  {n:5d} {d:3d} {H:3d} {B:5d} {kv.float().mean().item():11.1f}  {_span(plain):>11s} "
              f"{_span(keylen):>11s}")


def _captions():
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1000, BERT_LARGE["vocab_size"], (B_TEXT, L_TEXT), generator=g)
    lengths = torch.randint(5, L_TEXT + 1, (B_TEXT,), generator=g)
    mask = (torch.arange(L_TEXT)[None, :] < lengths[:, None]).long()
    ids[:, 0] = 101
    ids[torch.arange(B_TEXT), lengths - 1] = 102
    return (ids * mask).cuda(), mask.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs the H100"
    print("card:", card())
    attn_table(a.iters)
    ids, mask = _captions()
    torch.manual_seed(0)
    with torch.device("cuda"):
        port = BertModel(BERT_LARGE)
    port = port.bfloat16().eval().requires_grad_(False)
    run_port = lambda: port(ids, attention_mask=mask, mode="text")  # noqa: E731
    from oracle import bert_text
    if not bert_text.available():
        with torch.no_grad():
            print(f"\n2. ivb200 BertModel text mode, {B_TEXT} x {L_TEXT} (ms): {timed(run_port, a.iters):.3f}")
        print("\n3. reference BertModel: not staged, not measured")
        return
    with torch.device("cuda"):
        ref = bert_text.build_reference(BERT_LARGE)
    ref.load_state_dict(port.state_dict())
    ref = ref.bfloat16().eval().requires_grad_(False)
    run_ref = lambda: ref(ids, attention_mask=mask, return_dict=True, mode="text")  # noqa: E731
    ours, theirs = [], []
    with torch.no_grad():
        for _ in range(3):
            ours.append(timed(run_port, a.iters))
            theirs.append(timed(run_ref, a.iters))
        got = run_port().last_hidden_state[:, 0].float()
        want = run_ref().last_hidden_state[:, 0].float()
    rel = float((got - want).norm() / want.norm())
    print(f"\n2. ivb200 BertModel text mode (19 layers), {B_TEXT} captions x {L_TEXT} tokens, bf16 (ms): {_span(ours)}")
    print(f"3. reference xbert.BertModel, bf16, same GPU (ms): {_span(theirs)}   (ratio "
          f"{min(ours) / max(theirs):.2f}-{max(ours) / min(theirs):.2f}; pooled rows differ by {rel:.2e} relative)")


if __name__ == "__main__":
    main()
