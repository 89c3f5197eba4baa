"""The MobileCLIP-B text tower of the video-text recipe (cfg-3) on the H100, in one call that also prints the card name
and power limit:
  1. causal against non-causal attention (ivb_attn_fwd_causal / ivb_attn_fwd and the two backward passes), at the text
     tower's n = 77 (128 captions, 8 heads of 64) and at n = 1025 (16 clips, 16 heads of 64), ms per call;
  2. the text tower forward at the cfg-3 per-GPU batch (128 captions x 77 tokens), no-grad and differentiated (forward
     + backward), ms per call;
  3. where the staged reference is present (oracle/_ref/, which the build fills through oracle/text_tower.stage), the
     reference TextTransformer on the same GPU in bf16, same batch, same two measurements.

    python tools/text_tower_table.py [--iters 20]
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
from internvideo_b200.text_modules import MOBILECLIP_B, MOBILECLIP_B_PROJECTION_DIM, TextTransformer  # noqa: E402

B_TEXT = 128


def attn_table(iters):
    """Each arm is timed three times, alternating, over enough calls for a window of tens of ms at n = 77 (one call
    takes tens of microseconds there); the table shows the fastest and slowest of the three."""
    print("\n1. attention, causal vs non-causal (ms per call: fastest-slowest of 3 alternated windows)")
    print(f"  {'n':>5s} {'d':>3s} {'H':>3s} {'B':>4s}  {'fwd':>11s} {'fwd causal':>11s}  {'bwd':>11s} "
          f"{'bwd causal':>11s}")
    for n, d, H, B in ((77, 64, 8, 128), (1025, 64, 16, 16)):
        g = torch.Generator(device="cuda").manual_seed(n)
        D = H * d
        qkv = torch.randn((B * n, 3 * D), device="cuda", generator=g).to(torch.bfloat16)
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        dout = torch.randn((B * n, D), device="cuda", generator=g).to(torch.bfloat16)
        dq = torch.empty((B * n, 3 * D), device="cuda", dtype=torch.bfloat16)
        s = d ** -0.5
        calls = iters * (50 if n < 256 else 5)
        res = {(c, p): [] for c in (False, True) for p in ("fwd", "bwd")}
        for _ in range(3):
            for causal in (False, True):
                out, lse = ll.attn_fwd(q, k, v, B, n, H, d, s, causal=causal)
                res[causal, "fwd"].append(timed(lambda: ll.attn_fwd(q, k, v, B, n, H, d, s, out=out, causal=causal),
                                                calls))
                res[causal, "bwd"].append(timed(lambda: ll.attn_bwd(q, k, v, out, dout, lse, B, n, H, d, s, dq[:, :D],
                                                                    dq[:, D:2 * D], dq[:, 2 * D:], causal=causal),
                                                calls))
        cell = lambda c, p: f"{min(res[c, p]):.3f}-{max(res[c, p]):.3f}"  # noqa: E731
        print(f"  {n:5d} {d:3d} {H:3d} {B:4d}  {cell(False, 'fwd'):>11s} {cell(True, 'fwd'):>11s}  "
              f"{cell(False, 'bwd'):>11s} {cell(True, 'bwd'):>11s}")


def _ids():
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1, 49406, (B_TEXT, 77), generator=g)
    for b in range(B_TEXT):
        e = 5 + b % 60
        ids[b, 0], ids[b, e], ids[b, e + 1:] = 49406, 49407, 0
    return ids.cuda()


def tower_times(tower, ids, iters):
    with torch.no_grad():
        t_fwd = timed(lambda: tower(ids), iters)

    def step():
        tower.zero_grad(set_to_none=True)
        tower(ids).float().sum().backward()
    return t_fwd, timed(step, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs the H100"
    print("card:", card())
    attn_table(a.iters)
    ids = _ids()
    torch.manual_seed(0)
    tower = TextTransformer(MOBILECLIP_B, MOBILECLIP_B_PROJECTION_DIM)
    with torch.no_grad():
        tower.projection_layer.normal_(0, 512 ** -0.5)
    tower = tower.bfloat16().cuda()
    print(f"\n2. ivb200 text tower, {B_TEXT} captions x 77 tokens (ms): forward %.3f, forward + backward %.3f"
          % tower_times(tower, ids, a.iters))
    from oracle import text_tower
    if not text_tower.available():
        print("\n3. reference text tower: not staged, not measured")
        return
    ref = text_tower.reference().TextTransformer(
        # nn.LayerNorm in place of LayerNormFP32, which would pass fp32 rows to bf16 weights
        dict(MOBILECLIP_B, norm_layer="layer_norm"), MOBILECLIP_B_PROJECTION_DIM)
    ref.load_state_dict(tower.state_dict())
    ref = ref.bfloat16().cuda()
    with torch.no_grad():
        rel = float((ref(ids).float() - tower(ids).float()).norm() / ref(ids).float().norm())
    print(f"\n3. reference TextTransformer, bf16, same GPU (ms): forward %.3f, forward + backward %.3f"
          % tower_times(ref, ids, a.iters) + f"   (pooled outputs differ by {rel:.2e} relative)")


if __name__ == "__main__":
    main()
