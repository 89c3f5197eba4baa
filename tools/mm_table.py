"""InternVideo-MM-L/14 on the H100, in one call that also prints the card name and power limit:
  1. encode_video of 32 clips x 8 frames at 224^2 and encode_text of 256 captions of 77 tokens, ms per call over CUDA
     events, the library's VideoIntern against the staged unmodified reference modules (oracle/_ref/, filled by
     oracle/internvideo_mm.stage at build time) under bf16 autocast on the same card, no gradients, the two arms
     alternated in windows;
  2. ivb_dpe_ln_fwd alone at the L/14 extractor tap of that batch (fp32 stream, 32 x 8 x 257 rows of 1024) against the
     reference's torch ops for the same result (grouped Conv3d on the permuted patch tokens, cat with the cls rows,
     LayerNorm) in fp32, ms per call and GB/s of the bytes each row must move (one fp32 read, one bf16 write).

    python tools/mm_table.py [--batch 32] [--text-batch 256] [--iters 5] [--rounds 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from fp8_table import card, timed  # noqa: E402
from internvideo_b200 import internvideo_mm as mm  # noqa: E402
from internvideo_b200 import lowlevel as ll  # noqa: E402

bf = torch.bfloat16
T, RES, CTX, VOCAB = 8, 224, 77, 49408
L14 = dict(embed_dim=768, vision_width=1024, context_length=CTX, vocab_size=VOCAB, transformer_width=768,
           transformer_heads=12, transformer_layers=12, n_layers=4, n_dim=1024, n_head=16, t_size=T,
           backbone="vit_only_global_l14", return_list=[20, 21, 22, 23])


def _inputs(B, Bt):
    g = torch.Generator(device="cuda").manual_seed(0)
    video = torch.randn(B, 3, T, RES, RES, device="cuda", generator=g).to(bf)
    ids = torch.randint(1, VOCAB - 1, (Bt, CTX), device="cuda", generator=g)
    ids[:, -1] = VOCAB - 1                                # the EOT, the largest id
    return video, ids


def _arms(B, Bt):
    """{name: (encode_video, encode_text)} of the library and, when staged, the reference."""
    video, ids = _inputs(B, Bt)
    torch.manual_seed(0)
    ours = mm.VideoIntern(**L14).bfloat16().cuda().eval()
    arms = {"ivb200": (lambda: ours.encode_video(video), lambda: ours.encode_text(ids))}
    from oracle import internvideo_mm as om
    if om.available():
        ref_mod, _ = om.import_mm()
        torch.manual_seed(0)
        ref = ref_mod.VideoIntern(**L14).cuda().eval()
        vf = video.float()

        def rv():
            with torch.no_grad(), torch.autocast("cuda", dtype=bf):
                return ref.encode_video(vf)

        def rt():
            with torch.no_grad(), torch.autocast("cuda", dtype=bf):
                return ref.encode_text(ids)
        arms["reference (bf16)"] = (rv, rt)
    return arms


def encode_table(B, Bt, iters, rounds):
    print(f"\n1. InternVideo-MM-L/14 encode_video ({B} clips x {T} frames at {RES}^2) and encode_text ({Bt} x {CTX} "
          f"tokens), no gradients (ms per call; {rounds} alternated windows of {iters} calls)")
    arms = _arms(B, Bt)
    res = {(k, w): [] for k in arms for w in ("video", "text")}
    for _ in range(rounds):
        for k, (fv, ft) in arms.items():
            res[k, "video"].append(timed(fv, iters))
            res[k, "text"].append(timed(ft, iters))
    for w in ("video", "text"):
        for k in arms:
            v = res[k, w]
            print(f"  encode_{w:5s} {k:18s} min {min(v):8.2f}  max {max(v):8.2f}   ({', '.join(f'{x:.2f}' for x in v)})")
        if len(arms) > 1:
            print(f"  encode_{w:5s} ivb200 / reference (best windows): "
                  f"{min(res['ivb200', w]) / min(res['reference (bf16)', w]):.3f}")
    if len(arms) == 1:
        print("  reference not staged (oracle/_ref/): its arm is not measured")


def kernel_table(B, iters, rounds):
    Hg, C = RES // 14, 1024
    L = 1 + Hg * Hg
    M = B * T * L
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(M, C, device="cuda", generator=g)
    w = (0.2 * torch.randn(C, 1, 3, 3, 3, device="cuda", generator=g)).to(bf)
    b, lb = ((0.05 * torch.randn(C, device="cuda", generator=g)).to(bf) for _ in range(2))
    lw = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).to(bf)
    wf, bfl, lwf, lbf = (t.float() for t in (w, b, lw, lb))
    out = torch.empty(M, C, device="cuda", dtype=bf)

    def ours():
        ll._dpe_ln_fwd(x, w, b, lw, lb, 1e-5, B, T, Hg, Hg, out=out)

    def torch_ops():     # clip_vit_only_global.py:221-230 and ln_3, on the [(n t l), C] rows
        v = x.view(B, T, L, C)
        p = v[:, :, 1:].permute(0, 3, 1, 2).reshape(B, C, T, Hg, Hg)
        conv = F.conv3d(p, wf, bfl, padding=1, groups=C).reshape(B, C, T, L - 1).permute(0, 2, 3, 1)
        y = torch.cat([v[:, :, :1], v[:, :, 1:] + conv], 2)
        return F.layer_norm(y, (C,), lwf, lbf, 1e-5)

    res = {"ivb_dpe_ln_fwd": [], "torch Conv3d + cat + LayerNorm (fp32)": []}
    for _ in range(rounds):
        res["ivb_dpe_ln_fwd"].append(timed(ours, iters * 10))
        res["torch Conv3d + cat + LayerNorm (fp32)"].append(timed(torch_ops, iters * 10))
    nbytes = M * C * (4 + 2)
    print(f"\n2. The L/14 extractor tap: {B} x {T} x {L} rows of {C} (fp32 in, {M * C * 4 / 1e6:.0f} MB; bf16 out, "
          f"{M * C * 2 / 1e6:.0f} MB), ms per call, min-max of {rounds} alternated windows of {iters * 10}; GB/s of "
          "those bytes at the best window")
    for k, v in res.items():
        print(f"  {k:40s} {min(v):.4f}-{max(v):.4f} ms   {nbytes / min(v) / 1e6:7.0f} GB/s")
    ref = torch_ops()
    print(f"  max |ivb - torch| {float((out.float() - ref.reshape(M, C)).abs().max()):.3e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--text-batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/mm_table.py measures on the GPU"
    print(f"GPU: {card()} (name, power limit, max SM clock)")
    kernel_table(a.batch, a.iters, a.rounds)
    encode_table(a.batch, a.text_batch, a.iters, a.rounds)


if __name__ == "__main__":
    main()
