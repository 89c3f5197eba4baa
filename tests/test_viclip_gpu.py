"""ViCLIP on the H100 (gpu) against tests/golden/viclip.npz, the unmodified reference's fp32 outputs and gradients:
  - the masked vision embedding (p = 0.5, the reference's draw under its torch seed), the text embedding, the VTC loss
    with a duplicated idx, return_embed of both towers, an image (T = 1) and an injected DropPath draw, each within
    2e-2 relative (Frobenius) of the reference, the loss within 1e-2, and every parameter gradient but the temperature's
    within 3e-2 of the reference's on the elements the fixture stores (oracle/viclip.sample: all of a small tensor,
    1024 of a large one; bf16 parameters and activations against fp32).  The temperature's gradient is a sum whose
    terms cancel to about 1/50 of their magnitudes, so bf16 rounding of the embeddings moves it by several percent of
    itself; its error is held to 2^-7 of the sum of its terms' magnitudes (oracle/viclip.temp_grad_scale), below the
    gradient's own magnitude;
  - the masked tokens in the reference's order: return_embed under the mask against the CPU restatement fed the
    reference's kept positions;
  - checkpointed blocks give the plain blocks' outputs and gradients bit for bit;
  - FP8: the frozen text tower under set_fp8_inference within OUT_BOUND of its bf16 output, and the vision tower trained
    under set_fp8(scaling="token") within OUT_BOUND (output) and GRAD_BOUND (gradients) of bf16, the bounds
    tests/test_fp8_layernorm_gpu.py holds the other LayerNorm towers to.
"""
import json
from pathlib import Path

import pytest
import torch

from internvideo_b200 import modules as M
from internvideo_b200 import viclip
from internvideo_b200.contrastive import VTC_VTM_Loss
from oracle import viclip as ov

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden" / "viclip.npz"
bf = torch.bfloat16
U_E4M3 = 2.0 ** -4
OUT_BOUND = 2 * U_E4M3        # FP8 output against bf16 (tests/test_fp8_layernorm_gpu.py)
GRAD_BOUND = 4 * U_E4M3       # per-token FP8 training gradients against bf16 (same file)


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm())


def _towers():
    sd, z = ov.load(GOLD)
    vis, txt = viclip.VisionTransformer(**ov.VISION), viclip.CLIP_TEXT(**ov.TEXT)
    vis.load_state_dict({k[15:]: v for k, v in sd.items() if k.startswith("vision_encoder.")}, strict=True)
    txt.load_state_dict({k[13:]: v for k, v in sd.items() if k.startswith("text_encoder.")}, strict=True)
    temp = torch.nn.Parameter(sd["temp"].clone().cuda())
    return vis.bfloat16().cuda().train(), txt.bfloat16().cuda().train(), temp, sd, z


def _inputs(z):
    cfg = json.loads(bytes(z["cfg"]).decode())
    video, image = (t.cuda().to(bf) for t in ov.inputs())
    return cfg, video, image, ov.caption_ids().cuda(), ov.drop_path_factors(ov.N_TOKENS)


def _forward(vis, txt, temp, z):
    cfg, video, image, ids, f = _inputs(z)
    torch.manual_seed(cfg["mask_seed"])
    masked = vis(video, masking_prob=cfg["mask_p"])
    text = txt(ids)
    loss = VTC_VTM_Loss(False).vtc_loss(masked, text, torch.tensor(cfg["idx"], device="cuda"), temp, all_gather=True)
    out = {"vision_masked": masked, "text": text, "loss_vtc": loss, "embed": vis(video, return_embed=True),
           "image": vis(image), "droppath": vis(video, drop_path_factors=f), "text_all": txt(ids, return_embed=True)[0]}
    total = out["loss_vtc"]
    for k, freq in (("embed", 0.37), ("image", 0.53), ("droppath", 0.71), ("text_all", 0.29)):
        total = total + (out[k].float() * ov.weights(out[k].shape, freq).cuda()).sum()
    return out, total


def _params(vis, txt, temp):
    return [("vision_encoder." + k, p) for k, p in vis.named_parameters()] + \
           [("text_encoder." + k, p) for k, p in txt.named_parameters()] + [("temp", temp)]


def test_viclip_against_reference(cuda_lib):
    vis, txt, temp, _, z = _towers()
    out, total = _forward(vis, txt, temp, z)
    total.backward()
    torch.cuda.synchronize()
    for k, key in (("vision_masked", "vision_masked"), ("text", "text"), ("embed", "embed"), ("image", "image_out"),
                   ("droppath", "droppath"), ("text_all", "text_all")):
        r = _rel(out[k], torch.from_numpy(z[key]))
        assert r < 2e-2, (k, r)
    ref_loss = float(z["loss_vtc"])
    assert abs(float(out["loss_vtc"]) - ref_loss) < 1e-2 * abs(ref_loss)
    errs = {k: _rel(ov.sample(p.grad.cpu()), torch.from_numpy(z["g/" + k])) for k, p in _params(vis, txt, temp)
            if k != "temp"}
    bad = {k: r for k, r in errs.items() if not r < 3e-2}
    # the temperature's gradient (1 / temp) sum_ij dL/ds_ij s_ij cancels to ~1/50 of its terms' magnitudes (`scale`,
    # oracle/viclip.temp_grad_scale, from the reference's embeddings).  The loss computes the logits from bf16
    # normalised rows, so each logit carries a relative error of about 2^-8 and each term moves by about twice that:
    # the bound is 2^-7 of the scale, which on this fixture is 0.39 of the gradient, so its sign is held too
    ref_g = float(z["g/temp"][0])
    scale = ov.temp_grad_scale(torch.from_numpy(z["vision_masked"]), torch.from_numpy(z["text"]),
                               torch.tensor(ov.IDX), float(temp.detach()))
    assert abs(float(temp.grad) - ref_g) <= 2.0 ** -7 * scale < abs(ref_g), (float(temp.grad), ref_g, scale)
    assert not bad, f"gradients off by more than 3e-2 relative: {bad}; largest of all: {max(errs.values()):.3g}"


def test_masked_tokens_in_reference_order(cuda_lib):
    vis, _, _, sd, z = _towers()
    cfg, video, _, _, _ = _inputs(z)
    vs = {k[15:]: v for k, v in sd.items() if k.startswith("vision_encoder.")}
    with torch.no_grad():
        torch.manual_seed(cfg["mask_seed"])
        got = vis(video, masking_prob=cfg["mask_p"], return_embed=True)
        want = ov.restate_vision(vs, video.float().cpu(), torch.from_numpy(z["kept"]).long(), return_embed=True)
    assert got.shape == want.shape
    assert _rel(got, want) < 2e-2
    # every token where the reference puts it: each row is nearest to its own reference row
    d = torch.cdist(got.float().cpu().flatten(0, 1), want.flatten(0, 1))
    assert torch.equal(d.argmin(1), torch.arange(d.shape[0]))


def test_checkpointed_blocks_bit_identical(cuda_lib):
    grads = []
    for ckpt in (False, True):
        vis, txt, temp, _, z = _towers()
        for blk in list(vis.transformer.resblocks) + list(txt.transformer.resblocks):
            blk.checkpoint = ckpt
        out, total = _forward(vis, txt, temp, z)
        total.backward()
        grads.append(({k: v.detach().clone() for k, v in out.items()},
                      {k: p.grad.clone() for k, p in _params(vis, txt, temp)}))
    (o0, g0), (o1, g1) = grads
    for k in o0:
        assert torch.equal(o0[k], o1[k]), k
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_frozen_text_tower_fp8_inference(cuda_lib):
    _, txt, _, _, z = _towers()
    txt.requires_grad_(False)
    ids = ov.caption_ids().cuda()
    base = txt(ids)
    assert M.set_fp8_inference(txt) == ov.TEXT["transformer_layers"]
    fp8 = txt(ids)
    r = _rel(fp8, base)
    assert 0 < r <= OUT_BOUND, r
    assert M.set_fp8_inference(txt, False) == ov.TEXT["transformer_layers"]
    assert torch.equal(txt(ids), base)


def test_vision_tower_fp8_token_training(cuda_lib):
    results = []
    for fp8 in (False, True):
        vis, _, _, _, z = _towers()
        _, video, _, _, _ = _inputs(z)
        if fp8:
            assert M.set_fp8(vis, True, scaling="token") == ov.VISION["layers"]
        out = vis(video)
        (out.float() * ov.weights(out.shape, 0.41).cuda()).sum().backward()
        results.append((out.detach(), {k: p.grad.clone() for k, p in vis.named_parameters()}))
    (o0, g0), (o1, g1) = results
    assert 0 < _rel(o1, o0) <= OUT_BOUND
    for k in g0:
        r = _rel(g1[k], g0[k])
        assert r <= GRAD_BOUND, (k, r)
