"""ViCLIP's host side without a GPU: the port's parameters against the reference modules (state_dict keys, order and
shapes, init bytes under one seed), the masking draw bit for bit against the reference's mask_tokens and its mapping
to the library's token index, the CPU restatement (oracle/viclip.py) against tests/golden/viclip.npz, the refusals,
the InternVideo1 contrastive loss being InternVideo2's statement for statement, and the GEMM kernels' SASS (no local
memory with the QuickGELU epilogue added).  Tests that run the reference skip where it is absent."""
import ast
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import sass
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import ops, viclip
from oracle import viclip as ov

GOLD = Path(__file__).resolve().parent / "golden" / "viclip.npz"
needs_ref = pytest.mark.skipif(not ov.available(), reason="needs the reference ViCLIP sources")
# parameters the reference allocates with torch.empty (they come from a checkpoint): no init bytes to compare
UNINITIALISED = {"proj", "positional_embedding", "text_projection"}


def _towers(seed, vision_cfg, text_cfg):
    rv, rt = ov.import_viclip()
    torch.manual_seed(seed)
    ref_v = rv.VisionTransformer(**vision_cfg)
    torch.manual_seed(seed)
    port_v = viclip.VisionTransformer(**vision_cfg)
    torch.manual_seed(seed)
    ref_t = rt.CLIP_TEXT(**text_cfg)
    torch.manual_seed(seed)
    port_t = viclip.CLIP_TEXT(**text_cfg)
    return (ref_v, port_v), (ref_t, port_t)


B16_VISION = dict(input_resolution=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512, num_frames=8)
B16_TEXT = dict(embed_dim=512, context_length=32, vocab_size=49408, transformer_width=512, transformer_heads=8,
                transformer_layers=12, checkpoint_num=0)


@needs_ref
@pytest.mark.parametrize("cfg", ["fixture", "b16"])
def test_state_dict_and_init_match_reference(cfg):
    vcfg, tcfg = (ov.VISION, ov.TEXT) if cfg == "fixture" else (B16_VISION, B16_TEXT)
    for ref, port in _towers(11, vcfg, tcfg):
        rs, ps = ref.state_dict(), port.state_dict()
        assert list(rs) == list(ps)
        for k in rs:
            assert rs[k].shape == ps[k].shape, k
            if k not in UNINITIALISED:
                assert torch.equal(rs[k], ps[k]), f"init bytes differ: {k}"
        port.load_state_dict(rs, strict=True)


def test_factories_build_the_recipe_towers():
    v = viclip.clip_joint_b16(pretrained=False, num_frames=4)
    assert v.proj.shape == (768, 512) and len(v.transformer.resblocks) == 12 and not v.training
    t = viclip.clip_text_b16(pretrained=False, context_length=32)
    assert t.text_projection.shape == (512, 512) and t.positional_embedding.shape == (32, 512)


@needs_ref
@pytest.mark.parametrize("seed", [0, 5, 1234])
@pytest.mark.parametrize("B,L,p", [(4, 64, 0.5), (2, 2048, 0.9), (3, 17, 0.3)])
def test_mask_draw_bit_exact(seed, B, L, p):
    rv, _ = ov.import_viclip()
    ref = rv.VisionTransformer(**ov.VISION)
    pos = torch.arange(L, dtype=torch.float32)[None, :, None].expand(B, L, 1)
    torch.manual_seed(seed)
    want = ref.mask_tokens(pos, p)[..., 0].long()          # the kept positions, in the reference's order
    torch.manual_seed(seed)
    got = viclip.VisionTransformer.mask_tokens(B, L, p)
    assert torch.equal(got, want)


def test_mask_draw_matches_fixture_and_maps_to_the_library_order():
    z = np.load(GOLD)
    cfg = json.loads(bytes(z["cfg"]).decode())
    T, Lf = cfg["T"], (cfg["vision"]["input_resolution"] // cfg["vision"]["patch_size"]) ** 2
    torch.manual_seed(cfg["mask_seed"])
    kept = viclip.VisionTransformer.mask_tokens(cfg["B"], T * Lf, cfg["mask_p"])
    assert torch.equal(kept, torch.from_numpy(z["kept"]).long())
    torch.manual_seed(cfg["mask_seed"])
    idx = viclip.VisionTransformer.token_index(cfg["B"], T, Lf, cfg["mask_p"])
    assert idx.dtype == torch.int32 and (idx[:, 0] == 0).all()
    # reference position k = s T + t ((n t) order) -> library row 1 + t L + s ((t n) order), order kept
    s, t = kept // T, kept % T
    assert torch.equal(idx[:, 1:].long(), 1 + t * Lf + s)
    full = viclip.VisionTransformer.token_index(2, T, Lf)
    assert sorted(full[0, 1:].tolist()) == list(range(1, T * Lf + 1))


def test_restatement_against_fixture():
    sd, z = ov.load(GOLD)
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    out = ov.restate(params, z)
    for name, key in (("vision_masked", "vision_masked"), ("text", "text"), ("embed", "embed"), ("image", "image_out"),
                      ("droppath", "droppath"), ("text_all", "text_all"), ("loss_vtc", "loss_vtc")):
        torch.testing.assert_close(out[name].detach(), torch.from_numpy(z[key]), atol=2e-5, rtol=0, msg=name)
    ov.total_loss(out).backward()
    for k, p in params.items():
        g = torch.from_numpy(z["g/" + k])
        torch.testing.assert_close(ov.sample(p.grad), g, atol=2e-5 * max(1.0, float(g.abs().max())), rtol=0, msg=k)


@needs_ref
def test_iv1_contrastive_loss_is_iv2s():
    """ViCLIP's vtc_loss, get_sim and get_mask (criterions.py) are InternVideo2's statement for statement, so
    contrastive.VTC_VTM_Loss serves both."""
    def defs(src):
        return {n.name: ast.dump(n) for n in ast.walk(ast.parse(src))
                if isinstance(n, ast.FunctionDef) and n.name in ("vtc_loss", "get_sim", "get_mask")}
    iv1, iv2 = defs(ov.criterions_source("iv1")), defs(ov.criterions_source("iv2"))
    assert set(iv1) == {"vtc_loss", "get_sim", "get_mask"} and iv1 == iv2


# ---------------------------------------------------------------- refusals
def test_refusals():
    with pytest.raises(NotImplementedError, match="dropout"):
        viclip.VisionTransformer(**ov.VISION, dropout=0.1)
    with pytest.raises(NotImplementedError, match="kernel_size"):
        viclip.VisionTransformer(**dict(ov.VISION, kernel_size=2))
    with pytest.raises(ValueError, match="local checkpoint path"):
        viclip.clip_joint_b16(pretrained=True)
    with pytest.raises(ValueError, match="local checkpoint path"):
        viclip.clip_text_l14(pretrained="CLIP-ViT-L/14")
    cfg = _config()
    cfg["model"]["vision_encoder"]["name"] = "vit_h14"
    with pytest.raises(NotImplementedError, match="vit_h14"):
        viclip.ViCLIP(cfg)
    cfg = _config()
    cfg["model"]["text_encoder"]["name"] = "bert_base"
    with pytest.raises(NotImplementedError, match="bert_base"):
        viclip.ViCLIP(cfg)
    m = viclip.ViCLIP(_config())
    with pytest.raises(NotImplementedError, match="token ids"):
        m.encode_text(["a caption"])
    with pytest.raises(NotImplementedError, match="retrieval"):
        m(None, None, None, None, return_sims=True)
    spec = ops.BlockSpec(1, 1, 1, gelu_tanh=True, gelu_quick=True)
    with pytest.raises(ll._lib.IvbError, match="exclude each other"):
        spec.gelu_flags(False)
    assert ops.BlockSpec(1, 1, 1, gelu_quick=True).gelu_flags(True) == ll.FLAG_GELU_QUICK | ll.FLAG_GELU_SAVE_GRAD


def _config():
    v, t = ov.VISION, ov.TEXT
    return {"max_txt_l": t["context_length"],
            "inputs": {"image_res": v["input_resolution"], "video_input": {"num_frames": v["num_frames"]}},
            "model": {"vision_encoder": {"name": "vit_b16", "pretrained": False, "d_model": 768, "kernel_size": 1,
                                         "center": True, "drop_path_rate": 0.1, "masking_prob": 0.9,
                                         "checkpoint_num": 12},
                      "text_encoder": {"name": "vit_b16", "pretrained": "bert-base-uncased", "d_model": 512,
                                       "vocab_size": 49408},
                      "embed_dim": 512, "temp": 1 / 100.0, "temp_min": 1 / 100.0, "freeze_text": True}}


def test_viclip_recipe_wiring():
    """The recipe's settings reach the towers: freeze_text, checkpoint_num, the DropPath rates, the temperature."""
    m = viclip.ViCLIP(_config())
    assert not any(p.requires_grad for p in m.text_encoder.parameters())
    blocks = m.vision_encoder.transformer.resblocks
    assert [b.checkpoint for b in blocks] == [True] * 12
    rates = [b.drop_prob for b in blocks]
    assert rates[0] == 0.0 and abs(rates[-1] - 0.1) < 1e-7
    assert all(b.causal for b in m.text_encoder.transformer.resblocks) and not any(b.causal for b in blocks)
    assert float(m.temp) == pytest.approx(0.01) and "temp" in m.no_weight_decay()
    # the text tower's checkpoint_sequential(resblocks, segments) checkpoints every segment but the last
    t = viclip.CLIP_TEXT(64, 32, 512, 128, 2, 12, checkpoint_num=4)
    assert [b.checkpoint for b in t.transformer.resblocks] == [True] * 9 + [False] * 3


# ---------------------------------------------------------------- SASS
def test_gemm_kernels_use_no_local_memory_with_quickgelu():
    """Every GEMM kernel (bf16 and FP8) keeps its epilogue, QuickGELU included, in registers."""
    fns = {k: v for k, v in sass.functions("ivb_gemm.o").items() if "gemm" in k}
    assert fns
    for name, lines in fns.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, name
    for name, (_, stack, local) in sass.resources("ivb_gemm.o").items():
        if "gemm" in name:
            assert local == 0, name
