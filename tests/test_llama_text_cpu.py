"""InternVideo2-CLIP's LLaMA text tower without a GPU: the port's parameters against the reference LLaMA(use_lora=False)
(state_dict keys, order and shapes), the 7B shape built on the meta device, the fp32 restatement (oracle/llama_text.py)
against tests/golden/llama_text.npz, the wrapper's checkpoint key surgery against a restatement of
internvideo2_clip.py:194-254, every refusal, and the RoPE kernel's SASS (no local memory).  Tests that run the reference
skip where it is absent."""
from pathlib import Path

import pytest
import torch

import sass
from internvideo_b200 import lowlevel as ll
from internvideo_b200.clip_modules import InternVideo2_CLIP, remap_text_checkpoint
from internvideo_b200.llama_modules import LLAMA_7B, LLaMA
from oracle import llama_text as ol

GOLD = Path(__file__).resolve().parent / "golden" / "llama_text.npz"
needs_ref = pytest.mark.skipif(not ol.available(), reason="needs the reference internvideo2_clip_text.py")


def _tiny(**over):
    cfg = dict(ol.CFG, **over)
    return LLaMA(transformer_width=cfg["hidden_size"], use_lora=False, clip_embed_dim=ol.EMBED, config=cfg)


@needs_ref
def test_state_dict_matches_reference():
    ref = ol.build_reference()
    port = _tiny()
    assert [(k, tuple(v.shape)) for k, v in port.state_dict().items()] == \
           [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]


def test_llama_path_reads_config_json(tmp_path):
    import json
    (tmp_path / "config.json").write_text(json.dumps(ol.CFG))
    m = LLaMA(transformer_width=256, llama_path=str(tmp_path), clip_embed_dim=ol.EMBED)
    assert list(m.state_dict()) == list(_tiny().state_dict())


def test_7b_shapes_on_meta():
    with torch.device("meta"):
        m = LLaMA(config=LLAMA_7B)
    D, I, V, n = 4096, 11008, 49954, 32
    per_layer = 4 * D * D + 3 * D * I + 2 * D
    assert sum(p.numel() for p in m.parameters()) == V * D + n * per_layer + D + D * 768
    sd = m.state_dict()
    assert tuple(sd["transformer.layers.31.mlp.gate_proj.weight"].shape) == (I, D)
    assert tuple(sd["transformer.layers.31.mlp.down_proj.weight"].shape) == (D, I)
    assert tuple(sd["text_projection"].shape) == (D, 768)
    assert list(sd)[:2] == ["text_projection", "transformer.embed_tokens.weight"]
    assert list(sd)[-1] == "transformer.norm.weight"


def test_init_distributions():
    torch.manual_seed(0)
    m = _tiny(vocab_size=4096)
    e = m.transformer.embed_tokens.weight
    assert bool((e[0] == 0).all())
    assert abs(float(e[1:].std()) - 0.02) < 1e-3
    assert abs(float(m.transformer.layers[0].mlp.gate_proj.weight.std()) - 0.02) < 1e-3
    assert bool((m.transformer.norm.weight == 1).all())


def test_restatement_matches_fixture():
    cfg, sd, z = ol.load(GOLD)
    out = ol.restate(sd, torch.from_numpy(z["ids"]), cfg)
    torch.testing.assert_close(out, torch.from_numpy(z["out"]), atol=2e-5, rtol=0)


def _reference_surgery(test_ckpt):
    """internvideo2_clip.py:231-241, restated: unwrap 'module', keep transformer.* and text_projection under
    'text_encoder.'."""
    if "module" in test_ckpt.keys():
        test_ckpt = test_ckpt["module"]
    new_ckpt = {}
    for k, v in test_ckpt.items():
        if k.startswith("transformer.") or k == "text_projection":
            new_ckpt["text_encoder." + k] = v
    return new_ckpt


def _lora_checkpoint(model, lora_b=0.0):
    """model's weights as a use_lora=True checkpoint (peft's keys on q_proj and v_proj), with InternVL-C's extra keys.
    text_projection (torch.empty at construction) is drawn first."""
    torch.nn.init.normal_(model.text_projection)
    ck = {}
    for k, v in model.state_dict().items():
        if k.endswith(("self_attn.q_proj.weight", "self_attn.v_proj.weight")):
            base = k[:-len(".weight")]
            ck[base + ".base_layer.weight"] = v.clone()
            ck[base + ".lora_A.default.weight"] = torch.randn(16, v.shape[1])
            ck[base + ".lora_B.default.weight"] = torch.full((v.shape[0], 16), lora_b)
        else:
            ck[k] = v.clone()
    ck["transformer.layers.0.self_attn.rotary_emb.inv_freq"] = torch.ones(64)
    ck["logit_scale"] = torch.ones(())
    return {"module": ck}


def test_wrapper_text_key_surgery():
    torch.manual_seed(1)
    src = _tiny()
    ck = _lora_checkpoint(src)
    assert remap_text_checkpoint(ck) == _reference_surgery(ck)
    wrapper = torch.nn.Module()
    wrapper.text_encoder = _tiny()
    res = wrapper.load_state_dict(remap_text_checkpoint(ck), strict=False)
    assert not res.missing_keys and not res.unexpected_keys
    for k, v in src.state_dict().items():
        assert torch.equal(wrapper.text_encoder.state_dict()[k], v), k
    with pytest.raises(NotImplementedError, match="lora_B"):
        wrapper.load_state_dict(remap_text_checkpoint(_lora_checkpoint(src, lora_b=1e-3)), strict=False)


def test_wrapper_load_checkpoint(tmp_path):
    """InternVideo2_CLIP.load_checkpoint with a text checkpoint only: the text keys land, strict=False."""
    torch.manual_seed(2)
    src = _tiny()
    torch.save(_lora_checkpoint(src), tmp_path / "text.pth")
    te = dict(in_chans=3, patch_size=14, img_size=28, qkv_bias=False, drop_path_rate=0.0, embed_dim=64, num_heads=1,
              mlp_ratio=2, init_values=0.1, qk_normalization=True, depth=1, use_flash_attn=False,
              use_fused_rmsnorm=False, use_fused_mlp=False, attn_pool_num_heads=1, clip_embed_dim=ol.EMBED,
              num_frames=1)
    cfg = dict(model=dict(vision_encoder=te, temp=0.01, temp_min=0.01, freeze_vision=True,
                          open_vision_clip_projector=True, freeze_text=True, open_text_projection=False))
    model = InternVideo2_CLIP(cfg, text_encoder=_tiny())
    model.load_checkpoint(text_ckpt_path=str(tmp_path / "text.pth"))
    for k, v in src.state_dict().items():
        assert torch.equal(model.text_encoder.state_dict()[k], v), k
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    assert trainable == {"temp"} | {n for n in trainable if n.startswith("vision_encoder.clip_projector.")}


@pytest.mark.parametrize("over,match", [
    (dict(rope_scaling={"type": "linear", "factor": 2.0}), "rope_scaling"),
    (dict(num_key_value_heads=1), "grouped-query"),
    (dict(hidden_act="gelu"), "hidden_act"),
    (dict(attention_bias=True), "attention_bias"),
    (dict(mlp_bias=True), "mlp_bias"),
    (dict(hidden_size=288, num_attention_heads=2), "head_dim"),
    (dict(hidden_size=512, num_attention_heads=2), "head_dim"),
])
def test_config_refusals(over, match):
    with pytest.raises(NotImplementedError, match=match):
        _tiny(**over)


def test_call_refusals():
    m = _tiny().bfloat16()
    ids = torch.ones((2, 8), dtype=torch.int64)
    with pytest.raises(ll._lib.IvbError, match="CUDA tensor"):
        m.requires_grad_(False)(ids)
    m.transformer.norm.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="forward-only"):
        m(ids)
    m.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="max_position_embeddings"):
        m(torch.ones((2, ol.CFG["max_position_embeddings"] + 1), dtype=torch.int64))
    with pytest.raises(ll._lib.IvbError, match="bf16"):
        _tiny().requires_grad_(False)(ids)
    m.text_projection.requires_grad_(True)        # open_text_projection: still accepted (fails later: CPU ids)
    with pytest.raises(ll._lib.IvbError, match="CUDA tensor"):
        m(ids)


def test_rope_kernel_uses_no_local_memory():
    fns = sass.functions("ivb_rope.o")
    assert fns
    for name, lines in fns.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, name
