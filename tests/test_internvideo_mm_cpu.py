"""InternVideo-MM (internvideo_b200.internvideo_mm) without a GPU: state_dict keys, order and shapes against the live
reference at the B/16 and L/14 sizes, the init draws, build_model's inferred configuration and load_model's key
surgery, the fp32 restatement against the fixture, and the refusals."""
import contextlib
from unittest import mock

import pytest
import torch

from internvideo_b200 import _lib
from internvideo_b200 import internvideo_mm as mm
from oracle import internvideo_mm as om

needs_ref = pytest.mark.skipif(not om.available(), reason="needs the reference (or its staged copy)")
_linspace = torch.linspace


@contextlib.contextmanager
def meta_device():
    """Builds modules without memory: on the meta device, with torch.linspace (the DropPath rates, read with .item())
    still on the CPU."""
    with torch.device("meta"), mock.patch("torch.linspace", lambda *a, **k: _linspace(*a, **{**k, "device": "cpu"})):
        yield


def _config(width):
    """VideoIntern's arguments as build_model passes them for a vision width (model.py:292-325), with the CLIP text
    tower of that size."""
    b16 = width == 768
    return dict(embed_dim=512 if b16 else 768, vision_width=width, context_length=77, vocab_size=49408,
                transformer_width=512 if b16 else 768, transformer_heads=8 if b16 else 12, transformer_layers=12,
                n_layers=4, n_dim=width, n_head=12 if b16 else 16, t_size=8,
                backbone="vit_only_global_b16" if b16 else "vit_only_global_l14",
                return_list=[8, 9, 10, 11] if b16 else [20, 21, 22, 23])


def _shapes(m):
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


@needs_ref
@pytest.mark.parametrize("width", [768, 1024], ids=["b16", "l14"])
def test_state_dict_matches_reference(width):
    ref_mod, _ = om.import_mm()
    with meta_device():
        ref = ref_mod.VideoIntern(**_config(width))
        port = mm.VideoIntern(**_config(width))
    assert _shapes(port) == _shapes(ref)


@pytest.fixture
def narrow():
    om.register_narrow(mm.BACKBONES, mm.VisionTransformer)
    yield
    mm.BACKBONES.pop(om.NARROW, None)


@needs_ref
def test_init_draws_match_reference(narrow):
    ref_mod, _ = om.import_mm()
    torch.manual_seed(0)
    ref = ref_mod.VideoIntern(**om.MODEL).state_dict()
    torch.manual_seed(0)
    port = mm.VideoIntern(**om.MODEL).state_dict()
    assert list(port) == list(ref)
    for k in ref:
        assert torch.equal(port[k], ref[k]), k


@needs_ref
@pytest.mark.parametrize("width", [768, 1024], ids=["b16", "l14"])
def test_build_model_infers_reference_config(width):
    ref_mod, _ = om.import_mm()
    cfg = _config(width)
    with meta_device():
        sd = ref_mod.VideoIntern(**cfg).state_dict()
        port = mm.build_model(sd)
    assert _shapes(port) == [(k, tuple(v.shape)) for k, v in sd.items()]
    assert not port.training
    assert port.embed_dim == cfg["embed_dim"] and port.context_length == 77
    assert port.visual.transformer.T == 8 and port.visual.transformer.return_list == cfg["return_list"]
    assert port.visual.transformer.dec[0].attn.num_heads == cfg["n_head"]
    assert port.transformer.resblocks[0].attn.num_heads == cfg["transformer_heads"]


@needs_ref
def test_load_model_strips_the_clip_prefix():
    ref_mod, _ = om.import_mm()
    with meta_device():
        sd = ref_mod.VideoIntern(**_config(768)).state_dict()
    ckpt = {"state_dict": {**{"clip." + k: v for k, v in sd.items()}, "other.head.weight": torch.zeros(2)}}
    with mock.patch.object(torch, "load", lambda *a, **k: ckpt), meta_device():
        port = mm.load_model("checkpoint.ckpt")
    assert _shapes(port) == [(k, tuple(v.shape)) for k, v in sd.items()]
    bad = {"state_dict": {"clip." + k: v for k, v in sd.items() if k != "visual.transformer.balance"}}
    with mock.patch.object(torch, "load", lambda *a, **k: bad), meta_device(), pytest.raises(RuntimeError,
                                                                                            match="balance"):
        mm.load_model("checkpoint.ckpt")


def test_build_model_refuses_other_widths():
    sd = {"text_projection": torch.zeros(128, 64), "positional_embedding": torch.zeros(16, 128),
          "token_embedding.weight": torch.zeros(512, 128), "ln_final.weight": torch.zeros(128),
          "visual_proj": torch.zeros(128, 64)}
    with pytest.raises(NotImplementedError, match="vision width 128"):
        mm.build_model(sd)


def test_restatement_matches_fixture():
    sd, z = om.load()
    out = om.restate(sd)
    video, image = om.stored_inputs(z)
    assert torch.equal(video, om.inputs()[0]) and torch.equal(image, om.inputs()[1])
    assert torch.equal(torch.from_numpy(z["ids"]), om.caption_ids())
    for k, v in out.items():
        torch.testing.assert_close(v, torch.from_numpy(z[k]), atol=2e-5, rtol=0, msg=k)


def test_refusals(narrow):
    torch.manual_seed(0)
    m = mm.VideoIntern(**om.MODEL)
    video = torch.zeros(1, 3, om.T, 56, 56)
    with pytest.raises(_lib.IvbError, match="forward only"):
        m.train().encode_video(video)
    with pytest.raises(_lib.IvbError, match="forward only"):
        m.encode_text(torch.zeros(1, 16, dtype=torch.long))
    m.eval()
    with pytest.raises(_lib.IvbError, match="must not require a gradient"):
        m.encode_video(video.requires_grad_(True))
    with pytest.raises(_lib.IvbError, match="the video has 3 frames, the model t_size 4"):
        m.encode_video(torch.zeros(1, 3, 3, 56, 56))
    with pytest.raises(NotImplementedError, match="attn_mask"):
        mm.Extractor(128, 2, attn_mask=torch.zeros(4, 4))
    with pytest.raises(NotImplementedError, match="backbone 'vit_2plus1d_dw_bias_b16'"):
        mm.VideoIntern(**{**om.MODEL, "backbone": "vit_2plus1d_dw_bias_b16"})
    with pytest.raises(ValueError, match="pretrained must be a local checkpoint path"):
        mm.vit_only_global_b16(pretrained=True)
