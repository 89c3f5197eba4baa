"""InternVideo-Next's encoder on the host, without a GPU: the port's parameters against the unmodified reference module
(state_dict keys, order and shapes for both factories, init bytes under one seed), the CPU restatement
(oracle/internvideo_next.py) against tests/golden/internvideo_next.npz, and the model's refusals.  Tests that run the
reference skip where it is absent."""
from pathlib import Path

import pytest
import torch

from internvideo_b200 import _lib
from internvideo_b200 import internvideo_next as nx
from oracle import internvideo_next as on

GOLD = Path(__file__).resolve().parent / "golden" / "internvideo_next.npz"
needs_ref = pytest.mark.skipif(not on.available(), reason="needs the reference InternVideo-Next sources")


def _pair(seed, factory=None, **kw):
    torch.manual_seed(seed)
    ref = on.build(factory, **kw)
    torch.manual_seed(seed)
    port = getattr(nx, factory)(**on.NAIVE, **kw) if factory else nx.InternVideo2(**on.NAIVE, **kw)
    return ref, port


@needs_ref
@pytest.mark.parametrize("factory", ["internvideo_next_base_patch14_224", "internvideo_next_large_patch14_224"])
def test_factory_state_dict_matches_reference(factory):
    ref, port = _pair(0, factory)
    rs, ps = ref.state_dict(), port.state_dict()
    assert list(rs) == list(ps)
    for k in rs:
        assert rs[k].shape == ps[k].shape, k
    assert ps["cls_token"].shape == (1, 4, port.embed_dim)
    assert ps["pos_embed"].shape == (1, 4 + 16 * 256, port.embed_dim)
    assert ps["patch_embed.norm_before.weight"].shape == (588,)


@needs_ref
@pytest.mark.parametrize("kw", [dict(on.CFG), dict(on.CFG, tubelet_size=2, drop_path_rate=0.1, qkv_bias=True)],
                         ids=["fixture", "tubelet2"])
def test_init_bytes_match_reference(kw):
    ref, port = _pair(7, **kw)
    rs, ps = ref.state_dict(), port.state_dict()
    assert list(rs) == list(ps)
    for k in rs:
        assert torch.equal(rs[k], ps[k]), f"init bytes differ: {k}"
    port.load_state_dict(rs, strict=True)


def test_restatement_matches_fixture():
    sd, z = on.load(GOLD)
    x = on.video()
    for name, projected in (("tokens", False), ("pooled", True)):
        got = on.restate(sd, x, projected=projected)
        assert torch.allclose(got, torch.from_numpy(z[name]), rtol=0, atol=2e-5), name


def test_fixture_lists_the_port_parameters():
    """The fixture names the port's parameters, in its order and shapes, so draw_param fills the port exactly."""
    sd, _ = on.load(GOLD)
    port = nx.InternVideo2(**on.NAIVE, **on.CFG)
    assert [(k, tuple(v.shape)) for k, v in port.state_dict().items()] == [(k, tuple(v.shape)) for k, v in sd.items()]


def test_position_table_has_four_zero_cls_rows():
    port = nx.InternVideo2(**on.NAIVE, **on.CFG)
    pe = port.pos_embed.detach()
    assert pe.shape == (1, 4 + 4 * 16, 128)
    assert torch.count_nonzero(pe[0, :4]) == 0 and torch.count_nonzero(pe[0, 4]) > 0


def test_refusals():
    with pytest.raises(NotImplementedError, match="sep_pos_embed"):
        nx.InternVideo2(**on.NAIVE, **dict(on.CFG, sep_pos_embed=True))
    m = nx.InternVideo2(**on.NAIVE, **on.CFG)
    x = torch.zeros(1, 3, 4, 56, 56)
    with pytest.raises(_lib.IvbError, match="bfloat16"):       # fp32 parameters
        m(x)
    m = m.bfloat16()
    with pytest.raises(_lib.IvbError, match="CUDA"):           # CPU input
        m(x.bfloat16())
    for shape in ((1, 3, 8, 56, 56), (1, 3, 4, 112, 112)):      # frame count / resolution other than the table's
        with pytest.raises(_lib.IvbError, match="position table"):
            m(torch.zeros(shape, dtype=torch.bfloat16))


def test_head_drop_path_rate_accepted():
    """The reference constructs the projector's DropPath but never applies it; the port accepts the argument."""
    m = nx.InternVideo2(**on.NAIVE, **dict(on.CFG, head_drop_path_rate=0.1))
    assert sorted(m.state_dict()) == sorted(nx.InternVideo2(**on.NAIVE, **on.CFG).state_dict())
