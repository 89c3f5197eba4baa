"""The MobileCLIP text tower without a GPU: the port's construction against the unmodified reference (state_dict keys,
shapes and init bytes under one seed), the CPU restatement against tests/golden/text_tower.npz (outputs of the
unmodified reference), the module's refusals, and the argument checks of the causal attention and token-embedding
entry points through the raw C ABI."""
from pathlib import Path

import numpy as np
import pytest
import torch

from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib, ops
from internvideo_b200.text_modules import MOBILECLIP_B, TextTransformer
from oracle import text_tower

GOLD = Path(__file__).parent / "golden" / "text_tower.npz"
NARROW = dict(text_tower.CFG)


@pytest.mark.skipif(not text_tower.available(), reason="needs the reference's mobileclip sources")
@pytest.mark.parametrize("cfg", [NARROW, MOBILECLIP_B], ids=["narrow", "mobileclip_b"])
def test_state_dict_and_init_match_reference(cfg):
    """Same keys in the same order, same shapes, and the same bytes from the same seed, so that a MobileCLIP checkpoint
    loads unchanged and a tower built from scratch starts where the reference's would.  projection_layer is
    torch.empty in both (it comes from the checkpoint), so only its shape is compared."""
    ref_mod = text_tower.reference()
    torch.manual_seed(11)
    ref = ref_mod.TextTransformer(cfg, 512).state_dict()
    torch.manual_seed(11)
    port = TextTransformer(cfg, 512).state_dict()
    assert list(port) == list(ref)
    for k in ref:
        assert port[k].shape == ref[k].shape, k
        if k != "projection_layer":
            assert torch.equal(port[k], ref[k]), k


def test_restatement_matches_golden():
    cfg, sd, z = text_tower.load(GOLD)
    ids = torch.from_numpy(z["ids"])
    L, H = cfg["n_transformer_layers"], cfg["n_heads_per_layer"]
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    pooled = text_tower.restate(params, ids, L, H)
    every = text_tower.restate(params, ids[:text_tower.ALL_TOKENS_ROWS], L, H, return_all_tokens=True)
    torch.testing.assert_close(pooled, torch.from_numpy(z["pooled"]), atol=2e-5, rtol=0)
    torch.testing.assert_close(every, torch.from_numpy(z["all_tokens"]), atol=2e-5, rtol=0)
    wp, wa = text_tower.loss_weights(pooled.shape, every.shape)
    ((pooled * wp).sum() + (every * wa).sum()).backward()
    for k, p in params.items():
        torch.testing.assert_close(p.grad, torch.from_numpy(z["g/" + k]), atol=2e-5, rtol=1e-4, msg=k)


def test_golden_ids_cover_the_cases():
    """EOT at a different position in every row (the last slot included), zero padding, repeated ids in a row."""
    ids = np.load(GOLD)["ids"]
    eot = ids.argmax(-1)
    assert len(set(eot.tolist())) == len(eot) and eot.max() == ids.shape[1] - 1
    assert (ids == 0).any()
    assert any(len(set(r[1:e].tolist())) < e - 1 for r, e in zip(ids, eot))


def test_port_loads_the_golden_state_dict():
    cfg, sd, _ = text_tower.load(GOLD)
    tower = TextTransformer(cfg, cfg["projection_dim"])
    tower.load_state_dict(sd, strict=True)


def test_refusals():
    with pytest.raises(NotImplementedError):
        TextTransformer(dict(NARROW, model_name="mct"), 32)
    with pytest.raises(ValueError):
        TextTransformer(dict(NARROW, model_name="other"), 32)
    with pytest.raises(NotImplementedError):
        TextTransformer(dict(NARROW, embed_dropout=0.1), 32)
    tower = TextTransformer(NARROW, 32)
    with pytest.raises(_lib.IvbError, match="context_length"):
        tower(torch.zeros(2, 76, dtype=torch.int64))
    with pytest.raises(_lib.IvbError, match="bf16"):
        tower(torch.zeros(2, 77, dtype=torch.int64))
    with pytest.raises(_lib.IvbError, match="CUDA"):
        tower.bfloat16()(torch.zeros(2, 77, dtype=torch.int64))
    open_tower = TextTransformer(dict(NARROW, causal_masking=False), 32)
    with pytest.raises(NotImplementedError, match="key_padding_mask"):
        open_tower(torch.zeros(2, 77, dtype=torch.int64), key_padding_mask=torch.zeros(2, 77, dtype=torch.bool))


@pytest.mark.parametrize("extra", [dict(attn_fp8=True), dict(head_axis=True)])
def test_causal_block_refuses_fp8_and_head_axis(extra):
    spec = ops.BlockSpec(2, 77, 2, layernorm=True, causal=True, **extra)
    with pytest.raises(_lib.IvbError, match="causal"):
        ops.block_forward(torch.zeros(154, 64), spec, None, save=False)


def test_causal_block_refuses_droppath_plans():
    spec = ops.BlockSpec(2, 77, 2, layernorm=True, causal=True)
    with pytest.raises(_lib.IvbError, match="causal"):
        ops.block_forward(torch.zeros(154, 64), spec, None, plan1=torch.zeros(8, dtype=torch.int32))


# ------------------------------------------------------------------------------------------- C ABI refusals
D8 = 8 * 64


def _fwd(lib, d=64, H=8, ld=(3 * D8, 3 * D8, 3 * D8, D8), B=2, n=77):
    return lib.ivb_attn_fwd_causal(None, ld[0], None, ld[1], None, ld[2], None, ld[3], None, B, n, H, d, 0.125, None)


def _bwd(lib, d=64, H=8, ld=(3 * D8,) * 3 + (D8,) * 2 + (3 * D8,) * 3, B=2, n=77, lse=1, ws=1024):
    return lib.ivb_attn_bwd_causal(None, ld[0], None, ld[1], None, ld[2], None, ld[3], None, ld[4], lse, ws,
                                   None, ld[5], None, ld[6], None, ld[7], B, n, H, d, 0.125, None)


@pytest.mark.parametrize("d", [8, 12, 136, 0])
def test_causal_attn_head_dim_refused(d):
    lib = _lib.load()
    expect_refusal(_fwd(lib, d=d), "ivb_attn_fwd_causal: head_dim must be a multiple of 8 in [16,128]")
    expect_refusal(_bwd(lib, d=d), "ivb_attn_bwd_causal: head_dim must be a multiple of 8 in [16,128]")


@pytest.mark.parametrize("slot", range(8))
def test_causal_attn_pitch_refused(slot):
    lib = _lib.load()
    ld = [3 * D8] * 3 + [D8] * 2 + [3 * D8] * 3
    ld[slot] += 4
    expect_refusal(_bwd(lib, ld=ld), "ivb_attn_bwd_causal: pitches must be multiples of 8")
    if slot < 4:
        expect_refusal(_fwd(lib, ld=ld[:4]), "ivb_attn_fwd_causal: pitches must be multiples of 8")


def test_causal_attn_workspace_refused_and_empty_noop():
    lib = _lib.load()
    expect_refusal(_bwd(lib, lse=None), "ivb_attn_bwd_causal: lse2 and the workspace are required")
    expect_refusal(_bwd(lib, ws=1032), "ivb_attn_bwd_causal: workspace must be 16-byte aligned")
    for B, n in ((0, 77), (2, 0)):
        assert _fwd(lib, B=B, n=n) == 0
        assert _bwd(lib, B=B, n=n) == 0


def _emb_fwd(lib, ids=BASE, table=BASE, pos=BASE, out=BASE, err=BASE, V=1000, D=64, ldo=64, B=2, L=77):
    return lib.ivb_token_embed_fwd(ids, B, L, table, V, pos, D, out, ldo, err, None)


def _emb_bwd(lib, ids=BASE, g=BASE, dt=BASE, dp=BASE, ws=BASE, V=1000, D=64, ldg=64, B=2, L=77):
    return lib.ivb_token_embed_bwd(ids, B, L, g, ldg, V, D, dt, dp, ws, None)


@cpu_only
@pytest.mark.parametrize("kw", [dict(D=60), dict(ldo=68), dict(ldo=56), dict(V=0)])
def test_token_embed_fwd_shape_refused(kw):
    expect_refusal(_emb_fwd(_lib.load(), **kw), "ivb_token_embed_fwd: V > 0, D and ldo multiples of 8")


@cpu_only
@pytest.mark.parametrize("kw", [dict(table=BASE + 8), dict(pos=BASE + 4), dict(out=BASE + 8)])
def test_token_embed_fwd_alignment_refused(kw):
    expect_refusal(_emb_fwd(_lib.load(), **kw), "ivb_token_embed_fwd: table, pos and out must be 16-byte aligned")


@cpu_only
@pytest.mark.parametrize("kw", [dict(ids=BASE + 4), dict(err=None), dict(err=BASE + 2)])
def test_token_embed_fwd_ids_and_flag_refused(kw):
    expect_refusal(_emb_fwd(_lib.load(), **kw), "ivb_token_embed_fwd: ids must be 8-byte aligned")


@cpu_only
@pytest.mark.parametrize("kw", [dict(D=60), dict(ldg=68), dict(V=-1)])
def test_token_embed_bwd_shape_refused(kw):
    expect_refusal(_emb_bwd(_lib.load(), **kw), "ivb_token_embed_bwd: V > 0, D and ldg multiples of 8")


@cpu_only
@pytest.mark.parametrize("kw", [dict(g=BASE + 8), dict(dt=BASE + 4), dict(dp=BASE + 8)])
def test_token_embed_bwd_alignment_refused(kw):
    expect_refusal(_emb_bwd(_lib.load(), **kw), "ivb_token_embed_bwd: g, dtable and dpos must be 16-byte aligned")


@cpu_only
@pytest.mark.parametrize("kw", [dict(ids=BASE + 4), dict(ws=None), dict(ws=BASE + 2)])
def test_token_embed_bwd_ids_and_workspace_refused(kw):
    expect_refusal(_emb_bwd(_lib.load(), **kw), "ivb_token_embed_bwd: ids must be 8-byte aligned")


def test_token_embed_empty_is_a_noop_and_workspace_size():
    lib = _lib.load()
    assert _emb_fwd(lib, B=0) == 0 and _emb_fwd(lib, L=0) == 0
    assert _emb_bwd(lib, B=0) == 0 and _emb_bwd(lib, L=0) == 0
    assert lib.ivb_token_embed_bwd_workspace_ints(49408, 128, 77) == 2 * 49408 + 2 * 128 * 77


@pytest.mark.parametrize("wrapper,kwargs", [
    ("_token_embed_fwd", dict(ids=torch.zeros(2, 77, dtype=torch.int64), table=torch.zeros(8, 8, dtype=torch.bfloat16),
                              pos=torch.zeros(77, 8, dtype=torch.bfloat16))),
    ("_token_embed_bwd", dict(ids=torch.zeros(2, 77, dtype=torch.int64), g=torch.zeros(154, 8), V=8))])
def test_token_embed_wrappers_refuse_on_the_host(wrapper, kwargs, monkeypatch):
    from internvideo_b200 import lowlevel as ll
    monkeypatch.setattr(ll, "_call", lambda *a, **k: pytest.fail(f"{wrapper} reached the library"))
    with pytest.raises(_lib.IvbError, match="expected a CUDA tensor"):
        getattr(ll, wrapper)(**kwargs)
    for name, t in kwargs.items():
        if torch.is_tensor(t):
            with pytest.raises(_lib.IvbError, match=f"{name}: required operand is None"):
                getattr(ll, wrapper)(**{**kwargs, name: None})
