"""The stage-2 BERT text encoder without a GPU: the CPU restatement against tests/golden/bert_text.npz (outputs of the
unmodified reference BertModel), the port's state_dict keys, order and shapes against the reference's, the key lengths
of a padding mask, and the module's refusals."""
from pathlib import Path

import numpy as np
import pytest
import torch

from internvideo_b200 import _lib
from internvideo_b200.bert_modules import BERT_LARGE, BertModel, key_lengths
from oracle import bert_text

GOLD = Path(__file__).parent / "golden" / "bert_text.npz"
NARROW = dict(bert_text.CFG)


def test_restatement_matches_golden():
    cfg, sd, (pw, pb), z = bert_text.load(GOLD)
    last = bert_text.restate(sd, torch.from_numpy(z["ids"]), torch.from_numpy(z["mask"]), cfg)
    torch.testing.assert_close(last, torch.from_numpy(z["last_hidden_state"]), atol=2e-5, rtol=0)
    torch.testing.assert_close(last[:, 0], torch.from_numpy(z["pooled"]), atol=2e-5, rtol=0)
    torch.testing.assert_close(torch.nn.functional.linear(last[:, 0], pw, pb), torch.from_numpy(z["text_proj"]),
                               atol=2e-5, rtol=0)


def test_golden_captions_cover_the_cases():
    """Caption lengths 2, 17, 39 and 40 (the last unpadded), right padding, repeated ids inside a caption."""
    z = np.load(GOLD)
    assert z["mask"].sum(1).tolist() == [2, 17, 39, 40]
    assert (z["ids"][z["mask"] == 0] == 0).all()
    assert all(len(set(r[:n].tolist())) < n for r, n in zip(z["ids"][1:], (17, 39, 40)))


@pytest.mark.skipif(not bert_text.available(), reason="needs the reference's xbert.py")
@pytest.mark.parametrize("cfg", [NARROW, BERT_LARGE], ids=["narrow", "bert_large"])
def test_state_dict_matches_reference(cfg):
    """Same keys in the same order with the same shapes, so that a stage-2 checkpoint's text_encoder.bert.* loads with
    strict=True.  Built on the meta device: BERT-large's 335M parameters need no memory there."""
    with torch.device("meta"):
        ref = bert_text.build_reference(cfg).state_dict()
        port = BertModel(cfg).state_dict()
    assert list(port) == list(ref)
    for k in ref:
        assert port[k].shape == ref[k].shape and port[k].dtype == ref[k].dtype, k


def test_port_loads_the_golden_state_dict():
    cfg, sd, _, _ = bert_text.load(GOLD)
    BertModel(cfg).load_state_dict(sd, strict=True)


def test_key_lengths():
    """Right-padded rows give their token counts; a row with a gap, a leading zero or no ones gives 0; None gives L."""
    m = torch.tensor([[1, 1, 0, 0], [1, 1, 1, 1], [1, 0, 1, 0], [0, 1, 1, 0], [0, 0, 0, 0], [1, 0, 0, 0]])
    assert key_lengths(m, 6, 4, "cpu").tolist() == [2, 4, 0, 0, 0, 1]
    assert key_lengths(m.bool(), 6, 4, "cpu").tolist() == [2, 4, 0, 0, 0, 1]
    assert key_lengths(None, 3, 4, "cpu").tolist() == [4, 4, 4]
    assert key_lengths(m, 6, 4, "cpu").dtype == torch.int32


def _model(**kw):
    return BertModel(dict(NARROW, **kw)).eval().requires_grad_(False)


def test_constructor_refusals():
    with pytest.raises(NotImplementedError, match="absolute"):
        BertModel(dict(NARROW, position_embedding_type="relative_key"))
    with pytest.raises(NotImplementedError, match="gelu"):
        BertModel(dict(NARROW, hidden_act="relu"))
    with pytest.raises(NotImplementedError, match="pooler"):
        BertModel(NARROW, add_pooling_layer=True)


@pytest.mark.parametrize("mode", ["fusion", "multi_modal"])
def test_cross_attention_modes_refused(mode):
    with pytest.raises(NotImplementedError, match="cross-attention"):
        _model()(torch.zeros(2, 40, dtype=torch.int64), mode=mode)


def test_call_refusals():
    ids = torch.zeros(2, 40, dtype=torch.int64)
    with pytest.raises(NotImplementedError, match="dropout"):
        _model().train()(ids)
    with pytest.raises(NotImplementedError, match="forward-only"):
        BertModel(NARROW).eval()(ids)
    with pytest.raises(NotImplementedError, match="token type"):
        _model()(ids, token_type_ids=torch.ones_like(ids))
    with pytest.raises(_lib.IvbError, match="bf16"):
        _model()(ids)
    with pytest.raises(_lib.IvbError, match="CUDA"):
        _model().bfloat16()(ids)
    with pytest.raises(ValueError, match="mode"):
        _model()(ids, mode="image")


def test_no_grad_and_no_dropout_pass_the_checks():
    """A module in train mode without dropout, or one called under no_grad, or with all-zero token types, gets past
    the refusals to the input checks (bf16 parameters, CUDA ids)."""
    ids = torch.zeros(2, 40, dtype=torch.int64)
    train = BertModel(dict(NARROW, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)).train()
    with torch.no_grad(), pytest.raises(_lib.IvbError, match="bf16"):
        train(ids, token_type_ids=torch.zeros_like(ids), mode="temporal")
