"""The stage-2 BERT text encoder on the H100 against tests/golden/bert_text.npz (outputs of the unmodified reference
BertModel in text mode; <= 1e-2 relative, as for the text tower), its pooled feature through text_proj and
stage2.retrieval_scores, one forward replayed from a CUDA graph, and the NaN conventions for a bad mask and a bad id."""
from pathlib import Path

import pytest
import torch

from oracle import bert_text

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden" / "bert_text.npz"


def _rel(a, b):
    a = a.detach().float().cpu(); b = b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _model():
    from internvideo_b200.bert_modules import BertModel
    cfg, sd, proj, z = bert_text.load(GOLD)
    model = BertModel(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.bfloat16().cuda().eval().requires_grad_(False)
    ids, mask = (torch.from_numpy(z[k]).cuda() for k in ("ids", "mask"))
    return model, [t.cuda().to(torch.bfloat16) for t in proj], ids, mask, z


def test_bert_text_matches_reference_golden(cuda_lib):
    model, (pw, pb), ids, mask, z = _model()
    last = model(ids, attention_mask=mask, return_dict=True, mode="text").last_hidden_state
    assert last.shape == (4, 40, 128) and last.dtype == torch.bfloat16
    assert _rel(last, torch.from_numpy(z["last_hidden_state"])) < 1e-2
    for b, n in enumerate(bert_text.LENGTHS):        # the valid rows of each caption on their own
        assert _rel(last[b, :n], torch.from_numpy(z["last_hidden_state"][b, :n])) < 1e-2, b
    pooled = last[:, 0]
    assert _rel(pooled, torch.from_numpy(z["pooled"])) < 1e-2
    feat = cuda_lib.gemm(pooled.contiguous(), pw, bias=pb)
    assert _rel(feat, torch.from_numpy(z["text_proj"])) < 1e-2
    same = model(ids, attention_mask=mask, mode="temporal").last_hidden_state
    assert torch.equal(same, last)


def test_text_features_through_retrieval_scores(cuda_lib):
    """The text_proj features as stage-2 evaluation scores them: against 16 random video features, the port's scores
    are the reference features' scores (<= 2e-2 relative); with the reference features as the videos, each caption
    retrieves its own."""
    from internvideo_b200.stage2 import recall_at_k, retrieval_scores
    model, (pw, pb), ids, mask, z = _model()
    feat = cuda_lib.gemm(model(ids, attention_mask=mask).last_hidden_state[:, 0].contiguous(), pw, bias=pb)
    ref = torch.from_numpy(z["text_proj"]).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    video = torch.randn(16, ref.shape[1], device="cuda", generator=g)
    for name, got, want in zip(("i2t_dsl", "t2i_dsl", "i2t", "t2i"), retrieval_scores(video, feat),
                               retrieval_scores(video, ref)):
        assert got.shape == want.shape and _rel(got, want) < 2e-2, (name, _rel(got, want))
    dsl, dsl_t, _, _ = retrieval_scores(ref, feat)
    rec = recall_at_k(dsl, dsl_t, list(range(4)), list(range(4)), ks=(1,))
    assert rec["txt_r1"] == 100.0 and rec["img_r1"] == 100.0, (rec, dsl)


def test_forward_replays_from_a_cuda_graph(cuda_lib):
    model, _, ids, mask, _ = _model()
    eager = model(ids, attention_mask=mask).last_hidden_state
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model(ids, attention_mask=mask)              # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = model(ids, attention_mask=mask).last_hidden_state
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    mask2 = mask.clone()
    mask2[3, 20:] = 0                                # new key lengths, read on the device at replay
    mask.copy_(mask2)
    graph.replay()
    assert torch.equal(out, model(ids, attention_mask=mask2).last_hidden_state)


def test_bad_mask_poisons_only_its_caption_and_bad_id_everything(cuda_lib):
    model, _, ids, mask, _ = _model()
    good = model(ids, attention_mask=mask).last_hidden_state
    bad = mask.clone()
    bad[1, 5] = 0                                    # a gap: not right padding
    bad[2] = 0                                       # no token at all
    out = model(ids, attention_mask=bad).last_hidden_state
    assert bool(torch.isnan(out[1:3]).all())
    assert torch.equal(out[0], good[0]) and torch.equal(out[3], good[3])
    ids_bad = ids.clone()
    ids_bad[0, 1] = model.config.vocab_size
    assert bool(torch.isnan(model(ids_bad, attention_mask=mask).last_hidden_state).all())
