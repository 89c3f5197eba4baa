"""Host side of internvideo_b200/videomae_v1.py: constructor surface, state_dict keys and the fixed sinusoid tables of the
InternVideo1 VideoMAE model against the reference module's results stored in the committed golden fixtures."""
import json
from functools import partial
from pathlib import Path

import numpy as np
import pytest
import torch

from internvideo_b200 import videomae_v1 as v1

GOLD = Path(__file__).parent / "golden"


def test_state_dict_keys_match_the_golden_fixture():
    z = np.load(GOLD / "iv1_videomae.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    m = v1.PretrainVisionTransformer(norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), **cfg)
    assert set(m.state_dict()) == {k[2:] for k in z.files if k.startswith("w/")}
    assert m.encoder.patch_embed.num_patches == 32 and tuple(m.pos_embed.shape) == (1, 32, cfg["decoder_embed_dim"])
    assert not isinstance(m.pos_embed, torch.nn.Parameter)          # fixed table, like the reference
    with pytest.raises(Exception):
        m(torch.zeros(1, 3, 16, 32, 32), torch.zeros(1, 32, dtype=torch.bool))     # fp32 / CPU: no CPU path


def test_factories_have_the_published_sizes():
    for fn, enc, dec, p in ((v1.pretrain_mae_small_patch16_224, 384, 192, 16), (v1.pretrain_mae_base_patch16_224, 768, 384, 16)):
        m = fn(decoder_depth=4)
        assert m.encoder.embed_dim == enc and m.decoder.embed_dim == dec and m.decoder.num_classes == 3 * 2 * p * p
        assert m.encoder.blocks[0].attn.q_bias is not None and m.encoder.blocks[0].gamma_1 is None
        assert m.encoder.patch_embed.num_patches == 14 * 14 * 8


def test_tables_and_init_match_reference():
    """Bit-exact against the reference model built under the same seed (SHA-256 of every tensor in
    tests/golden/ref_checks.npz, written by oracle/make_golden.py)."""
    import hashlib
    ref = np.load(Path(__file__).resolve().parent / "golden" / "ref_checks.npz")
    sha = lambda t: np.frombuffer(hashlib.sha256(np.ascontiguousarray(t.detach().numpy()).tobytes()).digest(), np.uint8)
    kw = dict(img_size=32, patch_size=16, encoder_embed_dim=128, encoder_depth=1, encoder_num_heads=2, decoder_num_classes=1536,
              decoder_embed_dim=64, decoder_depth=1, decoder_num_heads=1, qkv_bias=True, init_values=0.1)
    torch.manual_seed(3); mine = v1.PretrainVisionTransformer(**kw)
    assert np.array_equal(ref["iv1/pos_embed"], sha(mine.pos_embed))
    assert np.array_equal(ref["iv1/encoder_pos_embed"], sha(mine.encoder.pos_embed))
    sd_m = mine.state_dict()
    assert bytes(ref["iv1/keys"]).decode().split("\n") == list(sd_m)   # same keys in the same registration order
    for k in sd_m:                                                 # same init draws (xavier / trunc-normal under one seed)
        assert tuple(ref[f"iv1/shape/{k}"]) == tuple(sd_m[k].shape), k
        if "mask_token" not in k:
            assert np.array_equal(ref[f"iv1/sha/{k}"], sha(sd_m[k])), k
    assert float(mine.mask_token.abs().max()) <= 0.02 + 1e-6
