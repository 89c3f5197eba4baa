"""Construction of every vision tower pinned byte for byte: for each configuration, built at a tiny size under a fixed
seed, the state_dict key order, the parameter order and requires_grad flags, every tensor's shape and SHA-256, the plain
(non-parameter) position tables and no_weight_decay() equal tests/golden/tower_init.npz.  The registration order sets the
engine's flat-buffer layout and the init draws set the starting weights, so a reordered registration or a shifted RNG
draw fails here.

The fixture was written by this file's __main__ (`python tests/test_towers_cpu.py`), run in a checkout of the commit
before the towers were built from shared pieces; rerun it only when a tower's construction is meant to change."""
import hashlib
import json
import sys
from functools import partial
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from internvideo_b200 import clip_modules, modules, stage2, teachers, videomae_v1  # noqa: E402

GOLDEN = Path(__file__).parent / "golden" / "tower_init.npz"
OFF = dict(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False)
STUDENT = dict(embed_dim=64, depth=3, num_heads=2, num_frames=4, tubelet_size=2, img_size=28, patch_size=14,
               attn_pool_num_heads=2, clip_embed_dim=16, clip_teacher_embed_dim=32, clip_teacher_final_dim=16,
               clip_return_layer=2, drop_path_rate=0.1, init_values=0.1, **OFF)
TOWER = dict(embed_dim=64, depth=3, num_heads=2, num_frames=4, tubelet_size=2, img_size=28, patch_size=14,
             attn_pool_num_heads=2, clip_embed_dim=16, drop_path_rate=0.1, **OFF)
IV1 = dict(img_size=32, patch_size=16, encoder_embed_dim=64, encoder_depth=2, encoder_num_heads=2,
           decoder_num_classes=1536, decoder_embed_dim=32, decoder_depth=2, decoder_num_heads=1, qkv_bias=True,
           init_values=0.1, drop_path_rate=0.1)

CONFIGS = {
    "student": lambda: modules.PretrainInternVideo2(mae_teacher_embed_dim=64, mae_return_layer=2, **STUDENT),
    "student_sep": lambda: modules.PretrainInternVideo2(mae_teacher_embed_dim=64, mae_return_layer=2,
                                                        sep_pos_embed=True, **STUDENT),
    "stage2": lambda: stage2.PretrainInternVideo2(**STUDENT),
    "stage2_sep_image": lambda: stage2.PretrainInternVideo2(sep_image_video_pos_embed=True, **STUDENT),
    "clip_tower": lambda: clip_modules.InternVideo2(**TOWER),
    "clip_tower_sep": lambda: clip_modules.InternVideo2(sep_pos_embed=True, **TOWER),
    "clip_small": lambda: clip_modules.InternVideo2_CLIP_small(dict(model=dict(
        vision_encoder=dict(TOWER, align_dim=24), temp=0.01, temp_min=0.01, freeze_vision=True,
        open_vision_clip_projector=True))),
    "internvl": lambda: teachers.InternVL_CLIP(img_size=28, patch_size=14, embed_dim=64, depth=3, num_heads=2,
                                               attn_pool_num_heads=2, clip_embed_dim=16, clip_return_layer=2, **OFF),
    "videomae_teacher": lambda: teachers.VisionTransformer(img_size=224, patch_size=16, embed_dim=32, depth=2,
                                                           num_heads=2, qkv_bias=True, init_values=0.1,
                                                           norm_layer=partial(nn.LayerNorm, eps=1e-6)),
    "iv1": lambda: videomae_v1.PretrainVisionTransformer(**IV1),
    "iv1_learnable": lambda: videomae_v1.PretrainVisionTransformer(use_learnable_pos_emb=True, **IV1),
}


def _sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().float().numpy()).tobytes()).hexdigest()


def describe(name):
    """Everything construction decides for one configuration, as a JSON-able dict."""
    torch.manual_seed(0)
    m = CONFIGS[name]()
    sd = m.state_dict()
    tables = {f"{mn}.{k}".lstrip("."): [list(v.shape), _sha(v)]
              for mn, mod in m.named_modules() for k, v in vars(mod).items()
              if isinstance(v, torch.Tensor) and not isinstance(v, nn.Parameter)}
    nwd = m.no_weight_decay() if hasattr(m, "no_weight_decay") else None
    return dict(keys=list(sd), shapes=[list(v.shape) for v in sd.values()], sha=[_sha(v) for v in sd.values()],
                params=[[n, p.requires_grad] for n, p in m.named_parameters()], tables=tables,
                no_weight_decay=None if nwd is None else sorted(nwd))


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_tower_construction_matches_golden(name):
    want = json.loads(bytes(np.load(GOLDEN)[name]).decode())
    got = describe(name)
    assert got["keys"] == want["keys"]                       # same keys in the same registration order
    assert got["params"] == want["params"]                   # parameters() order and requires_grad
    for k, shape, ws, gs in zip(got["keys"], got["shapes"], want["sha"], got["sha"]):
        assert shape == want["shapes"][got["keys"].index(k)], k
        assert gs == ws, k                                   # same init draws
    assert got["tables"] == want["tables"]
    assert got["no_weight_decay"] == want["no_weight_decay"]


if __name__ == "__main__":
    out = {name: np.frombuffer(json.dumps(describe(name)).encode(), np.uint8) for name in sorted(CONFIGS)}
    np.savez_compressed(GOLDEN, **out)
    print(f"wrote {GOLDEN}: {', '.join(sorted(out))}")
