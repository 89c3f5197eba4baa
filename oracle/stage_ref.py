"""TEST / BASELINE INFRASTRUCTURE ONLY — stage the handful of UNMODIFIED reference files this path needs into the
git-ignored oracle/_ref/reference/ (same relative layout as /root/reference), so that they travel to the GPU box
with the gpurun snapshot (oracle/_ref/ is git-ignored but not gpurun-ignored).  There `bench.py --impl reference`, the
`cpu_baseline` leg and tools/ref_gpu_compare.py then execute the reference's own modules (kind: "reference") instead
of the oracle port.  Nothing is copied into the tracked tree; the product never imports any of it.

  python oracle/stage_ref.py          # run where /root/reference is mounted (__graft_entry__.build() does it)
"""
from __future__ import annotations

import shutil
import sys
from pathlib import Path

SRC = Path("/root/reference")
DST = Path(__file__).resolve().parent / "_ref" / "reference"

FILES = [
    # stage-1 student: model, position tables, FA2 seam
    "InternVideo2/single_modality/models/internvideo2_pretrain.py",
    "InternVideo2/single_modality/models/pos_embed.py",
    "InternVideo2/single_modality/models/flash_attention_class.py",
    # contrastive: tower, loss, gather
    "InternVideo2/multi_modality/models/backbones/internvideo2/internvideo2_clip_vision.py",
    "InternVideo2/multi_modality/models/backbones/internvideo2/pos_embed.py",
    "InternVideo2/multi_modality/models/backbones/internvideo2/flash_attention_class.py",
    "InternVideo2/multi_modality/models/criterions.py",
    "InternVideo2/multi_modality/models/utils.py",
    "InternVideo2/multi_modality/utils/easydict.py",
    "InternVideo2/multi_modality/utils/distributed.py",
    # IV1 pixel-target statements
    "InternVideo1/Pretrain/VideoMAE/engine_for_pretraining.py",
    # frozen teachers
    "InternVideo2/single_modality/models/internvl_clip_vision.py",
    "InternVideo2/single_modality/models/videomae.py",
    # stage-2 consumers: tower form, recall@k
    "InternVideo2/multi_modality/models/backbones/internvideo2/internvideo2.py",
    "InternVideo2/multi_modality/tasks_clip/retrieval_utils.py",
    "InternVideo2/multi_modality/models/mask.py",
    "InternVideo2/single_modality/datasets/masking_generator.py",
    # IV1 VideoMAE model
    "InternVideo1/Pretrain/VideoMAE/modeling_pretrain.py",
    "InternVideo1/Pretrain/VideoMAE/modeling_finetune.py",
]


def _mounted() -> bool:
    try:
        return SRC.is_dir()
    except OSError:          # present but not readable by this user
        return False


def stage(verbose=True) -> bool:
    if not _mounted():
        if verbose:
            print(f"stage_ref: {SRC} not mounted; keeping whatever is already under {DST}")
        return DST.is_dir()
    for rel in FILES:
        d = DST / rel
        d.parent.mkdir(parents=True, exist_ok=True)
        shutil.copyfile(SRC / rel, d)
    (DST / "STAGED_FROM").write_text(f"{SRC} (unmodified copies, git-ignored; see oracle/stage_ref.py)\n")
    if verbose:
        print(f"stage_ref: {len(FILES)} reference files -> {DST}")
    return True


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
