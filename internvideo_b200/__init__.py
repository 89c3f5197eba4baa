"""internvideo_b200 — H100-native (sm_90a) compute path for InternVideo2 pre-training.

Only the hot path named in BASELINE.json/north_star lives here: the C-ABI CUDA library
(csrc/ -> libivb200.so, declared in include/ivb200.h) and the PyTorch-facing mirror of the
reference's nn.Module surface.  See DESIGN.md.
"""
__version__ = "0.1.0"
