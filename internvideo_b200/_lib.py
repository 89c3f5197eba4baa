"""ctypes binding of libivb200.so (the C ABI in include/ivb200.h).

There is no fallback: if the shared library is missing, or a compute entry point is called
without an H100-class (sm_90) device, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libivb200.so"

_vp, _i, _l, _f = C.c_void_p, C.c_int, C.c_long, C.c_float

# name -> (restype, argtypes); must list every symbol declared in include/ivb200.h
PROTOTYPES = {
    "ivb_last_error": (C.c_char_p, []),
    "ivb_version": (_i, []),
    "ivb_device_check": (_i, []),
    "ivb_launch_count": (_l, []),
    "ivb_reset_launch_count": (None, []),
    "ivb_set_default_2cta": (None, [_i]),
    "ivb_gemm_bf16": (_i, [_vp, _i, _l, _vp, _i, _l, _i, _i, _i, _i, _i, _vp, _l, _vp, _l, _vp, _vp,
                           _vp, _l, _vp, _i, _vp]),
    "ivb_fp8_quantize": (_i, [_vp, _l, _i, _i, _i, _vp, _l, _vp, _l, _vp, _vp, _vp]),
    "ivb_gemm_fp8": (_i, [_vp, _i, _l, _i, _vp, _vp, _i, _l, _vp, _i, _i, _i, _i, _i, _vp, _l, _vp, _l, _vp, _vp,
                          _vp, _l, _vp, _i, _vp]),
    "ivb_fp8_quantize_rows": (_i, [_vp, _l, _i, _i, _vp, _l, _vp, _vp]),
    "ivb_norm_fwd_fp8": (_i, [_vp, _i, _l, _vp, _vp, _f, _i, _i, _i, _vp, _l, _vp, _vp]),
    "ivb_norm_fwd": (_i, [_vp, _i, _l, _vp, _vp, _f, _i, _i, _i, _vp, _l, _vp, _vp, _vp]),
    "ivb_norm_bwd": (_i, [_vp, _l, _vp, _i, _l, _vp, _vp, _vp, _i, _i, _i, _vp, _l, _vp, _i, _l,
                          _vp, _vp, _vp]),
    "ivb_rmsnorm_pair_fwd": (_i, [_vp, _l, _l, _vp, _vp, _f, _i, _i, _vp, _l, _l, _vp, _vp]),
    "ivb_rmsnorm_pair_bwd": (_i, [_vp, _l, _l, _vp, _l, _l, _vp, _vp, _vp, _i, _i, _vp, _l, _l, _vp, _vp, _vp]),
    "ivb_rmsnorm_bwd_layerscale": (_i, [_vp, _l, _vp, _l, _vp, _vp, _i, _i, _vp, _l, _vp, _l, _vp, _vp, _l, _vp, _vp, _vp, _l,
                                        _vp, _vp, _vp]),
    "ivb_layerscale_bwd": (_i, [_vp, _l, _vp, _l, _vp, _i, _i, _vp, _l, _vp, _vp, _vp, _vp]),
    "ivb_colsum_bf16": (_i, [_vp, _l, _i, _i, _vp, _vp]),
    "ivb_attn_fwd": (_i, [_vp, _l, _vp, _l, _vp, _l, _vp, _l, _vp, _i, _i, _i, _i, _f, _vp]),
    "ivb_headaxis_attn_fwd": (_i, [_vp, _l, _i, _i, _i, _i, _f, _vp, _vp]),
    "ivb_attn_bwd": (_i, [_vp, _l, _vp, _l, _vp, _l, _vp, _l, _vp, _l, _vp, _vp, _vp, _l, _vp, _l,
                          _vp, _l, _i, _i, _i, _i, _f, _vp]),
    "ivb_attn_bwd_workspace_floats": (_l, [_i, _i, _i]),
    "ivb_visible_indices": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "ivb_im2col_visible": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ivb_gather_add": (_i, [_vp, _l, _vp, _vp, _i, _i, _i, _i, _i, _vp, _i, _l, _vp]),
    "ivb_scatter_add": (_i, [_vp, _i, _l, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "ivb_ln_l2_fwd": (_i, [_vp, _l, _vp, _vp, _f, _i, _i, _vp, _l, _vp, _vp, _i, _l, _vp, _vp]),
    "ivb_ln_l2_bwd": (_i, [_vp, _l, _vp, _vp, _vp, _i, _i, _vp, _i, _l, _f, _vp, _vp, _l, _vp, _vp, _vp]),
    "ivb_vtc_loss_fwd": (_i, [_vp, _vp, _i, _f, _vp, _vp, _vp, _vp, _vp]),
    "ivb_vtc_loss_bwd": (_i, [_vp, _vp, _i, _f, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp]),
    "ivb_l2norm_rows_fwd": (_i, [_vp, _i, _l, _i, _i, _vp, _l, _vp, _vp]),
    "ivb_l2norm_rows_bwd": (_i, [_vp, _l, _vp, _l, _vp, _i, _i, _vp, _l, _vp]),
    "ivb_pixel_targets": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "ivb_mse_loss": (_i, [_vp, _vp, _l, _vp, _f, _vp, _vp, _vp]),
    "ivb_pool_attn_fwd": (_i, [_vp, _vp, _l, _vp, _l, _i, _i, _i, _i, _f, _vp, _vp, _vp]),
    "ivb_pool_attn_bwd": (_i, [_vp, _vp, _l, _vp, _l, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _l, _vp, _l, _vp]),
    "ivb_adamw_step": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _l, _f, _f, _f, _f, _f, _i, _f, _vp, _vp, _vp]),
    "ivb_nvls_allreduce_bf16": (_i, [_vp, _l, _l, _vp, _i, _i, _i, _vp]),
    "ivb_nvls_flag_words": (_i, []),
}

_lib = None


class IvbError(RuntimeError):
    pass


def load(build_if_missing: bool = False) -> C.CDLL:
    """Load libivb200.so and attach prototypes. Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        if build_if_missing or os.environ.get("IVB200_AUTOBUILD") == "1":
            from . import build as _b
            _b.build()
        else:
            raise IvbError(
                f"{LIB_PATH} not found: build it with `python -m internvideo_b200.build` "
                "(there is no CPU / PyTorch fallback for the ivb200 compute path)")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().ivb_last_error().decode(errors="replace")
        raise IvbError(f"{what} failed (rc={rc}): {msg}")


def header_symbols() -> list[str]:
    """Function names declared in include/ivb200.h (used by the CPU ABI test)."""
    import re
    text = (_PKG.parent / "include" / "ivb200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ivb_[a-z0-9_]+)\s*\(", text)))
