"""The flash-attention kernels keep their accumulators in registers, and ptxas does not serialise their wgmmas.

A wgmma whose accumulator or A fragment is written between `wgmma.fence` and the commit makes ptxas wait for every
wgmma in flight (warning C7515), which shows in the SASS as one WARPGROUP.DEPBAR per MMA.  Without it the forward
waits four times per kernel (S_0, S_{j+1}, P_j V_j, the last P V), in its bf16 and its E4M3 form alike, and each
backward pass twice (S/dP, the accumulate MMAs).  Reads the SASS of the objects build.py compiled; skips when they or
cuobjdump are absent.
"""
import re

import pytest

import sass

# (object, kernel name, instantiations, WARPGROUP.DEPBAR per kernel)
KERNELS = [("ivb_attn.o", "attn_fwd_kernel", 8, 4), ("ivb_attn_fp8.o", "attn_fwd_fp8_kernel", 4, 4),
           ("ivb_attn_bwd.o", "attn_bwd_kernel", 16, 2)]
# The wgmma instruction of an object's kernels: E4M3 in the FP8 forward, bf16 (HGMMA) everywhere else.
MMA = {"ivb_attn_fp8.o": "QGMMA"}


def _kernels(obj, name):
    """{mangled kernel name: [SASS instruction lines]} of every instantiation of `name` in obj."""
    return {k: v for k, v in sass.functions(obj).items() if re.search(rf"\d{name}I", k)}


@pytest.mark.parametrize("obj,name,count,depbar", KERNELS)
def test_attn_kernels_use_no_local_memory(obj, name, count, depbar):
    kernels = _kernels(obj, name)
    assert len(kernels) == count, sorted(kernels)
    for k, lines in kernels.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, k


@pytest.mark.parametrize("obj,name,count,depbar", KERNELS)
def test_attn_wgmmas_are_not_serialised(obj, name, count, depbar):
    kernels = _kernels(obj, name)
    assert len(kernels) == count, sorted(kernels)
    for k, lines in kernels.items():
        assert sass.count(lines, MMA.get(obj, "HGMMA")) > 0, k
        assert sass.count(lines, r"WARPGROUP\.DEPBAR") == depbar, k
