"""The norm backward is two kernels: norm_bwd_kernel streams a row (RMSNorm, LayerNorm and the decoder head's LN -> L2
backward), norm_bwd_rows_kernel holds it in registers (RMSNorm up to D = 1536, the q/k pair, LN -> L2 up to C = 3328),
and no instantiation of either touches local memory.  The decoder head lives in ivb_norm.cu, so ivb_loss.o has no
LN -> L2 kernel and no column-sum scratch of its own.  Reads the SASS of the objects build.py compiled; skips when they
or cuobjdump are absent.
"""
import re

import pytest

import sass


@pytest.mark.parametrize("pattern, count", [
    # XF32 x LN x DXF32, and the LN -> L2 form with a bf16 or fp32 gradient
    (r"\d+norm_bwd_kernelI", 10),
    # XF32 x DXF32 x NCH 2/4/6, the pair at NCH 2/4/6, and LN -> L2 at NCH 3/6/13
    (r"\d+norm_bwd_rows_kernelI", 18),
])
def test_norm_bwd_instantiations_keep_nothing_in_local_memory(pattern, count):
    found = {k: v for k, v in sass.functions("ivb_norm.o").items() if re.search(pattern, k)}
    assert len(found) == count, sorted(found)
    for name, lines in found.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, name


def test_loss_object_has_no_norm_backward_or_colred_scratch():
    names = sass.functions("ivb_loss.o")
    assert names, "ivb_loss.o holds no kernels"
    assert not [k for k in names if "ln_l2" in k or "colred_finish_kernel" in k], sorted(names)
