"""Every floating-point sum the library returns is taken in a fixed order: no kernel adds floats with a global or shared
atomic, whose result would depend on the order in which CTAs finish (include/ivb200.h, Conventions).  The losses and
dtemp store one partial per CTA and a finish launch adds them in CTA order; the kernels that do so, and the pooling
kernels that share their CTA reduction, keep nothing in local memory.  Reads the SASS of the objects build.py compiled;
skips when they or cuobjdump are absent.
"""
import re

import pytest

import sass
from internvideo_b200 import build

FLOAT_ATOMIC_ADD = r"\b(ATOM|RED)[GS]?\.\S*ADD\.(F16|BF16|F32|F64)"

# scatter_add_kernel adds the position-table gradient with 128-bit vector reductions, but it runs one launch per clip
# and within a clip every table row is reached by exactly one token, so each element receives at most one add per
# launch and the launches are stream-ordered: the sum is still taken in clip order.
EXEMPT = {"scatter_add_kernel"}


def test_no_kernel_adds_floats_with_atomics():
    found = []
    for src in build.sources():
        for name, lines in sass.functions(src.stem + ".o").items():
            if any(re.search(rf"\d{k}[IE]", name) for k in EXEMPT):
                continue
            if sass.count(lines, FLOAT_ATOMIC_ADD):
                found.append(f"{src.stem}.o: {name}")
    assert not found, found


def test_scatter_add_is_the_exempt_kernel():
    """The exemption names a kernel that exists and still uses float reductions: it does not hide a renamed one."""
    kernels = {k: v for k, v in sass.functions("ivb_embed.o").items() if re.search(r"\d+scatter_add_kernelI", k)}
    assert kernels
    assert all(sass.count(lines, FLOAT_ATOMIC_ADD) for lines in kernels.values()), sorted(kernels)


@pytest.mark.parametrize("obj,name,count", [
    ("ivb_norm.o", "ln_l2_fwd_kernel", 2),      # bf16 or fp32 target
    ("ivb_loss.o", "vtc_stats_kernel", 1),
    ("ivb_loss.o", "vtc_grad_kernel", 1),
    ("ivb_loss.o", "mse_kernel", 1),
    ("ivb_loss.o", "pool_attn_fwd_kernel", 1),
    ("ivb_loss.o", "pool_attn_bwd_kernel", 1),
])
def test_loss_kernels_keep_nothing_in_local_memory(obj, name, count):
    found = {k: v for k, v in sass.functions(obj).items() if re.search(rf"\d{name}[IE]", k)}
    assert len(found) == count, sorted(found)
    for k, lines in found.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, k
