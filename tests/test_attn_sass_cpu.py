"""The flash-attention kernels keep their accumulators in registers, and ptxas does not serialise their wgmmas.

A wgmma whose accumulator or A fragment is written between `wgmma.fence` and the commit makes ptxas wait for every
wgmma in flight (warning C7515), which shows in the SASS as one WARPGROUP.DEPBAR per MMA.  Without it the forward
waits four times per kernel (S_0, S_{j+1}, P_j V_j, the last P V) and each backward pass twice (S/dP, the accumulate
MMAs).  Reads the SASS of the objects build.py compiled; skips when they or cuobjdump are absent.
"""
import os
import re
import shutil
import subprocess

import pytest

from internvideo_b200 import build

# (object, kernel name, instantiations, WARPGROUP.DEPBAR per kernel)
KERNELS = [("ivb_attn.o", "attn_fwd_kernel", 8, 4), ("ivb_attn_bwd.o", "attn_bwd_kernel", 16, 2)]


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _kernels(obj, name):
    """{mangled kernel name: [SASS instruction lines]} of every instantiation of `name` in obj."""
    tool = _cuobjdump()
    if tool is None or not (build.OBJ / obj).exists():
        pytest.skip(f"needs cuobjdump and the built internvideo_b200/build/{obj}")
    text = subprocess.run([tool, "-sass", str(build.OBJ / obj)], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", line):
            out[cur].append(line)
    return {k: v for k, v in out.items() if re.search(rf"\d{name}I", k)}


def _count(lines, pattern):
    return sum(1 for l in lines if re.search(pattern, l))


@pytest.mark.parametrize("obj,name,count,depbar", KERNELS)
def test_attn_kernels_use_no_local_memory(obj, name, count, depbar):
    kernels = _kernels(obj, name)
    assert len(kernels) == count, sorted(kernels)
    for k, lines in kernels.items():
        assert _count(lines, r"\b(LDL|STL)\b") == 0, k


@pytest.mark.parametrize("obj,name,count,depbar", KERNELS)
def test_attn_wgmmas_are_not_serialised(obj, name, count, depbar):
    kernels = _kernels(obj, name)
    assert len(kernels) == count, sorted(kernels)
    for k, lines in kernels.items():
        assert _count(lines, r"HGMMA") > 0, k
        assert _count(lines, r"WARPGROUP\.DEPBAR") == depbar, k
