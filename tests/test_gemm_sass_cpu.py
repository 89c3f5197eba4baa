"""The GEMM kernels hold one copy of the fused epilogue body, and their accumulators stay in registers.

The epilogue walks a tile in chunks of 32 columns in a rolled loop (epilogue_tile, ivb_gemm.cu).  Unrolled, each of the
8 chunks of a 128 x 128 tile carried its own copy of all six epilogue forms: 512 MUFU.TANH (8 copies x 4 tanh sites x
16 elements) and 17 K instructions per kernel, and the fc1 epilogue ran at the speed of the instruction fetch.  One copy
has 64.  Only the fragment -> staging copy is selected per chunk, with constant indices into the accumulators, so no
kernel may touch local memory.  Reads the SASS of the object build.py compiled; skips when it or cuobjdump is absent.
"""
import os
import re
import shutil
import subprocess

import pytest

from internvideo_b200 import build

OBJ = build.OBJ / "ivb_gemm.o"


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def kernels():
    """{kernel name: [SASS instruction lines]} of every GEMM kernel in ivb_gemm.o."""
    tool = _cuobjdump()
    if tool is None or not OBJ.exists():
        pytest.skip("needs cuobjdump and the built internvideo_b200/build/ivb_gemm.o")
    text = subprocess.run([tool, "-sass", str(OBJ)], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", line):
            out[cur].append(line)
    out = {k: v for k, v in out.items() if "gemm_bf16" in k}
    assert any("pingpong" in k for k in out), sorted(out)
    return out


def _count(lines, pattern):
    return sum(1 for l in lines if re.search(pattern, l))


def test_every_gemm_kernel_holds_one_epilogue_body(kernels):
    for name, lines in kernels.items():
        tanh = _count(lines, r"MUFU\.TANH")
        assert 0 < tanh <= 64, (name, tanh)


def test_gemm_kernels_use_no_local_memory(kernels):
    for name, lines in kernels.items():
        assert _count(lines, r"\b(LDL|STL)\b") == 0, name
