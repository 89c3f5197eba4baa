"""The GEMM kernels hold one copy of the fused epilogue body, and their accumulators stay in registers.

The epilogue walks a tile in chunks of 32 columns in a rolled loop (epilogue_tile, ivb_gemm.cu).  Unrolled, each of the
8 chunks of a 128 x 128 tile carried its own copy of all six epilogue forms: 512 MUFU.TANH (8 copies x 4 tanh sites x
16 elements) and 17 K instructions per kernel, and the fc1 epilogue ran at the speed of the instruction fetch.  One copy
has 64.  Only the fragment -> staging copy is selected per chunk, with constant indices into the accumulators, so no
kernel may touch local memory.  Reads the SASS of the object build.py compiled; skips when it or cuobjdump is absent.
"""
import pytest

import sass


@pytest.fixture(scope="module")
def kernels():
    """{kernel name: [SASS instruction lines]} of every GEMM kernel in ivb_gemm.o."""
    out = {k: v for k, v in sass.functions("ivb_gemm.o").items() if "gemm_bf16" in k}
    assert any("pingpong" in k for k in out), sorted(out)
    return out


def test_every_gemm_kernel_holds_one_epilogue_body(kernels):
    for name, lines in kernels.items():
        tanh = sass.count(lines, r"MUFU\.TANH")
        assert 0 < tanh <= 64, (name, tanh)


def test_gemm_kernels_use_no_local_memory(kernels):
    for name, lines in kernels.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, name
