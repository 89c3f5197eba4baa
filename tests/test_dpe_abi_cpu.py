"""ivb_dpe_ln_fwd (InternVideo-MM's extractor position conv + key LayerNorm): its prototype comes from the header, it
refuses bad operands before any CUDA call (fake device addresses, tests/abi_fake.py), its SASS keeps nothing in local
memory and has no float atomics, and every kernel of the other objects has the SASS recorded in
tests/golden/kernel_sass.json (cuobjdump -sass, function by function, address and encoding comments stripped;
tools/kernel_sass.py wrote it and rewrites it after an intended kernel change)."""
import ctypes as C
import json
import sys
from pathlib import Path

import pytest

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

X, CW, CB, LW, LB, Y = (BASE + k * 0x10000000 for k in range(6))
GOLDEN = Path(__file__).resolve().parent / "golden" / "kernel_sass.json"
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
from kernel_sass import digest  # noqa: E402


def test_prototype_from_header():
    res, args = _lib.PROTOTYPES["ivb_dpe_ln_fwd"]
    assert res is C.c_int
    assert args == [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long, C.c_void_p]


def _call(x=X, f32=1, ldx=1024, cw=CW, cb=CB, lw=LW, lb=LB, N=2, T=8, H=16, W=16, Cc=1024, y=Y, ldy=1024):
    return _lib.load().ivb_dpe_ln_fwd(x, f32, ldx, cw, cb, lw, lb, 1e-5, N, T, H, W, Cc, y, ldy, None)


@cpu_only
def test_refusals():
    for k in ("x", "cw", "cb", "lw", "lb", "y"):
        expect_refusal(_call(**{k: None}), "x, conv_w, conv_b, ln_w, ln_b and y are required")
    for bad in (dict(T=0), dict(H=0), dict(W=0), dict(N=-1)):
        expect_refusal(_call(**bad), "T, H, W >= 1")
    for c in (4, 1020, 4104):
        expect_refusal(_call(Cc=c, ldx=4104, ldy=4104), "C must be a multiple of 8 in [8, 4096]")
    expect_refusal(_call(ldx=1028), "ldx and ldy must be multiples of 8")
    expect_refusal(_call(ldy=1016), ">= C")
    for k in ("x", "cb", "lw", "lb", "y"):
        expect_refusal(_call(**{k: dict(x=X, cb=CB, lw=LW, lb=LB, y=Y)[k] + 8}), "must be 16-byte aligned")
    expect_refusal(_call(cw=CW + 1), "conv_w must be 2-byte aligned")
    assert _call(N=0) == 0                       # no clips: a no-op


def test_dpe_sass_no_local_memory_no_float_atomics():
    found = {k: v for k, v in sass.functions("ivb_dpe.o").items() if "dpe_ln_fwd_kernel" in k}
    assert len(found) == 2, sorted(found)              # the fp32 and the bf16 stream
    for k, lines in found.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, k
        assert sass.count(lines, r"\b(ATOM|RED)[GS]?\.\S*ADD\.(F16|BF16|F32|F64)") == 0, k


def test_other_kernels_keep_their_sass():
    golden = json.loads(GOLDEN.read_text())
    for obj, kernels in golden.items():
        got = {k: digest(v) for k, v in sass.functions(obj).items()}
        assert got == kernels, f"{obj}: SASS differs from the record (after an intended change: tools/kernel_sass.py)"
