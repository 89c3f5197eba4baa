"""Argument checks of the key-length attention forward (ivb_attn_fwd_keylen) through the raw C ABI, and its kernels'
SASS: no local memory, and the forward's four WARPGROUP.DEPBAR (the wgmmas are not serialised), as
tests/test_attn_sass_cpu.py checks for the other attention kernels."""
import re

import pytest

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

D8 = 16 * 64


def _fwd(lib, kv_len=BASE, d=64, H=16, ld=(3 * D8, 3 * D8, 3 * D8, D8), B=64, n=40):
    return lib.ivb_attn_fwd_keylen(BASE, ld[0], BASE, ld[1], BASE, ld[2], BASE, ld[3], None, B, n, H, d, 0.125, kv_len,
                                   None)


def test_null_kv_len_refused():
    lib = _lib.load()
    expect_refusal(_fwd(lib, kv_len=None), "ivb_attn_fwd_keylen: kv_len is null")
    expect_refusal(_fwd(lib, kv_len=None, B=0), "ivb_attn_fwd_keylen: kv_len is null")


@cpu_only
@pytest.mark.parametrize("d", [8, 12, 136, 0])
def test_head_dim_refused(d):
    expect_refusal(_fwd(_lib.load(), d=d), "ivb_attn_fwd_keylen: head_dim must be a multiple of 8 in [16,128]")


@cpu_only
@pytest.mark.parametrize("slot", range(4))
def test_pitch_refused(slot):
    ld = [3 * D8] * 3 + [D8]
    ld[slot] += 4
    expect_refusal(_fwd(_lib.load(), ld=ld), "ivb_attn_fwd_keylen: pitches must be multiples of 8")


def test_empty_is_a_noop():
    lib = _lib.load()
    assert _fwd(lib, B=0) == 0 and _fwd(lib, n=0) == 0


KERNEL = "attn_fwd_keylen_kernel"


def _kernels():
    return {k: v for k, v in sass.functions("ivb_attn_keylen.o").items() if re.search(rf"\d{KERNEL}I", k)}


def test_keylen_kernels_use_no_local_memory_and_keep_four_depbars():
    kernels = _kernels()
    assert len(kernels) == 8, sorted(kernels)
    for k, lines in kernels.items():
        assert sass.count(lines, r"\b(LDL|STL)\b") == 0, k
        assert sass.count(lines, r"HGMMA") > 0, k
        assert sass.count(lines, r"WARPGROUP\.DEPBAR") == 4, k
