"""FP8 attention for inference (modules.set_fp8_inference(..., attention=True)) without a GPU.

1. ivb_attn_fp8_pack and ivb_attn_fwd_fp8 refuse a call their kernels cannot serve before any CUDA call.  They are called
   through the raw C ABI with fake device addresses, which must never reach a launch, so these checks run only where no
   CUDA device is visible.
2. The binding's prototypes of the new entry points are the header's.
3. The pack keeps nothing in local memory and the forward issues E4M3 x E4M3 wgmmas only.  The forward's local memory
   and its four WARPGROUP.DEPBAR are checked with the bf16 forward's, in test_attn_sass_cpu.py.
4. set_fp8_inference's attention switch resolves to BlockSpec.attn_fp8, off for head-axis calls, and block_forward
   refuses attn_fp8 where it cannot run it.
"""
import ctypes as C
import re

import pytest
import torch

import sass
from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib

B, N, H, D = 2, 1025, 16, 64
N16 = 1040
SQ, SK, SV = BASE + 0x700000, BASE + 0x710000, BASE + 0x720000


def _pack(q=BASE, ldq=3 * H * D, k=BASE + 2 * H * D, ldk=3 * H * D, v=BASE + 4 * H * D, ldv=3 * H * D, b=B, n=N, h=H,
          d=D, q8=BASE + 0x100000, k8=BASE + 0x200000, ld8=H * D, sq=SQ, sk=SK, vt8=BASE + 0x300000, ldvt=N16, sv=SV):
    return _lib.load().ivb_attn_fp8_pack(q, ldq, k, ldk, v, ldv, b, n, h, d, q8, k8, ld8, sq, sk, vt8, ldvt, sv, None)


def _fwd(q8=BASE + 0x100000, k8=BASE + 0x200000, ld8=H * D, sq=SQ, sk=SK, vt8=BASE + 0x300000, ldvt=N16, sv=SV,
         out=BASE, ldo=H * D, b=B, n=N, h=H, d=D):
    return _lib.load().ivb_attn_fwd_fp8(q8, k8, ld8, sq, sk, vt8, ldvt, sv, out, ldo, b, n, h, d, 0.125, None)


@cpu_only
def test_pack_refusals():
    P = "ivb_attn_fp8_pack: "
    for d in (60, 136, 8):
        expect_refusal(_pack(d=d), P + "head_dim must be a multiple of 8 in [16,128]")
    for kw in (dict(ldq=3 * H * D + 4), dict(ldk=1020), dict(ldv=3)):
        expect_refusal(_pack(**kw), P + "pitches must be multiples of 8")
    for kw in (dict(q=None), dict(k=None), dict(v=None), dict(q8=None), dict(k8=None), dict(vt8=None), dict(sq=None),
               dict(sk=None), dict(sv=None)):
        expect_refusal(_pack(**kw), P + "an operand is null")
    for ld8 in (H * D + 8, H * D - 16):
        expect_refusal(_pack(ld8=ld8), P + "ld8 must be a multiple of 16 and >= H*round_up(d, 32)")
    expect_refusal(_pack(d=88, ld8=16 * 88), P + "ld8 must be a multiple of 16 and >= H*round_up(d, 32)")
    for ldvt in (N, 1032, 1048):   # unpadded, a multiple of 8 below round_up(n, 16), not a multiple of 16
        expect_refusal(_pack(ldvt=ldvt), P + "ldvt must be a multiple of 16 and >= round_up(n, 16)")
    for kw in (dict(q=BASE + 8), dict(k=BASE + 2 * H * D + 8), dict(v=BASE + 8), dict(q8=BASE + 0x100008),
               dict(k8=BASE + 0x200008), dict(vt8=BASE + 0x300008)):
        expect_refusal(_pack(**kw), P + "q, k, v, q8, k8 and vt8 must be 16-byte aligned")
    for kw in (dict(sq=SQ + 4), dict(sk=SK + 8), dict(sv=SV + 2)):
        expect_refusal(_pack(**kw), P + "q_scale_inv and k_scale_inv must be 16-byte aligned, v_scale_inv 4-byte")
    assert _pack(b=0) == 0 and _pack(n=0) == 0   # empty: a no-op, as ivb_attn_fwd


@cpu_only
def test_fwd_refusals():
    P = "ivb_attn_fwd_fp8: "
    for d in (60, 136, 8):
        expect_refusal(_fwd(d=d), P + "head_dim must be a multiple of 8 in [16,128]")
    expect_refusal(_fwd(ldo=H * D + 4), P + "pitches must be multiples of 8")
    for kw in (dict(q8=None), dict(k8=None), dict(vt8=None), dict(out=None), dict(sq=None), dict(sk=None),
               dict(sv=None)):
        expect_refusal(_fwd(**kw), P + "an operand is null")
    for ld8 in (H * D + 8, H * D - 16):
        expect_refusal(_fwd(ld8=ld8), P + "ld8 must be a multiple of 16 and >= H*round_up(d, 32)")
    expect_refusal(_fwd(d=88, ld8=16 * 88), P + "ld8 must be a multiple of 16 and >= H*round_up(d, 32)")
    for ldvt in (N, 1032, 1048):
        expect_refusal(_fwd(ldvt=ldvt), P + "ldvt must be a multiple of 16 and >= round_up(n, 16)")
    for kw in (dict(q8=BASE + 0x100008), dict(k8=BASE + 0x200008), dict(vt8=BASE + 0x300008), dict(sq=SQ + 4),
               dict(sk=SK + 8)):
        expect_refusal(_fwd(**kw), P + "q8, k8, vt8, q_scale_inv and k_scale_inv must be 16-byte aligned")
    for kw in (dict(sv=SV + 4), dict(out=BASE + 2)):
        expect_refusal(_fwd(**kw), P + "v_scale_inv must be 8-byte aligned, out 4-byte")
    assert _fwd(b=0) == 0 and _fwd(n=0) == 0


def test_prototypes_match_the_header():
    P = _lib.parse_prototypes(_lib.HEADER.read_text())
    V, I, L, F = C.c_void_p, C.c_int, C.c_long, C.c_float
    assert P["ivb_attn_fp8_scale_pitch"] == (I, [I])
    assert P["ivb_attn_fp8_pack"] == (I, [V, L, V, L, V, L, I, I, I, I, V, V, L, V, V, V, L, V, V])
    assert P["ivb_attn_fwd_fp8"] == (I, [V, V, L, V, V, V, L, V, V, L, I, I, I, I, F, V])
    lib = _lib.load()
    for name in ("ivb_attn_fp8_scale_pitch", "ivb_attn_fp8_pack", "ivb_attn_fwd_fp8"):
        fn = getattr(lib, name)
        assert (fn.restype, fn.argtypes) == P[name], name
    assert [lib.ivb_attn_fp8_scale_pitch(n) for n in (1, 64, 65, 257, 1025, 2049)] == [64, 64, 128, 320, 1088, 2112]


def test_fp8_attention_kernels_sass():
    funcs = sass.functions("ivb_attn_fp8.o")
    fwd = {k: v for k, v in funcs.items() if "attn_fwd_fp8_kernel" in k}
    pack = {k: v for k, v in funcs.items() if "attn_fp8_pack_kernel" in k}
    assert len(fwd) == 4 and len(pack) == 1, sorted(funcs)     # NO = 32, 64, 96, 128
    for name, lines in pack.items():
        assert not any(re.search(r"\b(LDL|STL)\b", l) for l in lines), name
    for name, lines in fwd.items():
        assert any("QGMMA" in l and "E4M3.E4M3" in l for l in lines), name
        assert not any("HGMMA" in l for l in lines), name


def _fake_quantize_rows(monkeypatch):
    """set_fp8_inference quantises the weights on the device; here a stand-in returns a marker per weight."""
    from internvideo_b200 import modules
    monkeypatch.setattr(modules.ll, "fp8_quantize_rows", lambda w: ("q8", w.shape))


def test_set_fp8_inference_attention_resolves_to_blockspec(monkeypatch):
    from internvideo_b200 import ops
    from internvideo_b200.modules import Block, VideoMAEBlock, set_fp8_inference
    _fake_quantize_rows(monkeypatch)
    blk = Block(64, 2, 4.0, init_values=0.1, qk_normalization=True)
    mae = VideoMAEBlock(64, 2, qkv_bias=True)
    for m in (blk, mae):
        spec = m._spec(2, 17, False)
        assert spec.precision == ops.BF16 and not spec.attn_fp8
        assert set_fp8_inference(m) == 1
        spec = m._spec(2, 17, False)
        assert not isinstance(spec.precision, str) and not spec.attn_fp8     # the default keeps bf16 attention
        assert set_fp8_inference(m, True, attention=True) == 1
        spec = m._spec(2, 17, False)
        assert not isinstance(spec.precision, str) and spec.attn_fp8
        with pytest.raises(_lib.IvbError, match="no gradient"):
            m._spec(2, 17, True)
    assert not mae._spec(2, 17, head_axis=True).attn_fp8               # head-axis attention keeps its kernel
    assert mae._spec(2, 17, head_axis=False).attn_fp8
    set_fp8_inference(blk, True)                                         # attention=False again: off
    assert not blk._spec(2, 17, False).attn_fp8
    set_fp8_inference(blk, True, attention=True)
    assert set_fp8_inference(blk, False, attention=True) == 1            # switching off turns both off
    spec = blk._spec(2, 17, False)
    assert spec.precision == ops.BF16 and not spec.attn_fp8 and not blk.fp8_attention


def test_block_forward_refuses_attn_fp8_outside_inference():
    from internvideo_b200 import ops
    x = torch.zeros((34, 64))                                            # never reaches a device: refused first
    for spec, save in ((ops.BlockSpec(2, 17, 2, attn_fp8=True), True),
                       (ops.BlockSpec(2, 17, 2, layernorm=True, head_axis=True, attn_fp8=True), False)):
        with pytest.raises(_lib.IvbError, match="FP8 attention"):
            ops.block_forward(x, spec, None, save=save)


@cpu_only
@pytest.mark.parametrize("wrapper", ["_attn_fp8_pack", "_attn_fwd_fp8"])
def test_wrappers_check_operands_on_the_host(wrapper, monkeypatch):
    """The lowlevel wrappers make the operand check of every wrapper (test_binding_cpu.py) before the library call."""
    from internvideo_b200 import lowlevel as ll
    monkeypatch.setattr(ll, "_call", lambda *a, **k: pytest.fail(f"{wrapper} reached the library"))
    bf, e4, f32 = torch.bfloat16, torch.float8_e4m3fn, torch.float32
    if wrapper == "_attn_fp8_pack":
        kwargs = dict(q=torch.zeros(8, 16, dtype=bf), k=torch.zeros(8, 16, dtype=bf), v=torch.zeros(8, 16, dtype=bf))
        dims = (1, 8, 1, 16)
    else:
        kwargs = dict(q8=torch.zeros(8, 16, dtype=e4), k8=torch.zeros(8, 16, dtype=e4),
                      q_scale_inv=torch.zeros(1, 1, 64, dtype=f32), k_scale_inv=torch.zeros(1, 1, 64, dtype=f32),
                      vt8=torch.zeros(1, 1, 16, 16, dtype=e4), v_scale_inv=torch.zeros(1, 1, 16, dtype=f32))
        dims = (1, 8, 1, 16, 0.25)
    fn = getattr(ll, wrapper)
    with pytest.raises(_lib.IvbError, match="expected a CUDA tensor"):
        fn(**kwargs, B=dims[0], n=dims[1], H=dims[2], d=dims[3], **({"scale": dims[4]} if len(dims) > 4 else {}))
    for name in kwargs:
        with pytest.raises(_lib.IvbError) as e:
            fn(**{**kwargs, name: None}, B=dims[0], n=dims[1], H=dims[2], d=dims[3],
               **({"scale": dims[4]} if len(dims) > 4 else {}))
        assert str(e.value) == f"{name}: required operand is None"
