"""FP8 attention for inference (lowlevel._attn_fp8_pack + _attn_fwd_fp8, modules.set_fp8_inference(attention=True))
on the H100 (gpu).

Kernel level, at d in {64, 88, 128} x n in {257, 417, 1025, 2049} (sequence tails at every n but 1025's 1024 + 1), at
every head dim at n = 190, and at n in {1, 63, 64, 65, 129} (SHAPES), two clips, q / k / v the three column slots of
one [B*n, 3*H*d] projection buffer (row pitch 3D), as the blocks pass them:
1. The pack is bit-exact against a torch emulation of its scale rule (the power-of-two rule of ivb_fp8_quantize_rows
   per (token, head) and per (clip, head, channel)) and of the E4M3 cast: q8 and k8 with their zero head padding, vt8
   with its zero key padding, and every scale; an Inf in one head of a q row or in one channel of v gives scale_inv NaN
   and the satfinite cast's +-448 for that group alone.
2. The forward against a float64 emulation of its own arithmetic on the dequantised q8, k8 and vt8: the online softmax
   over 64-key tiles with P = exp2(S - m + 8) rounded to E4M3 where the kernel rounds it.  That isolates the kernel's
   arithmetic from the casts.  The kernel's fp32 P (ex2.approx) and the emulation's float64 P fall on different sides
   of an E4M3 rounding midpoint for a few elements; each such element moves its output row by up to 2^-4 of one term
   P v, which next to an output element near 0 is a large relative error.  So the bound is on the tile error of
   attn_ref.tile_errors (rms error of a 64-row band over the rms of its head): EMULATION_BOUND, about twice the largest
   value measured on an H100 (0.0059-0.0267 over the twelve model shapes; the largest in one-row tail bands, where no
   averaging over rows takes place; the head-dim and short-sequence shapes at most 0.0077, H100 80GB HBM3 at 700 W).
3. The forward against the bf16 kernel on the same bf16 inputs, which adds the casts' error: the tile error of
   attn_ref.tile_errors is held to FP8_VS_BF16.  E4M3 rounds with relative error at most u = 2^-4, about 0.036 rms;
   q and k each carry one rounding, so S errs by about 0.05 rms of its terms' scale, which P inherits as a relative
   error, and P and V each carry one more: about 0.07 rms in all.  Measured on an H100: 0.058-0.106, the largest again in
   a one-row tail band (the head-dim and short-sequence shapes: at most 0.086); FP8_VS_BF16 is about twice that.  The
   inputs are N(0, 1) as in a normed block; spreading the tokens' magnitudes (the pack test's inputs) makes the
   softmax peaked and the same casts err by 0.15-0.43.

Model level: set_fp8_inference(model, attention=True) against set_fp8_inference(model) (FP8 GEMMs, bf16 attention) on a
depth-2 L-dims CLIP tower (n = 1025, d = 64), the unmasked stage-2 tower (n = 2049, d = 88) and the VideoMAEv2 teacher
with token-axis attention (n = 2048, d = 88): relative error at most MODEL_BOUND = 2u, the bound of one E4M3 rounding of
each GEMM operand (test_teachers_fp8_gpu.py).  The outputs stay far inside it, so they are also held to MODEL_LIMIT.
Switching attention off again gives the FP8-inference bits, switching FP8 inference off the bf16 bits, and a forward
that needs a gradient is refused.
"""
import math
from functools import partial

import pytest
import torch

from attn_ref import tile_errors, worst

pytestmark = pytest.mark.gpu

LOG2E = math.log2(math.e)
E4M3 = torch.float8_e4m3fn
EMULATION_BOUND = 0.06
FP8_VS_BF16 = 0.2
MODEL_BOUND = 2 * 2.0 ** -4
MODEL_LIMIT = 0.01       # about three times the largest H100 value (0.0026-0.0033)
# (d, H, n): the model head dims at their sequence lengths; every head dim the ABI accepts at a ragged n = 190 (d <= 32:
# the NO = 32 kernel; d = 16, 24: head columns padded to 32); and one key (n = 1) and either side of the 64-key tile
# and the 128-row block at d = 64 and 88
SHAPES = ([(d, H, n) for d, H in ((64, 16), (88, 16), (128, 25)) for n in (257, 417, 1025, 2049)]
          + [(d, 4, 190) for d in range(16, 129, 8)] + [(d, 4, n) for d in (64, 88) for n in (1, 63, 64, 65, 129)])


def _qkv(B, n, H, d, seed, spread=0.0):
    """A [B*n, 3*H*d] projection buffer of N(0, 1) values, each token's row times exp(spread N(0, 1)), and its q, k, v
    column slots."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = H * d
    x = torch.randn((B * n, 3 * D), device="cuda", generator=g)
    x = x * torch.exp(spread * torch.randn((B * n, 1), device="cuda", generator=g))
    qkv = x.to(torch.bfloat16)
    return qkv, qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]


def _pow2(amax):
    """(scale, scale_inv) of the ivb_fp8_quantize_rows rule from a finite fp32 amax: 2^e, e the largest integer with
    amax 2^e <= 448, clamped to [-126, 126]; 1 for amax 0."""
    bits = amax.contiguous().view(torch.int32)
    E = ((bits >> 23) & 0xFF) - 127
    e = (8 - E - ((bits & 0x7FFFFF) > 0x600000).to(torch.int32)).clamp(-126, 126)
    e = torch.where(amax == 0, torch.zeros_like(e), e).double()
    return torch.exp2(e).float(), torch.exp2(-e).float()


def _pack_ref(q, k, v, B, n, H, d):
    dp = (d + 31) // 32 * 32
    def rows(x):
        xf = x.float().reshape(B * n, H, d)
        scale, sinv = _pow2(xf.abs().amax(-1))
        q8 = torch.zeros((B * n, H, dp), dtype=torch.uint8, device=x.device)
        q8[..., :d] = (xf * scale[..., None]).to(E4M3).view(torch.uint8)
        return q8.reshape(B * n, H * dp), sinv.reshape(B, n, H).permute(0, 2, 1)
    vf = v.float().reshape(B, n, H, d)
    vscale, vsinv = _pow2(vf.abs().amax(1))                                        # [B, H, d]
    vt = (vf * vscale[:, None]).to(E4M3).view(torch.uint8).permute(0, 2, 3, 1)    # [B, H, d, n]
    return (*rows(q), *rows(k), vt, vsinv)


def _fwd_emulated(q8, k8, sq, sk, vt8, sv, B, n, H, d, scale):
    """float64 emulation of attn_fwd_fp8's arithmetic on its dequantised operands."""
    out = torch.empty((B * n, H * d), dtype=torch.float64, device=q8.device)
    for b in range(B):
        qd, kd = (t[b * n:(b + 1) * n].float().double().reshape(n, H, -1)[..., :d].transpose(0, 1)
                  * s[b, :, :n, None].double() for t, s in ((q8, sq), (k8, sk)))
        vd = (vt8[b, :, :, :n].float().double() * sv[b, :, :, None].double()).transpose(1, 2)    # [H, n, d]
        s2 = (qd @ kd.transpose(1, 2)) * (scale * LOG2E)
        m = torch.full((H, n, 1), -math.inf, dtype=torch.float64, device=q8.device)
        l = torch.zeros_like(m)
        o = torch.zeros((H, n, d), dtype=torch.float64, device=q8.device)
        for j0 in range(0, n, 64):
            st = s2[:, :, j0:j0 + 64]
            m_new = torch.maximum(m, st.amax(-1, keepdim=True))
            alpha = torch.exp2(m - m_new)
            p = torch.exp2(st - m_new + 8)
            l = l * alpha + p.sum(-1, keepdim=True)
            o = o * alpha + p.float().to(E4M3).double() @ vd[:, j0:j0 + 64]
            m = m_new
        out[b * n:(b + 1) * n] = (o / l).transpose(0, 1).reshape(n, H * d)
    return out


@pytest.mark.parametrize("d, H, n", SHAPES)
def test_pack_bit_exact(cuda_lib, d, H, n):
    from internvideo_b200 import lowlevel as ll
    B = 2
    _, q, k, v = _qkv(B, n, H, d, seed=n + d, spread=0.5)      # per-token magnitudes (and scales) differ
    q8, k8, sq, sk, vt8, sv = ll._attn_fp8_pack(q, k, v, B, n, H, d)
    rq8, rsq, rk8, rsk, rvt, rsv = _pack_ref(q, k, v, B, n, H, d)
    n16 = (n + 15) // 16 * 16
    assert vt8.shape == (B, H, d, n16) and sq.shape == (B, H, (n + 63) // 64 * 64)
    assert torch.equal(q8.view(torch.uint8), rq8) and torch.equal(k8.view(torch.uint8), rk8)
    assert torch.equal(sq[..., :n], rsq) and torch.equal(sk[..., :n], rsk)
    assert not sq[..., n:].any() and not sk[..., n:].any()
    assert torch.equal(vt8[..., :n].view(torch.uint8), rvt) and not vt8[..., n:].view(torch.uint8).any()
    assert torch.equal(sv, rsv)
    again = ll._attn_fp8_pack(q, k, v, B, n, H, d)
    assert all(torch.equal(a.view(torch.uint8) if a.dtype == E4M3 else a, b.view(torch.uint8) if b.dtype == E4M3 else b)
               for a, b in zip(again, (q8, k8, sq, sk, vt8, sv)))
    # an Inf in one head of a q row and a -Inf in one channel of v: that group's scale is 1 and its scale_inv NaN, the
    # satfinite cast makes the Inf +-448, and every other group keeps its bits
    t, h, c, dp = n // 2, H - 1, d - 1, (d + 31) // 32 * 32
    q2, v2 = q.clone(), v.clone()
    q2[t, h * d + c], v2[n + t, h * d + c] = float("inf"), -float("inf")
    sat = lambda x: x.float().clamp(-448, 448).to(E4M3).view(torch.uint8)   # noqa: E731
    e_q8, e_vt8 = q8.view(torch.uint8).clone(), vt8.view(torch.uint8).clone()
    e_q8[t, h * dp:h * dp + d] = sat(q2[t, h * d:(h + 1) * d])
    e_vt8[1, h, c, :n] = sat(v2[n:, h * d + c])
    e_sq, e_sv = sq.clone(), sv.clone()
    e_sq[0, h, t] = e_sv[1, h, c] = float("nan")
    got = ll._attn_fp8_pack(q2, k, v2, B, n, H, d)
    for a, b in zip(got, (e_q8, k8, e_sq, sk, e_vt8, e_sv)):
        assert torch.equal(a.view(torch.uint8) if a.dtype == E4M3 else a.view(torch.int32),
                           b.view(torch.uint8) if b.dtype in (E4M3, torch.uint8) else b.view(torch.int32))


@pytest.mark.parametrize("d, H, n", SHAPES)
def test_forward_against_emulation_and_bf16(cuda_lib, d, H, n):
    from internvideo_b200 import lowlevel as ll
    B = 2
    scale = d ** -0.5
    _, q, k, v = _qkv(B, n, H, d, seed=7 * n + d)
    packed = ll._attn_fp8_pack(q, k, v, B, n, H, d)
    out = ll._attn_fwd_fp8(*packed, B, n, H, d, scale)
    torch.cuda.synchronize()
    ref = _fwd_emulated(*packed, B, n, H, d, scale)
    emu, emu_at = worst(tile_errors(out, ref, B, n, H, d))
    bf16, _ = ll.attn_fwd(q, k, v, B, n, H, d, scale, want_lse=False)
    err, where = worst(tile_errors(out, bf16.double(), B, n, H, d))
    print(f"d {d} H {H} n {n}: tile error vs emulation {emu:.2e} at {emu_at}; vs bf16 kernel {err:.4f} at {where}")
    assert emu <= EMULATION_BOUND
    assert err <= FP8_VS_BF16
    assert torch.equal(ll._attn_fwd_fp8(*packed, B, n, H, d, scale), out)


def test_forward_writes_only_its_view(cuda_lib):
    """out as a column slot of a wider NaN-filled buffer: the call writes exactly that slot."""
    from internvideo_b200 import lowlevel as ll
    B, n, H, d = 2, 417, 16, 88
    _, q, k, v = _qkv(B, n, H, d, seed=3)
    packed = ll._attn_fp8_pack(q, k, v, B, n, H, d)
    ref = ll._attn_fwd_fp8(*packed, B, n, H, d, d ** -0.5)
    buf = torch.full((B * n, 3 * H * d), float("nan"), device="cuda", dtype=torch.bfloat16)
    got = ll._attn_fwd_fp8(*packed, B, n, H, d, d ** -0.5, out=buf[:, H * d:2 * H * d])
    assert got.data_ptr() == buf[:, H * d:].data_ptr() and torch.equal(got, ref)
    assert buf[:, :H * d].isnan().all() and buf[:, 2 * H * d:].isnan().all()


def _rel(a, b):
    a = a.detach().double(); b = b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _arms(model, run, blk, x_blk, B, n, name):
    """(FP8 attention vs FP8 GEMMs with bf16 attention, FP8 GEMMs vs bf16) relative errors of run()'s output, with the
    switching rules checked on the way."""
    from internvideo_b200 import _lib
    from internvideo_b200.modules import set_fp8_inference
    with torch.no_grad():
        y_bf16 = run()
        set_fp8_inference(model)
        y_fp8 = run()
        set_fp8_inference(model, True, attention=True)
        y_att = run()
        assert torch.equal(run(), y_att)
    with pytest.raises(_lib.IvbError, match="no gradient"):
        blk.forward_stream(x_blk.clone().requires_grad_(True), B, n)
    with torch.no_grad():
        set_fp8_inference(model, True)                  # attention back to bf16: the FP8-inference bits
        assert torch.equal(run(), y_fp8)
        set_fp8_inference(model, False)                 # off: the bf16 bits
        assert torch.equal(run(), y_bf16)
    r_att, r_fp8 = _rel(y_att, y_fp8), _rel(y_fp8, y_bf16)
    print(f"{name}: FP8 attention vs bf16 attention (both FP8 GEMMs) {r_att:.4f}; FP8 GEMMs vs bf16 {r_fp8:.4f}")
    return r_att


def test_clip_l_tower(cuda_lib):
    """The cfg-3 L tower's dims (D 1024, 16 heads of 64, mlp 4, 4 frames: n = 1025) at depth 2, unmasked."""
    from internvideo_b200.clip_modules import InternVideo2
    torch.manual_seed(0)
    tower = InternVideo2(embed_dim=1024, num_heads=16, mlp_ratio=4, depth=2, num_frames=4, attn_pool_num_heads=16,
                         clip_embed_dim=768, init_values=0.1, drop_path_rate=0.0, use_flash_attn=False,
                         use_fused_rmsnorm=False, use_fused_mlp=False).bfloat16().cuda().eval()
    B = 2
    x = torch.randn((B, 3, 4, 224, 224), device="cuda").to(torch.bfloat16)
    n = 1025
    x_blk = torch.randn((B * n, 1024), device="cuda")
    r = _arms(tower, lambda: tower(x), tower.blocks[0], x_blk, B, n, "L tower, n 1025")
    assert r <= MODEL_BOUND and r <= MODEL_LIMIT


def test_stage2_tower_unmasked(cuda_lib):
    """The 1B stage-2 tower's dims (D 1408, 16 heads of 88, 8 frames: n = 2049) at depth 2, every token visible."""
    from internvideo_b200.stage2 import PretrainInternVideo2
    torch.manual_seed(1)
    tower = PretrainInternVideo2(embed_dim=1408, num_heads=16, mlp_ratio=48 / 11, depth=2, num_frames=8,
                                 clip_embed_dim=768, init_values=0.1, drop_path_rate=0.0, use_flash_attn=False,
                                 use_fused_rmsnorm=False, use_fused_mlp=False, clip_teacher_embed_dim=1408,
                                 clip_teacher_final_dim=768, clip_return_layer=1).bfloat16().cuda().eval()
    B, n = 2, 2049
    x = torch.randn((B, 3, 8, 224, 224), device="cuda").to(torch.bfloat16)
    x_blk = torch.randn((B * n, 1408), device="cuda")
    r = _arms(tower, lambda: tower(x, x_vis_only=True), tower.blocks[0], x_blk, B, n, "stage-2 tower, n 2049")
    assert r <= MODEL_BOUND and r <= MODEL_LIMIT


def test_videomae_teacher_token_axis(cuda_lib):
    """The VideoMAEv2 teacher's dims (D 1408, 16 heads of 88, n = 2048) at depth 2 with token-axis attention; with
    head-axis attention FP8 attention does not apply and the outputs keep their bits."""
    from internvideo_b200.modules import set_fp8_inference
    from internvideo_b200.teachers import VisionTransformer
    torch.manual_seed(2)
    mk = partial(VisionTransformer, img_size=224, patch_size=14, embed_dim=1408, depth=2, num_heads=16,
                 mlp_ratio=48 / 11, qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), all_frames=16,
                 tubelet_size=2, init_values=0.1, mae_return_layer=2)
    teacher = mk(head_axis_attention=False).bfloat16().cuda().eval()
    B, n = 2, 2048
    x = torch.randn((B, 3, 16, 224, 224), device="cuda").to(torch.bfloat16)
    x_blk = torch.randn((B * n, 1408), device="cuda")
    r = _arms(teacher, lambda: teacher(x), teacher.blocks[0], x_blk, B, n, "VideoMAEv2 teacher, token axis, n 2048")
    assert r <= MODEL_BOUND and r <= MODEL_LIMIT
    teacher.head_axis_attention = True
    set_fp8_inference(teacher)
    y = teacher(x)
    set_fp8_inference(teacher, True, attention=True)
    assert torch.equal(teacher(x), y)
    set_fp8_inference(teacher, False)
