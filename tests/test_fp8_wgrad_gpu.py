"""FP8 weight gradients (modules.set_fp8(model, scaling="token", wgrad=True)) on the H100 (gpu).

- ivb_fp8_quantize_blocks_t: element by element and scale by scale against a float64 restatement of the rule, with a
  partial last block, an all-zero block, a zero column, blocks holding an Inf or a NaN (their E4M3 bytes included) and
  sizes that are not multiples of 128;
  two calls give the same bytes; the _plan form equals the plain cast of x with the dropped rows zeroed.
- ivb_gemm_fp8_wgrad: accumulation ratio against float64 at the four cfg-2 weight-gradient shapes and at tails; the
  four epilogue forms; a K plan gives the unplanned call's bits when the plan's dead rows of dy are zero.
The block and the model in this mode: test_fp8_modes_gpu.py.
"""
import numpy as np
import pytest
import torch

import droppath_ref as ref
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu
bf16, f32, e4m3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
NAN8 = 0x7f    # an E4M3 NaN byte


def _pad16(n):
    return (n + 15) // 16 * 16


# ------------------------------------------------------------------------------------------------ the cast
def _blocks_reference(x):
    """float64 restatement: per 128-row block b and column c, scale 2^e with e the largest integer such that
    amax_bc * 2^e <= 448 (e in [-126, 126]; 1 for a zero block column), q_t[c, 128b + i] = RNE_e4m3(x[128b + i, c] *
    scale), scale_inv NaN for a block column holding an Inf or NaN.  Returns (q_t, scale_inv [nb, C], finite [M, C])."""
    Mx, C = x.shape
    nb = (Mx + 127) // 128
    x64 = torch.zeros((nb * 128, C), device=x.device, dtype=torch.float64)
    x64[:Mx] = x.double()
    amax = x64.reshape(nb, 128, C).abs().amax(1)
    e = torch.floor(torch.log2(448.0 / amax.clamp_min(1e-300)))
    e = torch.where(amax * torch.exp2(e + 1) <= 448.0, e + 1, e)
    e = torch.where(amax * torch.exp2(e) > 448.0, e - 1, e)
    e = torch.where(amax == 0, torch.zeros_like(e), e.clamp(-126, 126))
    finite = torch.isfinite(amax)
    e = torch.where(finite, e, torch.zeros_like(e))
    scale = torch.exp2(e)
    rows = lambda t: t.repeat_interleave(128, 0)[:Mx]   # noqa: E731
    q = torch.where(rows(finite), x64[:Mx] * rows(scale), torch.zeros_like(x64[:Mx]))
    q_t = q.float().t().contiguous().to(e4m3)
    sinv = torch.where(finite, 1.0 / scale, torch.full_like(scale, float("nan")))
    return q_t, sinv, rows(finite).t()


@pytest.mark.parametrize("Mx, C", [(1251, 1408), (417, 200), (128, 64), (129, 8), (300, 4224)])
def test_quantize_blocks_t_against_float64(cuda_lib, Mx, C):
    g = torch.Generator(device="cuda").manual_seed(Mx * 31 + C)
    ldx = C + 24
    xb = torch.randn((Mx, ldx), device="cuda", generator=g) * 0.02
    xb[:, : C // 2] *= torch.exp2(torch.randint(-20, 20, (C // 2,), device="cuda", generator=g).float())
    xb *= torch.exp2(torch.randint(-6, 6, (Mx, 1), device="cuda", generator=g).float())     # per-token magnitudes
    xb = xb.to(bf16)
    x = xb[:, :C]
    if Mx > 256:
        x[128:256] = 0                                    # an all-zero block
    x[:, 3] = 0                                           # a zero column in every block
    x[Mx - 1, 5] = float("inf")                           # an Inf in the last (partial) block
    x[0, 6] = float("nan")                                # a NaN in the first block
    ldt = _pad16(Mx) + 16
    nb = (Mx + 127) // 128
    runs = []
    for _ in range(2):
        q_t = torch.full((C, ldt), NAN8, device="cuda", dtype=torch.uint8)
        sinv = torch.full((nb * C + 1,), float("nan"), device="cuda", dtype=f32)
        ll._call("fp8_quantize_blocks_t", x, ldx, Mx, C, q_t, ldt, sinv)
        runs.append((q_t, sinv))
    torch.cuda.synchronize()
    (q_t, sinv), (q_t2, sinv2) = runs
    assert torch.equal(q_t, q_t2) and torch.equal(sinv.view(torch.int32), sinv2.view(torch.int32))
    q_ref, s_ref, fin = _blocks_reference(x)
    s = sinv[:nb * C].reshape(nb, C)
    sfin = torch.isfinite(s_ref)
    assert not bool(sfin[nb - 1, 5]) and bool(torch.isnan(s[nb - 1, 5]))
    assert torch.equal(s[sfin].double(), s_ref[sfin]) and bool((s[:, 3] == 1.0).all())
    if Mx > 256:
        assert bool((s[1] == 1.0).all()) and bool((q_t[:, 128:256] == 0).all())
    assert torch.equal(q_t[:, :Mx][fin], q_ref.view(torch.uint8)[fin])
    assert (q_t[:, Mx:] == NAN8).all() and torch.isnan(sinv[nb * C])
    # the non-finite block columns: scale 1 and a satfinite cast, so an Inf becomes +-448 and a NaN stays NaN
    for blk, c in (~sfin).nonzero().tolist():
        col = x[128 * blk:128 * blk + 128, c].float()
        got, nan = q_t[c, 128 * blk:128 * blk + col.numel()], torch.isnan(col)
        assert torch.equal(got[~nan], col.clamp(-448, 448).to(e4m3).view(torch.uint8)[~nan])
        assert bool(((got[nan] & 0x7f) == 0x7f).all())
    # the lowlevel form gives the same bits; the _plan form casts the rows whose factor is 0 as zeros
    q3, s3 = ll._fp8_quantize_blocks_t(x)
    assert torch.equal(q3.view(torch.uint8), q_t[:, :Mx]) and torch.equal(s3.view(torch.int32), s.view(torch.int32))
    rs = (torch.rand(Mx, device="cuda", generator=g) > 0.3).float() * 1.25
    q4, s4 = ll._fp8_quantize_blocks_t(x, rowscale=rs)
    q5, s5 = ll._fp8_quantize_blocks_t(torch.where((rs != 0)[:, None], x, torch.zeros_like(x)))
    assert torch.equal(q4.view(torch.uint8), q5.view(torch.uint8)) and torch.equal(s4.view(torch.int32),
                                                                                    s5.view(torch.int32))


# ------------------------------------------------------------------------------------------------ the GEMM
def _operands(Mo, N, K, seed):
    """dy [K, Mo] with per-token magnitudes spread over 2^-8 .. 2^8 (gradients), act [K, N] (activations)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn((K, Mo), device="cuda", generator=g)
    dy *= torch.exp2(torch.randint(-8, 9, (K, 1), device="cuda", generator=g).float())
    act = torch.randn((K, N), device="cuda", generator=g) * (1 + torch.rand((1, N), device="cuda", generator=g))
    return dy.to(bf16), act.to(bf16)


def _deq(q_t, sinv):
    """float64 [rows, K] of a block-scaled transposed copy."""
    K = q_t.shape[1]
    return q_t.double() * sinv.double().t().repeat_interleave(128, 1)[:, :K]


# The four weight gradients of cfg-2 (B = 32 clips of 417 tokens: K = 13 344) and tails: K = 417 * 3, M and N not
# multiples of 128
CFG2 = [("qkv", 4224, 1408, 13344), ("proj", 1408, 1408, 13344), ("fc1", 6144, 1408, 13344),
        ("fc2", 1408, 6144, 13344), ("tail", 200, 328, 1251), ("tail_k", 1416, 136, 417)]


@pytest.mark.parametrize("name, Mo, N, K", CFG2, ids=[c[0] for c in CFG2])
def test_wgrad_accumulation_ratio(cuda_lib, name, Mo, N, K):
    """||C_kernel - C64(deq)|| / ||C64(deq) - C64(bf16)|| <= 0.25: the kernel's own accumulation error against the
    error the FP8 operands already carry (DESIGN.md 4.1)."""
    dy, act = _operands(Mo, N, K, seed=Mo + N + K)
    (qa, sa), (qb, sb) = ll._fp8_quantize_blocks_t(dy), ll._fp8_quantize_blocks_t(act)
    c = ll._gemm_fp8_wgrad(qa, sa, qb, sb, epi=ll.EPI_F32)
    c64_deq = _deq(qa, sa) @ _deq(qb, sb).t()
    c64_bf16 = dy.double().t() @ act.double()
    ratio = float((c.double() - c64_deq).norm() / (c64_deq - c64_bf16).norm())
    print(f"{name} {Mo}x{N}x{K}: accumulation ratio {ratio:.4f}, "
          f"fp8 error {float((c64_deq - c64_bf16).norm() / c64_bf16.norm()):.4f}")
    assert ratio <= 0.25, ratio


def test_wgrad_epilogues(cuda_lib):
    """EPI_BF16 is EPI_F32 rounded; IVB_FLAG_ACCUM adds the old out0 in fp32 (before the bf16 rounding)."""
    Mo, N, K = 200, 328, 1251
    dy, act = _operands(Mo, N, K, seed=5)
    (qa, sa), (qb, sb) = ll._fp8_quantize_blocks_t(dy), ll._fp8_quantize_blocks_t(act)
    g = torch.Generator(device="cuda").manual_seed(6)
    c32 = ll._gemm_fp8_wgrad(qa, sa, qb, sb, epi=ll.EPI_F32)
    c16 = ll._gemm_fp8_wgrad(qa, sa, qb, sb, epi=ll.EPI_BF16)
    assert torch.equal(c16, c32.to(bf16))
    old32 = torch.randn((Mo, N + 8), device="cuda", generator=g)[:, :N]          # a padded pitch
    o32 = old32.clone()
    ll._gemm_fp8_wgrad(qa, sa, qb, sb, epi=ll.EPI_F32, flags=ll.FLAG_ACCUM, out0=o32)
    assert torch.equal(o32, old32 + c32)
    old16 = torch.randn((Mo, N), device="cuda", generator=g).to(bf16)
    o16 = old16.clone()
    ll._gemm_fp8_wgrad(qa, sa, qb, sb, epi=ll.EPI_BF16, flags=ll.FLAG_ACCUM, out0=o16)
    assert torch.equal(o16, (old16.float() + c32).to(bf16))


KEEPS = {"random": np.random.default_rng(3).random(32) >= 0.25, "alternating": np.arange(32) % 2 == 0,
         "none_dropped": np.ones(32, bool), "all_dropped": np.zeros(32, bool)}


@pytest.mark.parametrize("n, Mo, N", [(417, 1408, 1408), (65, 200, 328)])
@pytest.mark.parametrize("draw", list(KEEPS))
def test_wgrad_k_plan(cuda_lib, draw, n, Mo, N):
    """With the plan's dead rows of dy zeroed, a planned call gives the unplanned call's bits, in every epilogue form;
    an empty plan gives 0, or leaves out0 as it was under ACCUM."""
    keep = KEEPS[draw]
    rs = torch.from_numpy(ref.clip_rows(keep, n)).cuda()
    K = rs.numel()
    dy, act = _operands(Mo, N, K, seed=n + Mo)
    dy = dy * (rs != 0)[:, None].to(bf16)                 # layerscale_bwd's zero rows
    plan = ops.droppath_plan(rs[None].contiguous())[0]
    _, k_plan = ops._branch_plans(plan, K, ops.FP8_TOKEN_WGRAD)
    (qa, sa), (qb, sb) = ll._fp8_quantize_blocks_t(dy), ll._fp8_quantize_blocks_t(act)
    g = torch.Generator(device="cuda").manual_seed(9)
    for epi, dt in ((ll.EPI_F32, f32), (ll.EPI_BF16, bf16)):
        for flags in (0, ll.FLAG_ACCUM):
            old = torch.randn((Mo, N), device="cuda", generator=g).to(dt)
            res = []
            for kp in (None, k_plan):
                out = old.clone()
                ll._gemm_fp8_wgrad(qa, sa, qb, sb, epi=epi, flags=flags, out0=out, k_plan=kp)
                res.append(out)
            assert torch.equal(res[1], res[0]), (epi, flags)
            if draw == "all_dropped":
                assert torch.equal(res[1], old if flags else torch.zeros_like(old)), (epi, flags)
