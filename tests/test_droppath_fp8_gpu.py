"""DropPath skipping in per-token FP8 and in attention, on the H100.  Each planned call against the same call without a
plan: ivb_gemm_fp8_plan's live rows equal ivb_gemm_fp8's and its dead tiles hold the dead-tile table (ivb200.h);
ivb_attn_fwd_plan / ivb_attn_bwd_plan give the kept clips ivb_attn_fwd / ivb_attn_bwd's bits and the dropped clips
zeros.  Equality is torch.equal: the same values, where a zero may come out as +0 instead of -0.  The training block
and the model step with the skipping against without: test_fp8_modes_gpu.py."""
import numpy as np
import pytest
import torch

import droppath_ref as ref
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu

B = 32
DRAWS = {
    "none_dropped": np.ones(B, bool),
    "all_dropped": np.zeros(B, bool),
    "random": np.random.default_rng(3).random(B) >= 0.25,
    "alternating": np.arange(B) % 2 == 0,
}


def _rows(keep, n):
    return torch.from_numpy(ref.clip_rows(keep, n)).cuda()


def _m_plan(rs):
    return ops._branch_plans(ops.droppath_plan(rs[None].contiguous())[0], rs.numel(), ops.FP8_TOKEN)[0]


def _dead_rows(keep, n):
    order, live, _ = ref.plan(ref.clip_rows(keep, n))
    dead = torch.zeros(keep.size * n, dtype=torch.bool, device="cuda")
    for t in order[live:]:
        dead[128 * t:128 * t + 128] = True
    return dead


def _case(epi, Mr, N, K, g):
    """Per-token FP8 operands (row-scaled A, per-channel B) and the epilogue arguments of one GEMM."""
    a = torch.randn((Mr, K), generator=g, device="cuda").to(torch.bfloat16)
    w = (0.1 * torch.randn((N, K), generator=g, device="cuda")).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device="cuda").to(torch.bfloat16)
    ops_ = (*ll.fp8_quantize_rows(a), *ll.fp8_quantize_rows(w))
    if epi == "bf16":
        return ops_, dict(bias=bias), ["out0"]
    if epi == "bias_gelu_save":
        return ops_, dict(epi=ll.EPI_BIAS_GELU, bias=bias, flags=ll.FLAG_GELU_SAVE_GRAD, out1=True), ["out0", "out1"]
    if epi == "resid":
        gamma = (1e-2 * torch.randn(N, generator=g, device="cuda")).to(torch.bfloat16)
        aux = torch.randn((Mr, N), generator=g, device="cuda")
        return ops_, dict(epi=ll.EPI_RESID, bias=bias, gamma=gamma, aux=aux, out1=True), ["out0", "out1"]
    aux = torch.rand((Mr, N), generator=g, device="cuda").to(torch.bfloat16)
    return ops_, dict(epi=ll.EPI_GELU_BWD, flags=ll.FLAG_GELU_SAVE_GRAD, aux=aux), ["out0"]


def _check_m_plan(epi, n, N, K, flags, tile_n, draws, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Mr = B * n
    for draw in draws:
        keep = DRAWS[draw]
        rs = _rows(keep, n)
        (qa, sa, qb, sb), kw, outs = _case(epi, Mr, N, K, g)
        kw["flags"] = kw.get("flags", 0) | flags
        if kw.get("epi") == ll.EPI_RESID:
            kw["rowscale"] = rs
        res = []
        for plan, tn in ((None, tile_n), (_m_plan(rs), 128 if tile_n == 192 else tile_n)):
            o1 = torch.full((Mr, N), float("nan"), device="cuda").to(torch.bfloat16) if kw.get("out1") else None
            o0 = ll._gemm_fp8_plan(qa, sa, qb, sb, plan, tile_n=tn, **{**kw, "out1": o1})
            res.append({"out0": o0, "out1": o1})
        dead = _dead_rows(keep, n)
        for o in outs:
            full, planned = res[0][o], res[1][o]
            assert torch.equal(planned[~dead], full[~dead]), (draw, o)
            want = kw["aux"][dead] if (kw.get("epi") == ll.EPI_RESID and o == "out0") else torch.zeros_like(planned[dead])
            assert torch.equal(planned[dead], want), (draw, o)


# the eight block GEMMs of cfg-2 (n = 417: M = 13 344), each with the epilogue the block gives it
CFG2 = [("qkv", 4224, 1408, "bf16"), ("proj", 1408, 1408, "resid"), ("fc1", 6144, 1408, "bias_gelu_save"),
        ("fc2", 1408, 6144, "resid"), ("dh", 6144, 1408, "gelu_bwd_save"), ("dn2", 1408, 6144, "bf16"),
        ("da", 1408, 1408, "bf16"), ("dn1", 1408, 4224, "bf16")]


@pytest.mark.parametrize("name, N, K, epi", CFG2, ids=[c[0] for c in CFG2])
def test_fp8_m_plan_cfg2_shapes(cuda_lib, name, N, K, epi):
    """The library's default kernel at the step's shapes, with a random, an all-live and an all-dead draw."""
    _check_m_plan(epi, 417, N, K, 0, 0, ["random", "none_dropped", "all_dropped"], seed=1)


EPILOGUES = ["bf16", "resid", "bias_gelu_save", "gelu_bwd_save"]
# ping-pong; the cooperative kernel at the width the library picks, at 128, and forced to 192 without a plan (a plan
# runs it at 128)
FORMS = [(ll.FLAG_PINGPONG, 0), (ll.FLAG_1CTA, 0), (ll.FLAG_1CTA, 128), (ll.FLAG_1CTA, 192)]


@pytest.mark.parametrize("form", FORMS, ids=["pingpong", "coop", "coop128", "coop192"])
@pytest.mark.parametrize("epi", EPILOGUES)
def test_fp8_m_plan_forms_and_tails(cuda_lib, epi, form):
    """Both kernel forms at a row tail (32 clips of 65 rows: M = 2080, 32 rows into the last tile) and a column tail
    (N = 1416), with every draw."""
    _check_m_plan(epi, 65, 1416, 256, form[0], form[1], list(DRAWS), seed=7)


# ---- attention
@pytest.mark.parametrize("n", [417, 130])
@pytest.mark.parametrize("d", [64, 88, 128])
def test_attn_plan(cuda_lib, d, n):
    Bc, H = 6, 3
    D = H * d
    g = torch.Generator(device="cuda").manual_seed(d + n)
    qkv = torch.randn((Bc * n, 3 * D), generator=g, device="cuda").to(torch.bfloat16)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    dout = torch.randn((Bc * n, D), generator=g, device="cuda").to(torch.bfloat16)
    scale = d ** -0.5
    for keep in (np.ones(Bc, bool), np.array([1, 0, 1, 1, 0, 0], bool), np.zeros(Bc, bool)):
        res = []
        for rs in (None, _rows(keep, n)):
            out, lse = ll.attn_fwd(q, k, v, Bc, n, H, d, scale, rowscale=rs)
            dqkv = torch.full((Bc * n, 3 * D), float("nan"), device="cuda").to(torch.bfloat16)
            ll.attn_bwd(q, k, v, out, dout, lse, Bc, n, H, d, scale, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:],
                        rowscale=rs)
            res.append((out.reshape(Bc, n, D), lse, dqkv.reshape(Bc, n, 3 * D)))
        kept = torch.from_numpy(keep).cuda()
        (o0, l0, g0), (o1, l1, g1) = res
        assert torch.equal(o1[kept], o0[kept]) and torch.equal(l1[kept], l0[kept]) and torch.equal(g1[kept], g0[kept])
        assert torch.all(o1[~kept] == 0) and torch.all(g1[~kept] == 0)
        assert torch.isfinite(l1[~kept]).all()
