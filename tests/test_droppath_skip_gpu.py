"""DropPath plans on the H100: ivb_droppath_plan against the restatement (tests/droppath_ref.py), and every planned call
against the same call without a plan.  Live rows are equal, dead rows hold what the plan's epilogue table gives them
(ivb200.h), weight gradients over the listed k-blocks equal the full sums, and a training block (BlockFn, cfg-2 dims)
gives the same output, input gradient and parameter gradients.  Equality is torch.equal: the same values, where a zero
may come out as +0 instead of -0."""
import numpy as np
import pytest
import torch

import droppath_ref as ref
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import modules as M
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu

B = 32
DRAWS = {
    "none_dropped": np.ones(B, bool),
    "all_dropped": np.zeros(B, bool),
    "single_clip": np.arange(B) == 5,
    "alternating": np.arange(B) % 2 == 0,
}


def _rows(keep, n):
    return torch.from_numpy(ref.clip_rows(keep, n)).cuda()


def _plans(rs):
    """(M plan, K plan) of one branch's factors rs [M]."""
    return ops._branch_plans(ops.droppath_plan(rs[None].contiguous())[0], rs.numel(), ops.BF16)


@pytest.mark.parametrize("n", [417, 65, 256])
def test_plan_kernel_matches_restatement(cuda_lib, n):
    rs = torch.stack([_rows(keep, n) for keep in DRAWS.values()])
    got = ops.droppath_plan(rs).cpu().numpy()
    for i, keep in enumerate(DRAWS.values()):
        want = ref.flat(*ref.plan(ref.clip_rows(keep, n)), B * n)
        written = want != -1
        assert np.array_equal(got[i][written], want[written]), list(DRAWS)[i]


GEMM_ROWS_N = 65                      # 32 clips of 65 rows: clips shorter than a 128-row tile
EPILOGUES = ["bf16", "f32", "bias_gelu_save", "bias_gelu_h", "resid", "gelu_bwd_save"]
FORMS = [(ll.FLAG_PINGPONG, 0), (ll.FLAG_1CTA, 128), (ll.FLAG_1CTA, 176), (ll.FLAG_1CTA, 192), (ll.FLAG_1CTA, 256)]


def _gemm_case(name, Mr, N, K, g):
    a = torch.randn((Mr, K), generator=g, device="cuda").to(torch.bfloat16)
    w = (0.1 * torch.randn((N, K), generator=g, device="cuda")).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device="cuda").to(torch.bfloat16)
    if name == "bf16":
        return a, w, dict(bias=bias), ["out0"]
    if name == "f32":
        return a, w, dict(epi=ll.EPI_F32, bias=bias), ["out0"]
    if name.startswith("bias_gelu"):
        flags = ll.FLAG_GELU_SAVE_GRAD if name.endswith("save") else 0
        return a, w, dict(epi=ll.EPI_BIAS_GELU, bias=bias, flags=flags, out1=True), ["out0", "out1"]
    if name == "resid":
        gamma = (1e-2 * torch.randn(N, generator=g, device="cuda")).to(torch.bfloat16)
        aux = torch.randn((Mr, N), generator=g, device="cuda")
        return a, w, dict(epi=ll.EPI_RESID, bias=bias, gamma=gamma, aux=aux, out1=True), ["out0", "out1"]
    aux = torch.rand((Mr, N), generator=g, device="cuda").to(torch.bfloat16)
    return a, w, dict(epi=ll.EPI_GELU_BWD, flags=ll.FLAG_GELU_SAVE_GRAD, aux=aux), ["out0"]


@pytest.mark.parametrize("form", FORMS, ids=["pingpong", "coop128", "coop176", "coop192", "coop256"])
@pytest.mark.parametrize("epi", EPILOGUES)
def test_m_plan_epilogues(cuda_lib, epi, form):
    """Live rows as without a plan; dead rows: EPI_RESID out0 = aux, out1 = 0; every other output 0."""
    g = torch.Generator(device="cuda").manual_seed(7)
    flags, tile_n = form
    n, N, K = GEMM_ROWS_N, 1408, 256
    Mr = B * n
    for draw, keep in DRAWS.items():
        rs = _rows(keep, n)
        a, w, kw, outs = _gemm_case(epi, Mr, N, K, g)
        kw["flags"] = kw.get("flags", 0) | flags
        if kw.get("epi") == ll.EPI_RESID:
            kw["rowscale"] = rs
        res = []
        for plan in (None, _plans(rs)[0]):
            o1 = torch.full((Mr, N), float("nan"), device="cuda").to(torch.bfloat16) if kw.get("out1") else None
            o0 = ll.gemm(a, w, tile_n=tile_n, m_plan=plan, **{**kw, "out1": o1})
            res.append({"out0": o0, "out1": o1})
        order, live, _ = ref.plan(ref.clip_rows(keep, n))
        dead = torch.zeros(Mr, dtype=torch.bool, device="cuda")
        for t in order[live:]:
            dead[128 * t:128 * t + 128] = True
        for o in outs:
            full, planned = res[0][o], res[1][o]
            assert torch.equal(planned[~dead], full[~dead]), (draw, o)
            want = kw["aux"][dead] if (kw.get("epi") == ll.EPI_RESID and o == "out0") else torch.zeros_like(planned[dead])
            assert torch.equal(planned[dead], want), (draw, o)


@pytest.mark.parametrize("accum", [False, True])
@pytest.mark.parametrize("form", [ll.FLAG_PINGPONG, ll.FLAG_1CTA], ids=["pingpong", "coop"])
def test_k_plan_wgrad(cuda_lib, form, accum):
    """dW = dy^T x over the listed k-blocks equals the full sum when dy is zero on the dropped rows."""
    g = torch.Generator(device="cuda").manual_seed(11)
    n, N1, N2 = 417, 1408, 512
    T = B * n
    x = torch.randn((T, N2), generator=g, device="cuda").to(torch.bfloat16)
    for draw, keep in DRAWS.items():
        rs = _rows(keep, n)
        dy = (torch.randn((T, N1), generator=g, device="cuda") * rs[:, None]).to(torch.bfloat16)
        init = torch.randn((N1, N2), generator=g, device="cuda")
        res = []
        for plan in (None, _plans(rs)[1]):
            out = init.clone() if accum else None
            res.append(ll.gemm(dy, x, a_t=True, b_t=True, epi=ll.EPI_F32, out0=out, flags=form | (ll.FLAG_ACCUM if accum else 0),
                               k_plan=plan))
        assert torch.equal(res[1], res[0]), draw


def _block_run(keep, plans_on, D=1408, H=16, n=417, seed=3):
    torch.manual_seed(seed)
    blk = M.Block(D, H, 4.3637, init_values=1e-5, qk_normalization=True, use_fused_mlp=True,
                  drop_path=0.1).bfloat16().cuda()
    x = torch.randn(B * n, D, device="cuda").requires_grad_(True)
    rs1, rs2 = _rows(keep, n), _rows(np.roll(keep, 1), n)
    plans = tuple(ops.droppath_plan(torch.stack([rs1, rs2]))) if plans_on else None
    y = blk.forward_stream(x, B, n, rowscale=(rs1, rs2), plans=plans)
    y.backward(torch.randn(y.shape, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda"))
    grads = {nm: p.grad.clone() for nm, p in blk.named_parameters()}
    return y.detach(), x.grad.clone(), grads


@pytest.mark.parametrize("draw", list(DRAWS))
def test_block_planned_equals_unplanned(cuda_lib, draw):
    """A training block at cfg-2 dims (D = 1408, 16 heads, n = 417, 32 clips): x2, dx0 and every parameter gradient
    are the same with the plans as without."""
    y0, dx0, g0 = _block_run(DRAWS[draw], False)
    y1, dx1, g1 = _block_run(DRAWS[draw], True)
    assert torch.equal(y1, y0)
    assert torch.equal(dx1, dx0)
    for nm in g0:
        assert torch.equal(g1[nm], g0[nm]), nm
