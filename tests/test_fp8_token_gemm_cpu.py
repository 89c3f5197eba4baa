"""tests/fp8_exact.py on the CPU: the exactness bounds hold at every shape and value range
tests/test_fp8_token_gemm_gpu.py uses, the builders' operands dequantise to exactly v, and the weight-gradient
reference equals an int64 restatement."""
import pytest
import torch

import fp8_exact as fx


def test_vector_scale_bounds_at_every_shape():
    cases = [(fx.TAIL_VMAX, K) for K in fx.TAIL_K] + [(fx.PLAN_VMAX, fx.PLAN_K)]
    cases += [(fx.STEP_VMAX, K) for t in fx.TOWERS for _, _, K, _ in fx.step_gemms(t)]
    for vmax, K in cases:
        partial, result = fx.vec_bounds(vmax, K)
        assert partial < fx.PARTIAL_LIMIT, (vmax, K)
        # + an epilogue input on the 2^-8 grid below 16 (bias, old out0), or a bf16 factor (saved GELU'): exact in fp32
        assert (result + 16) * 2 ** fx.GRID < fx.RESULT_LIMIT, (vmax, K)


def test_block_scale_bounds_at_every_shape():
    for K in fx.WGRAD_K + (fx.WGRAD_CFG2_K,):
        partial, result = fx.block_bounds(fx.WGRAD_VMAX, K)
        assert partial < fx.PARTIAL_LIMIT and result < 2 ** 18, K
        # FLAG_ACCUM: result + old (on the 2^-8 grid, |old| < 1) is exact in float64, so its rounding to fp32 is the
        # one rounding of the kernel's fp32 add of the exact accumulator and old
        assert (result + 1) * 2 ** fx.GRID < 2 ** 53, K


def test_accum_reference_is_the_fp32_add():
    """The weight-gradient FLAG_ACCUM reference, fp32(float64(ref + old)), is the fp32 add of the two exact fp32
    operands, also where that sum is not exact in fp32 (|ref| past 2^16)."""
    g = torch.Generator().manual_seed(0)
    ref = torch.randint(-213504, 213505, (100000,), generator=g).double()
    old = fx.grid_values((100000,), 1, device="cpu")
    want = (ref + old.double()).float()
    assert torch.equal(want, ref.float() + old)
    assert not torch.equal(want.double(), ref + old.double())      # inexact sums do occur


def test_step_gemms_match_the_cfg2_step():
    """cfg-2's eight GEMMs are those of tests/test_gemm_fp8_gpu.STEP (M = 13 344)."""
    assert fx.TOWERS["cfg2"][0] == 13344
    assert [(n, N, K) for n, N, K, _ in fx.step_gemms("cfg2")] == [
        ("qkv", 4224, 1408), ("proj", 1408, 1408), ("fc1", 6144, 1408), ("fc2", 1408, 6144),
        ("dh", 6144, 1408), ("dn2", 1408, 6144), ("da", 1408, 1408), ("dn1", 1408, 4224)]


def _normal_e4m3(q):
    """Every nonzero value is a normal E4M3 number (2^-6 <= |x| <= 448)."""
    x = q.float().abs()
    nz = x[x != 0]
    return bool(((nz >= 2.0 ** -6) & (nz <= 448)).all())


@pytest.mark.parametrize("vmax", [fx.TAIL_VMAX, fx.STEP_VMAX])
@pytest.mark.parametrize("rows,K", [(333, 40), (136, 200), (2080, 256), (77, 1408)])
def test_vec_operand_dequantises_to_v(rows, K, vmax):
    pitch = (K + 15) // 16 * 16 + 16
    q, sinv, v = fx.vec_operand(rows, K, pitch, rows + K, vmax, device="cpu")
    assert q.shape == (rows, K) and q.stride(0) == pitch and sinv.shape == (rows,)
    assert torch.equal(fx.deq_vec(q, sinv), v.double())
    assert int(v.abs().max()) == vmax and _normal_e4m3(q)
    e = -torch.log2(sinv)
    assert torch.equal(e, e.round()) and int(e.min()) >= fx.EXP_LO and int(e.max()) <= fx.EXP_HI
    assert len(torch.unique(e)) > 6                     # the rows do carry different scales
    pad = q.view(torch.uint8).as_strided((rows, pitch), (pitch, 1))[:, K:]
    assert bool((pad == fx.NAN8).all())


@pytest.mark.parametrize("rows,K", [(200, 100), (328, 128), (136, 417), (1416, 1251)])
def test_block_operand_dequantises_to_v(rows, K):
    pitch = (K + 15) // 16 * 16 + 16
    q, sinv, v = fx.block_operand(rows, K, pitch, rows * K, fx.WGRAD_VMAX, device="cpu")
    nkb = (K + fx.BK - 1) // fx.BK
    assert sinv.shape == (nkb, rows) and sinv.is_contiguous()
    assert torch.equal(fx.deq_block(q, sinv), v.double()) and _normal_e4m3(q)
    e = -torch.log2(sinv)
    assert torch.equal(e, e.round()) and int(e.min()) >= fx.EXP_LO and int(e.max()) <= fx.EXP_HI
    if nkb > 1:   # a row's exponent changes from k-block to k-block
        assert bool((e[0] != e[1]).any())


@pytest.mark.parametrize("M,N", fx.WGRAD_MN)
@pytest.mark.parametrize("K", [k for k in fx.WGRAD_K if k <= 1251])
def test_wgrad_ref_equals_int64(M, N, K):
    g = torch.Generator().manual_seed(M + K)
    va = torch.randint(-4, 5, (M, K), generator=g).float()
    vb = torch.randint(-4, 5, (N, K), generator=g).float()
    nkb = (K + fx.BK - 1) // fx.BK
    for blocks in (None, list(range(1, nkb, 2)), [nkb - 1], []):
        ref = fx.wgrad_ref(va, vb, blocks)
        assert torch.equal(ref, fx.wgrad_ref_int(va, vb, blocks).double()), blocks
    assert float(fx.wgrad_ref(va, vb).abs().max()) <= fx.block_bounds(4, K)[1]


def test_k_plan_layout():
    kp = fx.k_plan([4, 1, 9], 1251, device="cpu")
    assert kp.dtype == torch.int32 and kp.tolist() == [1, 4, 9, 0, 2, 3, 5, 6, 7, 8, 3]
    assert fx.k_plan([], 100, device="cpu").tolist() == [0, 0]


def test_grid_values_are_exact_in_bf16():
    x = fx.grid_values((4096,), 3, device="cpu", limit=1.0)
    assert torch.equal(x.to(torch.bfloat16).float(), x) and float(x.abs().max()) < 1.0
    assert torch.equal(x * 2 ** fx.GRID, (x * 2 ** fx.GRID).round())
