"""Operands whose per-token FP8 GEMMs are exact, the shapes the exact tests run at, and their float64 references.

Every E4M3 operand element is v * 2^e: v an integer in [-vmax, vmax], e in [EXP_LO, EXP_HI] (so every value is a normal
E4M3 number), and the operand's scale_inv is 2^-e.  The exponent is drawn
  - per row of A and per row of B (= column of the output) for the vector-scale GEMM (OpVecFp8 / OpPlannedFp8),
  - per (128-token k-block, row) of A_t and of B_t for the block-scaled weight gradient (OpBlockFp8).
So the dequantised operand is exactly v, and every product that goes into one output element (of one k-block, for the
weight gradient) carries the same power of two.  While the partial sums stay below PARTIAL_LIMIT = 2^13 the tensor
core's fp8 accumulation is exact (the assumption tests/test_gemm_fp8_gpu.py makes), the dequantising multiply by a
power of two is exact, and the fp32 result is an integer.  A wrong row, column, k-block or stage scale then moves a
result by a power of two, never by rounding noise, and the check can ask for bits.

The bounds (tests/test_fp8_token_gemm_cpu.py asserts them for every shape below):
  - vector scales: the ping-pong kernel accumulates the whole K in the tensor core, so vmax^2 K < 2^13: vmax = 4 up to
    K = 256 (the tail shapes), vmax = 1 at the step shapes (K <= 6144).  With an epilogue input on a 2^-GRID grid
    (bias, old out0) the fp32 sum is exact while |result| < 2^(24 - GRID).
  - block scales: each 128-token k-block's partial sum is at most 128 vmax^2 = 2048 < 2^13 (vmax = 4), and K <= 13 344
    keeps |result| <= 213 504 < 2^18, so the fp32 accumulator holds the exact integer.  That is past 2^16, so under
    FLAG_ACCUM the sum with an old out0 on the 2^-8 grid need not be exact in fp32; the kernel forms it with one fp32
    add of two exact operands, which is the round-to-nearest-even of the exact sum, and the test asks for exactly that
    rounding (of the float64 sum, itself exact), then the bf16 rounding of it for a bf16 out0.
Padding columns of the operand buffers (K .. pitch) hold E4M3 NaN, so a kernel that read past K would give NaN.
"""
from __future__ import annotations

import torch

E4 = torch.float8_e4m3fn
NAN8 = 0x7f                 # an E4M3 NaN byte
EXP_LO, EXP_HI = -6, 6      # |v| 2^e in [2^-6, 4 * 2^6]: normal E4M3 (min normal 2^-6, max 448)
PARTIAL_LIMIT = 2 ** 13     # exact tensor-core fp8 accumulation below this
RESULT_LIMIT = 2 ** 24      # exact fp32 integers below this
GRID = 8                    # bias / old out0 values on a 2^-8 grid
BK = 128                    # tokens per k-block of the block-scaled weight gradient
ROW_CHUNK = 2048

# ---------------------------------------------------------------- the shapes the GPU tests run at
TAIL_M, TAIL_N, TAIL_K = (333, 2080), (136, 392, 1416), (40, 200, 256)
TAIL_VMAX = 4
STEP_VMAX = 1
# tower: (M = clips x tokens, D, hidden, tanh GELU, LayerScale)
TOWERS = {
    "cfg2": (32 * 417, 1408, 6144, True, True),        # InternVideo2 cfg-2 student
    "videomae": (32 * 157, 768, 3072, False, False),   # InternVideo1 VideoMAE-B
    "text": (16 * 77, 512, 2048, False, False),        # MobileCLIP-B text tower
}
PLAN_CLIPS, PLAN_ROWS, PLAN_N, PLAN_K, PLAN_VMAX = 32, (65, 417), 1416, 256, 4
WGRAD_K = (100, 128, 417, 1251, 13344)
WGRAD_MN = ((200, 328), (1416, 136))
WGRAD_CFG2 = (("qkv", 4224, 1408), ("proj", 1408, 1408), ("fc1", 6144, 1408), ("fc2", 1408, 6144))
WGRAD_CFG2_K = 13344
WGRAD_VMAX = 4


def step_gemms(tower):
    """The eight GEMMs of one block step of a tower: (name, N, K, epilogue name), M = TOWERS[tower][0]."""
    _, D, Hd, _, _ = TOWERS[tower]
    return [("qkv", 3 * D, D, "qkv"), ("proj", D, D, "proj"), ("fc1", Hd, D, "fc1"), ("fc2", D, Hd, "fc2"),
            ("dh", Hd, D, "dh"), ("dn2", D, Hd, "dgrad"), ("da", D, D, "dgrad"), ("dn1", D, 3 * D, "dgrad")]


def vec_bounds(vmax, K):
    """(largest |partial sum|, largest |result|) of an output of the vector-scale GEMM, in units of its scale."""
    return vmax * vmax * K, vmax * vmax * K


def block_bounds(vmax, K):
    """(largest |partial sum| of one k-block, largest |result|) of the block-scaled weight gradient."""
    return vmax * vmax * min(K, BK), vmax * vmax * K


# ---------------------------------------------------------------- operand builders
def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def _ints(shape, vmax, g, device):
    return torch.randint(-vmax, vmax + 1, shape, generator=g, device=device).float()


def _pack(x, K):
    """E4M3 [rows, K] view of x's [rows, pitch] buffer, with NaN bytes in columns K .. pitch."""
    q = x.to(E4)
    q.view(torch.uint8)[:, K:] = NAN8
    return q[:, :K]


def vec_operand(rows, K, pitch, seed, vmax, device="cuda"):
    """One exponent per row: (E4M3 [rows, K] view of a [rows, pitch] buffer, scale_inv fp32 [rows] = 2^-e,
    v fp32 [rows, K] = the dequantised operand)."""
    g = _gen(seed, device)
    v = _ints((rows, K), vmax, g, device)
    e = torch.randint(EXP_LO, EXP_HI + 1, (rows,), generator=g, device=device).float()
    x = torch.zeros((rows, pitch), device=device)
    x[:, :K] = v * torch.exp2(e)[:, None]
    return _pack(x, K), torch.exp2(-e), v


def block_operand(rows, K, pitch, seed, vmax, device="cuda"):
    """One exponent per (k-block, row): (E4M3 [rows, K] view of a [rows, pitch] buffer, scale_inv fp32 [nkb, rows] =
    2^-e, v fp32 [rows, K])."""
    g = _gen(seed, device)
    nkb = (K + BK - 1) // BK
    v = _ints((rows, K), vmax, g, device)
    e = torch.randint(EXP_LO, EXP_HI + 1, (nkb, rows), generator=g, device=device).float()
    x = torch.zeros((rows, pitch), device=device)
    x[:, :K] = v * torch.exp2(e).t().repeat_interleave(BK, 1)[:, :K]
    return _pack(x, K), torch.exp2(-e).contiguous(), v


def deq_vec(q, sinv):
    """float64 dequantised operand of vec_operand."""
    return q.double() * sinv.double()[:, None]


def deq_block(q, sinv):
    """float64 dequantised operand of block_operand."""
    return q.double() * sinv.double().t().repeat_interleave(BK, 1)[:, :q.shape[1]]


def grid_values(shape, seed, device="cuda", limit=1.0):
    """Values k 2^-GRID with |k 2^-GRID| < limit (at most 8 significant bits: exact in bf16), float32."""
    g = _gen(seed, device)
    k = int(limit * 2 ** GRID) - 1
    return torch.randint(-k, k + 1, shape, generator=g, device=device).float() * 2.0 ** -GRID


# ---------------------------------------------------------------- references
def wgrad_ref(va, vb, blocks=None):
    """float64 [M, N] = sum over the k-blocks `blocks` (None: all) of va[:, kb] vb[:, kb]^T, in row chunks."""
    K = va.shape[1]
    nkb = (K + BK - 1) // BK
    cols = torch.zeros(K, dtype=torch.bool, device=va.device)
    for kb in (range(nkb) if blocks is None else blocks):
        cols[kb * BK:(kb + 1) * BK] = True
    b = vb[:, cols].double().t()
    out = torch.empty((va.shape[0], vb.shape[0]), dtype=torch.float64, device=va.device)
    for r in range(0, va.shape[0], ROW_CHUNK):
        out[r:r + ROW_CHUNK] = va[r:r + ROW_CHUNK][:, cols].double() @ b
    return out


def wgrad_ref_int(va, vb, blocks=None):
    """int64 restatement of wgrad_ref, one k-block at a time (CPU)."""
    K = va.shape[1]
    nkb = (K + BK - 1) // BK
    out = torch.zeros((va.shape[0], vb.shape[0]), dtype=torch.int64)
    for kb in (range(nkb) if blocks is None else blocks):
        a = va[:, kb * BK:(kb + 1) * BK].long()
        b = vb[:, kb * BK:(kb + 1) * BK].long()
        out += (a[:, None, :] * b[None, :, :]).sum(-1)
    return out


def k_plan(blocks, K, device="cuda"):
    """int32 K plan of the weight gradient: the listed k-blocks ascending, the others after them (never read), then
    the count at [ceil(K / 128)]."""
    nkb = (K + BK - 1) // BK
    listed = sorted(blocks)
    rest = [kb for kb in range(nkb) if kb not in listed]
    return torch.tensor(listed + rest + [len(listed)], dtype=torch.int32, device=device)
