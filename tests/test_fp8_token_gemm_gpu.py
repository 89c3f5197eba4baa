"""The per-token FP8 training GEMMs on the H100 (gpu), element by element: every kernel form of the vector-scale GEMM
(OpVecFp8) with the epilogues training gives it, the DropPath-planned form (OpPlannedFp8) and the block-scaled weight
gradient (OpBlockFp8), on operands whose products are exact (tests/fp8_exact.py).

1. Vector scales (lowlevel.gemm_fp8 with [M] / [N] scale vectors), on ping-pong, the cooperative kernel at tile_n 128
   and 192, and the default: at ragged tails with every training epilogue, and at the full size of each tower's block
   step (cfg-2, VideoMAE, text tower) with each GEMM's own epilogue.  Where the fp32 value is exact the output must be
   its bits (rounded to nearest even for bf16): EPI_F32 (+ FLAG_ACCUM), EPI_BF16 (+ a bias on a 2^-8 grid), the
   pre-activation out1 of BIAS_GELU, RESID's out1 = y and save-grad GELU_BWD.  The GELU forms and the RESID sum are
   within tests/gemm_ref.py's per-element tolerance.  Outputs are views into NaN-filled wider buffers, and nothing
   outside a view may change.  A NaN row scale and a NaN column scale poison exactly their row and column.
2. The planned form (lowlevel._gemm_fp8_plan) against float64 itself, not against the unplanned call: live tiles,
   dropped clips' rows inside them included, match the reference; dead tiles hold the dead-tile table of ivb200.h.
3. The block-scaled weight gradient (lowlevel._gemm_fp8_wgrad): bits of the float64 integer sum, over all k-blocks or
   over a K plan's only (the others hold nonzero data), with K below, at and past k-block boundaries.
4. Accumulation at the per-token step shapes of the three towers: Gaussian operands cast as training casts them,
   ||C_kernel - C64(deq)||_F <= 0.25 ||C64(deq) - C64(bf16)||_F (DESIGN.md 4.1).
"""
import numpy as np
import pytest
import torch

import droppath_ref
import fp8_exact as fx
from gemm_ref import elem_errors, gemm_ref, worst
from internvideo_b200 import lowlevel as ll
from internvideo_b200 import ops

pytestmark = pytest.mark.gpu

bf, f32 = torch.bfloat16, torch.float32
LIMIT_BF16, LIMIT_F32 = 1.9, 1.4     # the limits of the bf16 epilogue tests (test_gemm_epilogue_gpu.LIMITS)
KERNELS = [("pingpong", ll.FLAG_PINGPONG, 0), ("coop128", ll.FLAG_1CTA, 128), ("coop192", ll.FLAG_1CTA, 192),
           ("default", 0, 0)]
KERNEL = {k[0]: k for k in KERNELS}


def _pad16(n):
    return (n + 15) // 16 * 16


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nan_view(M, N, dtype, init=None):
    """(buffer, [M, N] view): the view sits at row 1, column 8 of a NaN-filled [M + 2, N + 24] buffer (16-byte aligned
    rows, pitch a multiple of 8), holding `init` if given."""
    buf = torch.full((M + 2, N + 24), float("nan"), device="cuda", dtype=dtype)
    view = buf[1:M + 1, 8:N + 8]
    if init is not None:
        view.copy_(init)
    return buf, view


def _outside_untouched(buf, M, N):
    inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    inside[1:M + 1, 8:N + 8] = True
    return bool(torch.isnan(buf[~inside]).all())


def _mk(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=_gen(seed), device="cuda") * scale).to(bf)


def _epilogue(kind, M, N, seed, tanh=False, gamma=True, rowscale=None):
    """(epilogue kwargs of gemm_fp8 / gemm_ref, out0's old values or None) of one epilogue: a tail case of
    TAIL_EPILOGUES, or a step GEMM's training epilogue (qkv, proj, fc1, fc2, dh, dgrad).  The first word of `kind` names
    the epilogue, the others its variant.  Bias on the 2^-8 grid; out1 = True asks for an out1 buffer."""
    head, variant = kind.split()[0], kind.split()[1:]
    bias = fx.grid_values((N,), seed + 1).to(bf)
    tf = ll.FLAG_GELU_TANH if tanh or "tanh" in variant else 0
    if head == "f32":
        if "accum" in variant:
            return dict(epi=ll.EPI_F32, flags=ll.FLAG_ACCUM), fx.grid_values((M, N), seed + 2, limit=16.0)
        return dict(epi=ll.EPI_F32), None
    if head in ("bf16", "qkv", "dgrad"):
        return dict(epi=ll.EPI_BF16, bias=bias if "bias" in variant or head == "qkv" else None), None
    if head in ("gelu", "fc1"):
        save = head == "fc1" or "save" in variant
        out1 = head == "fc1" or "out1" in variant
        return dict(epi=ll.EPI_BIAS_GELU, bias=bias, out1=out1 or None,
                    flags=tf | (ll.FLAG_GELU_SAVE_GRAD if save else 0)), None
    if head in ("gelu_bwd", "dh"):
        save = head == "dh" or "save" in variant
        if save:   # the saved GELU' in bf16, as fc1's save-grad epilogue writes it
            aux = (torch.rand((M, N), generator=_gen(seed + 7), device="cuda") * 1.4 - 0.2).to(bf)
        else:      # the bf16 pre-activation
            aux = _mk((M, N), seed + 7, 2.0)
        return dict(epi=ll.EPI_GELU_BWD, aux=aux, flags=ll.FLAG_GELU_SAVE_GRAD if save else tf), None
    if head in ("resid", "proj", "fc2"):
        kw = dict(epi=ll.EPI_RESID, aux=torch.randn((M, N), generator=_gen(seed + 5), device="cuda"))
        if "plain" in variant:     # no bias, gamma, rowscale or out1
            return kw, None
        kw["bias"] = bias
        if gamma:   # LayerScale: gamma, the DropPath rowscale and out1 = y for gamma's gradient
            rs = rowscale if rowscale is not None else torch.rand((M,), generator=_gen(seed + 4), device="cuda") * 2
            kw.update(gamma=_mk((N,), seed + 6, 0.1), rowscale=rs, out1=True)
        return kw, None     # a tower without LayerScale: bias only, no out1 (as ops.block_forward calls it)
    raise ValueError(kind)


TAIL_EPILOGUES = ["f32", "f32 accum", "bf16", "bf16 bias",
                  "gelu", "gelu out1", "gelu save", "gelu save out1",
                  "gelu tanh", "gelu tanh out1", "gelu tanh save", "gelu tanh save out1",
                  "resid", "resid plain", "gelu_bwd", "gelu_bwd tanh", "gelu_bwd save"]


def _exact(kw, slot):
    """Whether output `slot` of the epilogue is the rounding of an exact fp32 value."""
    epi, flags = kw["epi"], kw.get("flags", 0)
    if slot == "out0":
        return epi in (ll.EPI_F32, ll.EPI_BF16) or (epi == ll.EPI_GELU_BWD and flags & ll.FLAG_GELU_SAVE_GRAD)
    return epi == ll.EPI_RESID or not flags & ll.FLAG_GELU_SAVE_GRAD      # out1: y, or the pre-activation h


def _check(got, ref, scale, exact, what, rows=None):
    """got against the float64 reference: the rounding of ref when exact, else within the per-element tolerance.
    rows: a boolean mask of the rows to check (default all)."""
    if rows is not None:
        if not bool(rows.any()):
            return
        got, ref = got[rows], ref[rows]
        scale = scale[rows] if scale is not None else None
    if exact:
        want = ref.float().to(got.dtype)
        same = (got == want) | (torch.isnan(got) & torch.isnan(want))
        if not bool(same.all()):
            _, where = worst((~same).float())
            raise AssertionError(f"{what}: {int((~same).sum())} elements differ from the exact result; first at {where}")
        return
    e, where = worst(elem_errors(got, ref, scale))
    lim = LIMIT_F32 if got.dtype == f32 else LIMIT_BF16
    assert e <= lim, (what, e, where)


def _run_vec(a8, sa, b8, sb, va, vb, kw, old, flags, tile_n, what, m_plan=None, live=None):
    """One call of the vector-scale GEMM (planned when m_plan is given) into NaN-padded outputs, checked against
    gemm_ref.  live: boolean [M] of the rows the reference applies to (the rest: the dead-tile table)."""
    kw = dict(kw)
    M, N = a8.shape[0], b8.shape[0]
    fl = kw.pop("flags", 0)
    out_dtype = f32 if kw["epi"] in (ll.EPI_F32, ll.EPI_RESID) else bf
    buf0, out0 = _nan_view(M, N, out_dtype, old)
    buf1, out1 = _nan_view(M, N, bf) if kw.get("out1") else (None, None)
    kw["out1"] = out1
    if m_plan is None:
        ll.gemm_fp8(a8, sa, b8, sb, out0=out0, flags=fl | flags, tile_n=tile_n, **kw)
    else:
        ll._gemm_fp8_plan(a8, sa, b8, sb, m_plan, out0=out0, flags=fl | flags, tile_n=tile_n, **kw)
    refs = gemm_ref(va, vb, out0=old, flags=fl, **kw)
    outs = [("out0", out0, buf0)] + ([("out1", out1, buf1)] if out1 is not None else [])
    for (ref, scale), (slot, got, buf) in zip(refs, outs):
        assert _outside_untouched(buf, M, N), (what, slot, "wrote outside its view")
        _check(got, ref, scale, _exact(kw | {"flags": fl}, slot), (what, slot), rows=live)
        if live is not None:
            dead = got[~live]
            want = kw["aux"][~live] if (kw["epi"] == ll.EPI_RESID and slot == "out0") else torch.zeros_like(dead)
            assert torch.equal(dead, want), (what, slot, "dead tile")


# ------------------------------------------------------------------------------------------------ 1. vector scales
TAILS = [(M, N, K) for M in fx.TAIL_M for N in fx.TAIL_N for K in fx.TAIL_K]


@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
@pytest.mark.parametrize("M,N,K", TAILS)
def test_vector_scales_training_epilogues_at_tails(cuda_lib, kernel, M, N, K):
    name, flag, tile_n = kernel
    pitch = _pad16(K) + 16
    a8, sa, va = fx.vec_operand(M, K, pitch, M + K, fx.TAIL_VMAX)
    b8, sb, vb = fx.vec_operand(N, K, pitch, N + K + 1, fx.TAIL_VMAX)
    seen = set()
    for ename in TAIL_EPILOGUES:
        kw, old = _epilogue(ename, M, N, seed=M + N + K)
        form = (kw["epi"], kw.get("flags", 0), old is not None) + tuple(k for k in sorted(kw) if kw[k] is not None)
        assert form not in seen, (ename, "repeats an earlier case")
        seen.add(form)
        _run_vec(a8, sa, b8, sb, va, vb, kw, old, flag, tile_n, (name, ename))


STEPS = [(tower, g) for tower in fx.TOWERS for g in fx.step_gemms(tower)]


@pytest.mark.parametrize("kernel", ["default", "pingpong"])
@pytest.mark.parametrize("tower,gemm", STEPS, ids=[f"{t}-{g[0]}" for t, g in STEPS])
def test_vector_scales_at_step_shapes(cuda_lib, tower, gemm, kernel):
    """Each GEMM of a tower's block step at full size, with its training epilogue, v in {-1, 0, 1}."""
    M, _, _, tanh, gamma = fx.TOWERS[tower]
    gname, N, K, ename = gemm
    _, flag, tile_n = KERNEL[kernel]
    a8, sa, va = fx.vec_operand(M, K, _pad16(K), M + K, fx.STEP_VMAX)
    b8, sb, vb = fx.vec_operand(N, K, _pad16(K), N + K + 1, fx.STEP_VMAX)
    kw, old = _epilogue(ename, M, N, seed=N + K, tanh=tanh, gamma=gamma)
    _run_vec(a8, sa, b8, sb, va, vb, kw, old, flag, tile_n, (tower, gname, kernel))


@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
@pytest.mark.parametrize("col", [202, 203], ids=["even_col", "odd_col"])
def test_nan_scale_poisons_its_row_and_column(cuda_lib, kernel, col):
    """A NaN in a_scale_inv[r] and in b_scale_inv[col] gives NaN in exactly row r and column col: not in the other
    column of col's 8-byte scale pair, not in row r +- 8 (the thread's other fragment row) or in row r + 64 (its other
    band).  Every other element keeps its exact value."""
    name, flag, tile_n = kernel
    M, N, K = 333, 392, 200
    pitch = _pad16(K) + 16
    a8, sa, va = fx.vec_operand(M, K, pitch, 5, fx.TAIL_VMAX)
    b8, sb, vb = fx.vec_operand(N, K, pitch, 6, fx.TAIL_VMAX)
    r = 139
    sa[r] = float("nan")
    sb[col] = float("nan")
    buf, out = _nan_view(M, N, f32)
    ll.gemm_fp8(a8, sa, b8, sb, epi=ll.EPI_F32, out0=out, flags=flag, tile_n=tile_n)
    assert _outside_untouched(buf, M, N), name
    want = (va.double() @ vb.double().t()).float()
    want[r] = float("nan")
    want[:, col] = float("nan")
    nan = torch.isnan(out)
    assert torch.equal(nan, torch.isnan(want)), (name, nan.nonzero()[:8].tolist())
    assert torch.equal(out[~nan], want[~nan]), name


# ------------------------------------------------------------------------------------------------ 2. planned form
DRAWS = {
    "random": np.random.default_rng(3).random(fx.PLAN_CLIPS) >= 0.25,
    "alternating": np.arange(fx.PLAN_CLIPS) % 2 == 0,
    "none_dropped": np.ones(fx.PLAN_CLIPS, bool),
    "all_dropped": np.zeros(fx.PLAN_CLIPS, bool),
}
PLAN_EPILOGUES = ["fc1", "proj", "dh", "dgrad"]


@pytest.mark.parametrize("kernel", ["pingpong", "coop128", "default"])
@pytest.mark.parametrize("n", fx.PLAN_ROWS)
@pytest.mark.parametrize("draw", list(DRAWS))
def test_planned_against_float64(cuda_lib, draw, n, kernel):
    """fc1 save-grad, proj RESID with the draw's rowscale (zeros on dropped clips), dh save-grad GELU_BWD and a plain
    dgrad.  Rows of dropped clips that share a live tile with kept rows are computed and checked like the others."""
    _, flag, tile_n = KERNEL[kernel]
    keep = DRAWS[draw]
    M, N, K = fx.PLAN_CLIPS * n, fx.PLAN_N, fx.PLAN_K
    rs_np = droppath_ref.clip_rows(keep, n)
    rs = torch.from_numpy(rs_np).cuda()
    m_plan = ops._branch_plans(ops.droppath_plan(rs[None].contiguous())[0], M, ops.FP8_TOKEN)[0]
    order, nlive, _ = droppath_ref.plan(rs_np)
    live = torch.zeros(M, dtype=torch.bool, device="cuda")
    for t in order[:nlive]:
        live[128 * t:128 * t + 128] = True
    pitch = _pad16(K) + 16
    a8, sa, va = fx.vec_operand(M, K, pitch, n + 1, fx.PLAN_VMAX)
    b8, sb, vb = fx.vec_operand(N, K, pitch, n + 2, fx.PLAN_VMAX)
    for ename in PLAN_EPILOGUES:
        kw, old = _epilogue(ename, M, N, seed=n, tanh=True, rowscale=rs)
        _run_vec(a8, sa, b8, sb, va, vb, kw, old, flag, tile_n, (kernel, draw, ename), m_plan=m_plan, live=live)


# ------------------------------------------------------------------------------------------------ 3. weight gradient
def _wgrad_operands(M, N, K, seed):
    pitch = _pad16(K) + 16
    a8, sa, va = fx.block_operand(M, K, pitch, seed, fx.WGRAD_VMAX)
    b8, sb, vb = fx.block_operand(N, K, pitch, seed + 1, fx.WGRAD_VMAX)
    return a8, sa, va, b8, sb, vb


def _wgrad_check(a8, sa, b8, sb, ref, k_plan, what, seed):
    """EPI_F32 and EPI_BF16 into NaN-padded views, and FLAG_ACCUM into a padded fp32 and a padded bf16 out0 holding
    values on the 2^-8 grid: the bits of ref, of its RNE rounding, and of fp32(ref + old) (rounded to bf16)."""
    M, N = ref.shape
    for epi, dt in ((ll.EPI_F32, f32), (ll.EPI_BF16, bf)):
        buf, out = _nan_view(M, N, dt)
        ll._gemm_fp8_wgrad(a8, sa, b8, sb, epi=epi, out0=out, k_plan=k_plan)
        assert _outside_untouched(buf, M, N), (what, epi)
        _check(out, ref, None, True, (what, epi))
        old = fx.grid_values((M, N), seed).to(dt)
        buf, out = _nan_view(M, N, dt, old)
        ll._gemm_fp8_wgrad(a8, sa, b8, sb, epi=epi, flags=ll.FLAG_ACCUM, out0=out, k_plan=k_plan)
        assert _outside_untouched(buf, M, N), (what, epi, "accum")
        want = (ref + old.double()).float().to(dt)
        diff = out != want
        assert not bool(diff.any()), (what, epi, "accum", worst(diff.float()))


WGRAD_SHAPES = [(M, N, K) for M, N in fx.WGRAD_MN for K in fx.WGRAD_K] + \
               [(M, N, fx.WGRAD_CFG2_K) for _, M, N in fx.WGRAD_CFG2]


@pytest.mark.parametrize("M,N,K", WGRAD_SHAPES)
def test_wgrad_exact(cuda_lib, M, N, K):
    a8, sa, va, b8, sb, vb = _wgrad_operands(M, N, K, M + N + K)
    _wgrad_check(a8, sa, b8, sb, fx.wgrad_ref(va, vb), None, (M, N, K), seed=K)


def _plans(nkb):
    rng = np.random.default_rng(nkb)
    plans = {"odd": list(range(1, nkb, 2)), "tail only": [nkb - 1], "all but tail": list(range(nkb - 1)),
             "random": sorted(rng.choice(nkb, size=max(1, nkb // 3), replace=False).tolist()), "empty": []}
    return plans


@pytest.mark.parametrize("M,N", fx.WGRAD_MN)
@pytest.mark.parametrize("K", [1251, 13344])
def test_wgrad_k_plan_sums_listed_blocks_only(cuda_lib, M, N, K):
    """Every k-block holds nonzero data; the result is the float64 sum over the listed ones.  An empty plan gives zeros,
    or leaves out0 as it was under FLAG_ACCUM."""
    a8, sa, va, b8, sb, vb = _wgrad_operands(M, N, K, 7 * K + M)
    nkb = (K + fx.BK - 1) // fx.BK
    for kb in range(nkb):   # no k-block is all zero in either operand
        assert bool(va[:, kb * fx.BK:(kb + 1) * fx.BK].any()) and bool(vb[:, kb * fx.BK:(kb + 1) * fx.BK].any())
    for pname, blocks in _plans(nkb).items():
        kp = fx.k_plan(blocks, K)
        ref = fx.wgrad_ref(va, vb, blocks)
        _wgrad_check(a8, sa, b8, sb, ref, kp, (M, N, K, pname), seed=len(blocks))
        if not blocks:
            assert not bool(ref.any())


# ------------------------------------------------------------------------------------------------ 4. accumulation
def token_accumulation_ratio(M, N, K, dgrad, seed=0):
    """||C_kernel - C64(deq)||_F / ||C64(deq) - C64(bf16)||_F on the default kernel, operands cast as per-token
    training casts them: forward, activation rows x weight rows (per output channel); dgrad, gradient rows x the
    weight [K, N] cast per input channel (fp8_quantize_rows(w, transposed=True))."""
    a = _mk((M, K), seed)
    if dgrad:
        w = _mk((K, N), seed + 1, 0.02)
        qb, sb = ll.fp8_quantize_rows(w, transposed=True)
        b = w.t()
    else:
        b = _mk((N, K), seed + 1, 0.02)
        qb, sb = ll.fp8_quantize_rows(b)
    qa, sa = ll.fp8_quantize_rows(a)
    c = ll.gemm_fp8(qa, sa, qb, sb, epi=ll.EPI_F32)
    num = den = 0.0
    bd = fx.deq_vec(qb, sb).t()
    b64 = b.double().t()
    for r in range(0, M, fx.ROW_CHUNK):
        rows = slice(r, min(r + fx.ROW_CHUNK, M))
        c_deq = fx.deq_vec(qa[rows], sa[rows]) @ bd
        c_bf = a[rows].double() @ b64
        num += float(((c[rows].double() - c_deq) ** 2).sum())
        den += float(((c_deq - c_bf) ** 2).sum())
    return (num / den) ** 0.5


@pytest.mark.parametrize("tower,gemm", STEPS, ids=[f"{t}-{g[0]}" for t, g in STEPS])
def test_accumulation_at_token_step_shapes(cuda_lib, tower, gemm):
    M = fx.TOWERS[tower][0]
    gname, N, K, _ = gemm
    r = token_accumulation_ratio(M, N, K, dgrad=gname in ("dh", "dn2", "da", "dn1"))
    print(f"{tower} {gname} {M}x{N}x{K}: per-token accumulation ratio {r:.4f}")
    assert r <= 0.25, (tower, gname, r)
