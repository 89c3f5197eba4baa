"""Per-token FP8 training of the ViT blocks (modules.set_fp8(model, scaling="token")) on the H100 (gpu).

- ivb_norm_fwd_fp8_train: bf16 row, mean and rstd bit-identical to ivb_norm_fwd; E4M3 rows and scales bit-identical
  to ivb_norm_fwd_fp8; padding of every output keeps its bits.
- ivb_fp8_quantize_cols_t: element by element against a float64 restatement of the scale rule, with tails in both
  dimensions, a zero column, an Inf column and a NaN column; the same bits on two runs.
- Row independence of the input-gradient GEMM: scaling one gradient row by a power of two leaves every other row of dx
  bit-identical.
- The block at the block_cfg2 size against the bf16 block, and the mode end to end on the pretrain_tiny model.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
bf16, f32, e4m3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
NAN8 = 0x7f    # an E4M3 NaN byte


def _pad16(n):
    return (n + 15) // 16 * 16


# ------------------------------------------------------------------------------------------------ kernel (a)
@pytest.mark.parametrize("layernorm", [False, True], ids=["rms", "ln"])
@pytest.mark.parametrize("x_f32", [True, False], ids=["xf32", "xbf16"])
@pytest.mark.parametrize("D", [8, 384, 1408, 1544, 4096])
def test_norm_fwd_fp8_train_bits(cuda_lib, layernorm, x_f32, D):
    ll = cuda_lib
    M = 333
    g = torch.Generator(device="cuda").manual_seed(D + 7 * layernorm + 3 * x_f32)
    xb = torch.randn((M, D + 24), device="cuda", generator=g) * 3 + 0.5
    x = (xb if x_f32 else xb.to(bf16))[:, :D]                     # padded pitch ldx = D + 24
    w = (1 + 0.2 * torch.randn(D, device="cuda", generator=g)).to(bf16)
    b = (0.1 * torch.randn(D, device="cuda", generator=g)).to(bf16) if layernorm else None
    eps = 1e-5 if layernorm else 1e-6
    ldy, ldo = D + 8, _pad16(D) + 16
    y = torch.full((M, ldy), float("nan"), device="cuda", dtype=bf16)
    q = torch.full((M, ldo), NAN8, device="cuda", dtype=torch.uint8)
    stats = torch.full((3, M + 1), float("nan"), device="cuda", dtype=f32)   # sinv, mean, rstd; one guard element each
    ll._call("norm_fwd_fp8_train", x, int(x_f32), x.stride(0), w, b, eps, int(layernorm), M, D, q, ldo, stats[0], y,
             ldy, stats[1], stats[2])
    y_ref, mean_ref, rstd_ref = ll.norm_fwd(x, w, b, eps=eps, layernorm=layernorm)
    q_ref, s_ref = ll.norm_fwd_fp8(x, w, b, eps=eps, layernorm=layernorm)
    torch.cuda.synchronize()
    assert torch.equal(y[:, :D].view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(stats[2, :M].view(torch.int32), rstd_ref.view(torch.int32))
    if layernorm:
        assert torch.equal(stats[1, :M].view(torch.int32), mean_ref.view(torch.int32))
    else:
        assert torch.isnan(stats[1]).all()                       # RMSNorm writes no mean
    assert torch.equal(q[:, :D], q_ref.view(torch.uint8))
    assert torch.equal(stats[0, :M].view(torch.int32), s_ref.view(torch.int32))
    assert torch.isnan(y[:, D:].float()).all() and (q[:, D:] == NAN8).all() and torch.isnan(stats[:, M]).all()
    # the lowlevel form returns the same bits
    q2, s2, y2, mean2, rstd2 = ll.norm_fwd_fp8(x, w, b, eps=eps, layernorm=layernorm, save=True)
    assert torch.equal(q2.view(torch.uint8), q[:, :D]) and torch.equal(y2.view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(rstd2, rstd_ref) and (mean2 is None) == (not layernorm)


# ------------------------------------------------------------------------------------------------ kernel (b)
def _cols_reference(w):
    """float64 restatement: per column k, scale 2^e with e the largest integer such that amax_k * 2^e <= 448 (e in
    [-126, 126]; 1 for a zero column), q_t[k] = RNE_e4m3(w[:, k] * scale), scale_inv NaN for a non-finite column."""
    w64 = w.double()
    amax = w64.abs().amax(0)
    e = torch.floor(torch.log2(448.0 / amax.clamp_min(1e-300)))
    e = torch.where(amax * torch.exp2(e + 1) <= 448.0, e + 1, e)
    e = torch.where(amax * torch.exp2(e) > 448.0, e - 1, e)
    e = torch.where(amax == 0, torch.zeros_like(e), e.clamp(-126, 126))
    finite = torch.isfinite(amax)
    e = torch.where(finite, e, torch.zeros_like(e))
    scale = torch.exp2(e)
    q_t = (w64 * scale).float().t().contiguous().to(e4m3)
    sinv = torch.where(finite, 1.0 / scale, torch.full_like(scale, float("nan")))
    return q_t, sinv, amax


@pytest.mark.parametrize("N,K", [(197, 133), (64, 64), (6144, 1408), (1408, 6144), (77, 4224)])
def test_quantize_cols_t_against_float64(cuda_lib, N, K):
    ll = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(N * 31 + K)
    ldx = (K + 7) // 8 * 8 + 8
    wb = (torch.randn((N, ldx), device="cuda", generator=g) * 0.02)
    wb[:, : K // 2] *= torch.exp2(torch.randint(-20, 20, (K // 2,), device="cuda", generator=g).float())
    wb = wb.to(bf16)
    w = wb[:, :K]
    w[:, 5] = 0                                       # a zero column
    w[N // 2, 7] = float("inf")                       # an Inf column
    w[N // 3, 7] = -float("inf")
    w[1, 9] = float("nan")                            # a NaN column
    ldt = _pad16(N) + 16
    runs = []
    for _ in range(2):
        q_t = torch.full((K, ldt), NAN8, device="cuda", dtype=torch.uint8)
        amax = torch.full((K + 1,), float("nan"), device="cuda", dtype=f32)
        sinv = torch.full((K + 1,), float("nan"), device="cuda", dtype=f32)
        ll._call("fp8_quantize_cols_t", w, ldx, N, K, q_t, ldt, amax, sinv)
        runs.append((q_t, amax, sinv))
    torch.cuda.synchronize()
    (q_t, amax, sinv), (q_t2, amax2, sinv2) = runs
    assert torch.equal(q_t, q_t2) and torch.equal(sinv.view(torch.int32), sinv2.view(torch.int32))
    q_ref, s_ref, a_ref = _cols_reference(w)
    fin = torch.isfinite(a_ref)
    assert not bool(fin[7]) and bool(torch.isnan(sinv[7]))
    assert torch.equal(sinv[:K][fin].double(), s_ref[fin])
    assert torch.equal(amax[:K].double()[fin], a_ref[fin]) and float(sinv[5]) == 1.0
    assert torch.equal(q_t[:, :N][fin], q_ref.view(torch.uint8)[fin])
    assert (q_t[:, N:] == NAN8).all() and torch.isnan(amax[K]) and torch.isnan(sinv[K])
    # the non-finite columns: scale 1 and a satfinite cast, so an Inf becomes +-448 and a NaN stays NaN
    for k in (7, 9):
        col, nan = w[:, k].float(), torch.isnan(w[:, k].float())
        assert torch.equal(q_t[k, :N][~nan], col.clamp(-448, 448).to(e4m3).view(torch.uint8)[~nan])
        assert bool(((q_t[k, :N][nan] & 0x7f) == 0x7f).all()) and bool(torch.isnan(sinv[k]))
    # the lowlevel form: the rows of w^T, the same bits as the per-row cast of w^T
    qt3, s3 = ll.fp8_quantize_rows(w, transposed=True)
    assert torch.equal(qt3.view(torch.uint8), q_t[:, :N])
    wt = torch.zeros((K, (N + 7) // 8 * 8), device="cuda", dtype=bf16)   # the row cast wants a pitch of 8 elements
    wt[:, :N] = w.t()
    q_rows, s_rows = ll.fp8_quantize_rows(wt[:, :N])
    assert torch.equal(q_rows.view(torch.uint8)[fin], q_t[:, :N][fin]) and torch.equal(s_rows[fin], sinv[:K][fin])


# ------------------------------------------------------------------------------------------------ row independence
def test_dgrad_rows_are_independent(cuda_lib):
    ll = cuda_lib
    M, N, K = 777, 1408, 640
    g = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn((M, N), device="cuda", generator=g).to(bf16)
    w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(bf16)
    w_t, ws = ll.fp8_quantize_rows(w, transposed=True)

    def dgrad(d):
        q, s = ll.fp8_quantize_rows(d)
        return ll.gemm_fp8(q, s, w_t, ws, epi=ll.EPI_F32)
    dx = dgrad(dy)
    dy2 = dy.clone()
    r = 300
    dy2[r] *= 2.0 ** 12
    dx2 = dgrad(dy2)
    others = torch.arange(M, device="cuda") != r
    assert torch.equal(dx2[others], dx[others])
    assert torch.equal(dx2[r], dx[r] * 2.0 ** 12)


# ------------------------------------------------------------------------------------------------ the block
# Relative Frobenius errors against the bf16 block at block_cfg2 (D = 1408, 16 heads, hidden 6144, B = 2 x 417 tokens).
# The derived bounds, from E4M3's unit roundoff u = 2^-4: output 2u = 0.125 (E4M3 x E4M3 GEMMs); dx and parameter
# gradients 4u = 0.25 (E4M3 gradients x E4M3 weights, and weight gradients reading the FP8 forward's activations).
# Each limit is the smaller of its derived bound and 1.5 times the value measured on an H100 80GB HBM3 (MEASURED; the
# computation is deterministic).  Per-tensor FP8 on the same inputs measured y 0.0546, dx 0.0894, gradients up to 0.104.
U = 2.0 ** -4
MEASURED = {"y": 0.0546, "dx": 0.0623, "norm1.weight": 0.0849, "attn.qkv.weight": 0.0770, "attn.proj.weight": 0.0643,
            "attn.proj.bias": 0.0081, "attn.q_norm.weight": 0.0902, "attn.k_norm.weight": 0.0902, "ls1.gamma": 0.0708,
            "norm2.weight": 0.0602, "mlp.fc1.weight": 0.0489, "mlp.fc1.bias": 0.0490, "mlp.fc2.weight": 0.0390,
            "mlp.fc2.bias": 0.0, "ls2.gamma": 0.0547}
LIMITS = {k: min(2 * U if k == "y" else 4 * U, 1.5 * v) for k, v in MEASURED.items()}


def _rel(a, b):
    a = a.detach().double(); b = b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _block(with_cp=False):
    from internvideo_b200 import modules as M
    from oracle.make_golden import block_cfg2_inputs
    z = np.load(GOLD / "block_cfg2.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd, x, dy = block_cfg2_inputs(cfg)
    D, H, B, n = cfg["dim"], cfg["num_heads"], cfg["B"], cfg["n"]
    blk = M.Block(D, H, cfg["mlp_ratio"], init_values=cfg["init_values"], qk_normalization=True, with_cp=with_cp)
    blk.load_state_dict(sd, strict=True)
    blk = blk.bfloat16().cuda()
    return blk, x.reshape(B * n, D).cuda(), dy.reshape(B * n, D).cuda(), B, n


def _run(blk, x, dy, B, n):
    for p in blk.parameters():
        p.grad = None
    xs = x.clone().requires_grad_(True)
    y = blk.forward_stream(xs, B, n)
    y.backward(dy)
    return y.detach(), xs.grad, {k: p.grad.clone() for k, p in blk.named_parameters()}


def _errors(res, ref, x, dy):
    (y1, dx1, g1), (y0, dx0, g0) = res, ref
    r = {"y": _rel(y1 - x, y0 - x), "dx": _rel(dx1 - dy, dx0 - dy)}   # the branches' share: the residual is exact
    r.update({k: _rel(g1[k], g0[k]) for k in g0})
    return r


def test_token_block_within_limits_of_bf16(cuda_lib):
    from internvideo_b200.modules import set_fp8
    blk, x, dy, B, n = _block()
    ref = _run(blk, x, dy, B, n)
    errs = {}
    for scaling in ("tensor", "token"):
        set_fp8(blk, True, scaling=scaling)
        errs[scaling] = _errors(_run(blk, x, dy, B, n), ref, x, dy)
        print(f"{scaling} FP8 vs bf16 relative errors:", {k: round(v, 4) for k, v in errs[scaling].items()})
    r = errs["token"]
    assert set(r) == set(LIMITS), sorted(r)
    bad = {k: (v, LIMITS[k]) for k, v in r.items() if v > LIMITS[k]}
    assert not bad, bad
    assert r["y"] > 0     # not the bf16 bits: the FP8 path ran


def test_token_checkpointed_block_is_bit_identical(cuda_lib):
    from internvideo_b200.modules import set_fp8
    res = []
    for with_cp in (False, True):
        blk, x, dy, B, n = _block(with_cp)
        set_fp8(blk, True, scaling="token")
        res.append(_run(blk, x, dy, B, n))
    (y0, dx0, g0), (y1, dx1, g1) = res
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_token_no_grad_forward_matches_training_forward(cuda_lib):
    from internvideo_b200.modules import set_fp8
    blk, x, dy, B, n = _block()
    set_fp8(blk, True, scaling="token")
    y_train, _, _ = _run(blk, x, dy, B, n)
    with torch.no_grad():
        y_infer = blk.forward_stream(x.clone(), B, n)
    assert torch.equal(y_infer, y_train)


def test_token_off_restores_bf16_bits_and_excludes_fp8_inference(cuda_lib):
    from internvideo_b200 import _lib
    from internvideo_b200.modules import set_fp8, set_fp8_inference
    blk, x, dy, B, n = _block()
    y0, dx0, g0 = _run(blk, x, dy, B, n)
    set_fp8(blk, True, scaling="token")
    _run(blk, x, dy, B, n)
    with pytest.raises(_lib.IvbError, match="switch that off first"):
        set_fp8_inference(blk)
    assert set_fp8(blk, False) == 1
    y1, dx1, g1 = _run(blk, x, dy, B, n)
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    set_fp8_inference(blk)
    set_fp8(blk, True, scaling="token")
    with pytest.raises(_lib.IvbError, match="both on"), torch.no_grad():
        blk.forward_stream(x.clone(), B, n)


# ------------------------------------------------------------------------------------------------ end to end
def _setup(fp8, direct=True, check_finite=False):
    from internvideo_b200.engine import PretrainEngine
    from internvideo_b200.modules import PretrainInternVideo2, set_fp8
    z = np.load(GOLD / "pretrain_tiny.npz")
    cfg = json.loads(bytes(z["cfg"]).decode())
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    model = PretrainInternVideo2(use_flash_attn=False, use_fused_rmsnorm=False, use_fused_mlp=False, **cfg)
    model.load_state_dict(sd, strict=True)
    model = model.bfloat16().cuda().train()
    assert set_fp8(model, fp8, scaling="token") > 0
    eng = PretrainEngine(model, lr=1e-3, clip_grad=0.0, direct_grads=direct, check_finite=check_finite)
    x = torch.from_numpy(z["x"]).cuda().to(torch.bfloat16)
    mask = torch.from_numpy(z["mask"]).cuda()
    tg = [torch.from_numpy(z[k]).cuda() for k in ("tgt_clip", "tgt_final", "tgt_mae")]
    return model, eng, x, mask, tg


def _loss(model, x, mask, tg, n_visible=None):
    lc, lf, lm = model.forward_loss(x, mask, tg[0], tg[1], tg[2], n_visible=n_visible)
    return lc + lf + lm


def _train(fp8, steps=100):
    torch.manual_seed(0)
    model, eng, x, mask, tg = _setup(fp8)
    losses = []
    for _ in range(steps):
        eng.zero_grad()
        loss = _loss(model, x, mask, tg)
        loss.backward()
        eng.step()
        losses.append(float(loss))
    return losses


def test_token_training_loss_drops_like_bf16(cuda_lib):
    bf = _train(False)
    f8 = _train(True)
    drop_bf, drop_f8 = bf[0] - bf[-1], f8[0] - f8[-1]
    print(f"loss bf16 {bf[0]:.4f} -> {bf[-1]:.4f}, per-token fp8 {f8[0]:.4f} -> {f8[-1]:.4f}")
    assert drop_bf > 0
    assert drop_f8 >= 0.9 * drop_bf, (drop_f8, drop_bf)


def test_token_gradient_sink_matches_autograd(cuda_lib):
    flats = []
    for direct in (False, True):
        torch.manual_seed(0)
        model, eng, x, mask, tg = _setup(True, direct=direct)
        eng.zero_grad()
        _loss(model, x, mask, tg).backward()
        flats.append(eng.flat_grad.float().clone())
    rel = float((flats[1] - flats[0]).norm() / flats[0].norm())
    assert float(flats[0].norm()) > 0 and rel < 2e-3, rel


def test_token_step_with_inf_input_is_skipped(cuda_lib):
    torch.manual_seed(0)
    model, eng, x, mask, tg = _setup(True, check_finite=True)
    before = [p.detach().clone() for p in model.parameters()]
    x = x.clone()
    x.fill_(float("inf"))
    eng.zero_grad()
    _loss(model, x, mask, tg).backward()
    eng.step()
    assert float(eng.skipped) == 1.0
    for p, b in zip(model.parameters(), before):
        assert torch.equal(p.detach(), b)


def test_token_step_replays_in_a_cuda_graph(cuda_lib):
    """The whole per-token FP8 step (forward, backward, AdamW) captured in engine.GraphedStep replays with the eager
    step's loss.  Both arms start from the same model and take one warm-up step first.  The loss sums per-block
    partials with atomics, so its last bits may differ between any two runs: 8 fp32 ulps are allowed."""
    from internvideo_b200.engine import GraphedStep
    arms = []
    for _ in range(2):
        torch.manual_seed(0)
        model, eng, x, mask, tg = _setup(True)
        n_visible = int(mask.shape[1] - int(mask[0].sum()))    # given, so the captured step reads nothing to the host

        def step(v, model=model, eng=eng, mask=mask, tg=tg, n_visible=n_visible):
            eng.zero_grad()
            loss = _loss(model, v, mask, tg, n_visible)
            loss.backward()
            eng.step()
            return loss
        arms.append((step, x))
    step, x = arms[0]
    step(x)
    loss_eager = float(step(x))
    step, x = arms[1]
    graphed = GraphedStep(step, [x.clone()], warmup=1)
    loss_graph = float(graphed(x)[0])
    torch.cuda.synchronize()
    print(f"per-token FP8 step: eager loss {loss_eager!r}, graph replay {loss_graph!r}")
    assert loss_eager == loss_eager and abs(loss_graph - loss_eager) <= 8 * 2.0 ** -23 * abs(loss_eager)
