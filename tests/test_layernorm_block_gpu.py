"""The LayerNorm block (modules.VideoMAEBlock: InternVideo1's encoder and decoder blocks, the VideoMAEv2 teacher's block)
trained through ops.BlockFn, forward and every gradient against a float64 autograd restatement of the reference block
(oracle.restate's layernorm / linear / gelu, as restate._iv1_block, plus per-row DropPath factors).  Tolerances as
tests/test_model_gpu.py::test_block_cfg2_matches_reference_golden: 1e-2 relative for the output and the input gradient,
3e-2 for the parameter gradients.  The output and input gradient are compared without their identity part (x, dy), so
the bound is on what the block's two branches add.

Also: BlockFn refuses the teacher's head-axis attention (it has no backward), and the RMSNorm block's library calls
for one forward + backward are still exactly the ones listed below."""
from functools import partial

import pytest
import torch
import torch.nn as nn

from internvideo_b200 import _lib, ops
from internvideo_b200.modules import VideoMAEBlock
from oracle import restate as R

B = 2
SHAPES = {"iv1_s_encoder": (384, 6, 4.0, 157), "iv1_s_decoder": (192, 3, 4.0, 392), "giant": (1408, 16, 48 / 11, 157)}


def _rel(a, b):
    a = a.detach().double().cpu(); b = b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _block(D, H, mlp_ratio, gamma, qv_bias, checkpoint):
    torch.manual_seed(0)
    blk = VideoMAEBlock(D, H, mlp_ratio, qkv_bias=qv_bias, init_values=0.1 if gamma else None,
                        norm_layer=partial(nn.LayerNorm, eps=1e-6), with_cp=checkpoint)
    with torch.no_grad():
        for nm, p in blk.named_parameters():
            if nm.endswith("weight") and p.ndim == 1:          # norm weights
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif nm.endswith("bias"):
                p.normal_(0, 0.1)
            elif nm.startswith("gamma"):
                p.mul_(1 + 0.5 * torch.rand_like(p))
    return blk.bfloat16().cuda().train()


def _reference(p, x, H, eps, rs1, rs2):
    """The block in float64 on [B, n, D]; p: name -> float64 leaf tensor; rs1 / rs2: [B, n, 1] factors or None."""
    Bn, n, D = x.shape
    y = R.layernorm(x, p["norm1.weight"], p["norm1.bias"], eps)
    bias = None
    if "attn.q_bias" in p:
        bias = torch.cat((p["attn.q_bias"], torch.zeros_like(p["attn.v_bias"]), p["attn.v_bias"]))
    qkv = R.linear(y, p["attn.qkv.weight"], bias).reshape(Bn, n, 3, H, D // H).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    o = (((q * (D // H) ** -0.5) @ k.transpose(-2, -1)).softmax(-1) @ v).transpose(1, 2).reshape(Bn, n, D)
    a = R.linear(o, p["attn.proj.weight"], p["attn.proj.bias"])
    a = p["gamma_1"] * a if "gamma_1" in p else a
    h = x + (a if rs1 is None else rs1 * a)
    y = R.layernorm(h, p["norm2.weight"], p["norm2.bias"], eps)
    m = R.linear(R.gelu(R.linear(y, p["mlp.fc1.weight"], p["mlp.fc1.bias"])), p["mlp.fc2.weight"], p["mlp.fc2.bias"])
    m = p["gamma_2"] * m if "gamma_2" in p else m
    return h + (m if rs2 is None else rs2 * m)


@pytest.mark.gpu
@pytest.mark.parametrize("checkpoint", [False, True], ids=["saved", "checkpoint"])
@pytest.mark.parametrize("rowscale", [False, True], ids=["no_droppath", "droppath"])
@pytest.mark.parametrize("gamma,qv_bias", [(True, True), (False, True), (True, False), (False, False)],
                         ids=["gamma_qvbias", "qvbias", "gamma", "plain"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_layernorm_block_fn_matches_float64(cuda_lib, shape, gamma, qv_bias, rowscale, checkpoint):
    D, H, mlp_ratio, n = SHAPES[shape]
    blk = _block(D, H, mlp_ratio, gamma, qv_bias, checkpoint)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((B * n, D), generator=g)
    dy = torch.randn((B * n, D), generator=g)
    rs1 = rs2 = None
    if rowscale:     # DropPath factors per clip (0 or 1/keep), expanded to rows; each branch drops one clip
        rs1 = torch.tensor([0.0, 1.25]).repeat_interleave(n)
        rs2 = torch.tensor([1.25, 0.0]).repeat_interleave(n)
    xs = x.cuda().requires_grad_(True)
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    y = ops.BlockFn.apply(xs, blk._spec(B, n, training=True), dev(rs1), dev(rs2), *blk._param_tuple())
    y.backward(dy.cuda())

    p = {k: v.detach().double().cpu().requires_grad_(True) for k, v in blk.named_parameters()}
    x64 = x.double().reshape(B, n, D).requires_grad_(True)
    r3 = lambda t: None if t is None else t.double().reshape(B, n, 1)  # noqa: E731
    y64 = _reference(p, x64, H, blk.norm1.eps, r3(rs1), r3(rs2))
    y64.backward(dy.double().reshape(B, n, D))

    assert _rel(y - xs, (y64 - x64).reshape(B * n, D)) < 1e-2
    assert _rel(xs.grad - dy.cuda(), x64.grad.reshape(B * n, D) - dy.double()) < 1e-2
    bad = {}
    for k, prm in blk.named_parameters():
        r = _rel(prm.grad, p[k].grad)
        if not r < 3e-2:
            bad[k] = r
    assert not bad, bad


def test_layernorm_block_refusals():
    """BlockFn refuses the head-axis attention (no backward) before any library call; a head split that does not
    cover dim is refused at construction."""
    blk = VideoMAEBlock(64, 2, qkv_bias=True)
    x = torch.zeros((2 * 8, 64), requires_grad=True)
    with pytest.raises(_lib.IvbError, match="head-axis"):
        ops.BlockFn.apply(x, blk._spec(2, 8, training=True, head_axis=True), None, None, *blk._param_tuple())
    with pytest.raises(NotImplementedError, match="head_dim"):
        VideoMAEBlock(64, 2, attn_head_dim=16)


# The library calls (OpProfiler names) of one forward + backward of the RMSNorm block in tests/test_binding_gpu.py.  The
# LayerNorm path of block_backward must leave them as they are: the same calls in the same order, the same GEMM
# layouts, epilogues and shapes.
RMSNORM_BLOCK_CALLS = [
    "norm_fwd", "gemm[NN epi0] 1028x384x128", "rmsnorm_pair_fwd", "attn_fwd", "gemm[NN epi3] 1028x128x128", "norm_fwd",
    "gemm[NN epi2] 1028x512x128", "gemm[NN epi3] 1028x128x512", "layerscale_bwd", "gemm[TT epi0] 128x512x1028",
    "gemm[NT epi4] 1028x512x128", "colsum_bf16", "gemm[TT epi0] 512x128x1028", "gemm[NT epi0] 1028x128x512",
    "rmsnorm_bwd_layerscale", "gemm[TT epi0] 128x128x1028", "gemm[NT epi0] 1028x128x128", "attn_bwd",
    "rmsnorm_pair_bwd", "gemm[TT epi0] 384x128x1028", "gemm[NT epi0] 1028x128x384", "norm_bwd",
]


@pytest.mark.gpu
def test_rmsnorm_block_library_calls_unchanged(cuda_lib):
    from internvideo_b200 import lowlevel as ll
    from test_binding_gpu import _block_step
    _block_step()                                                  # warm-up
    prof = ll.OpProfiler()
    prof.enable()
    try:
        _block_step()
    finally:
        prof.disable()
    assert [r[0] for r in prof.records] == RMSNORM_BLOCK_CALLS
