"""The row-kernel entry points of ivb_norm.cu, ivb_loss.cu and ivb_embed.cu refuse a bad pitch or a misaligned row
operand before any CUDA call (include/ivb200.h, Conventions), checked through the raw C ABI: each returns non-zero with
its message in ivb_last_error().  ivb_gather_add and ivb_scatter_add move rows in 16-byte vectors like the norm kernels;
ivb_im2col_visible moves 4-byte words, so its video and cols need 4-byte alignment.  The refused calls pass null or fake device addresses; were a check missing, the call would go on to
launch a kernel on them, so those cases run only where no CUDA device is present."""
import pytest

from abi_fake import cpu_only, expect_refusal
from internvideo_b200 import _lib

A = 1 << 20          # a fake 16-byte aligned device address
M, D = 417, 1408


# One call per entry point, taking a {operand: address} dict and a {pitch name: pitch} dict (default pitch D).
def _norm_fwd(p, ld):
    return _lib.load().ivb_norm_fwd(p["x"], 1, ld.get("ldx", D), p["weight"], p["bias"], 1e-5, 1, M, D, p["y"],
                                    ld.get("ldy", D), p["mean"], p["rstd"], None)


def _norm_bwd(p, ld):
    return _lib.load().ivb_norm_bwd(p["dy"], ld.get("lddy", D), p["x"], 1, ld.get("ldx", D), p["weight"], p["mean"],
                                    p["rstd"], 1, M, D, p["dx_in"], ld.get("lddx_in", D), p["dx_out"], 1,
                                    ld.get("lddx", D), p["dweight"], p["dbias"], None)


def _layerscale_bwd(p, ld):
    return _lib.load().ivb_layerscale_bwd(p["dx"], ld.get("lddx", D), p["y"], ld.get("ldy", D), p["gamma"], M, D,
                                          p["dy"], ld.get("lddy", D), p["dgamma"], p["dcolsum"], p["rowscale"], None)


def _colsum(p, ld):
    return _lib.load().ivb_colsum_bf16(p["x"], ld.get("ldx", D), M, D, p["out"], None)


def _pair_fwd(p, ld):
    return _lib.load().ivb_rmsnorm_pair_fwd(p["x"], 3 * D, D, p["w0"], p["w1"], 1e-6, M, D, p["y"], 2 * D, D, p["rstd"],
                                            None)


def _pair_bwd(p, ld):
    return _lib.load().ivb_rmsnorm_pair_bwd(p["dy"], 3 * D, D, p["x"], 3 * D, D, p["w0"], p["w1"], p["rstd"], M, D,
                                            p["dx_out"], 3 * D, D, p["dw0"], p["dw1"], None)


def _bwd_layerscale(p, ld):
    return _lib.load().ivb_rmsnorm_bwd_layerscale(p["dy"], D, p["x"], D, p["weight"], p["rstd"], M, D, p["dx_in"], D,
                                                  p["dx_out"], D, p["dweight"], p["ybr"], D, p["gamma"], p["rowscale"],
                                                  p["dyb"], D, p["dgamma"], p["dcolsum"], None)


def _ln_l2_fwd(p, ld):
    return _lib.load().ivb_ln_l2_fwd(p["z"], D, p["weight"], p["bias"], 1e-5, M, D, p["out"], ld.get("ldo", D),
                                     p["stats"], p["target"], 0, ld.get("ldt", D), p["loss_sum"], None)


def _ln_l2_bwd(p, ld):
    return _lib.load().ivb_ln_l2_bwd(p["z"], D, p["weight"], p["bias"], p["stats"], M, D, p["dout"], 0, D, -1.0, None,
                                     p["dz"], D, p["dweight"], p["dbias"], None)


def _l2n_fwd(p, ld):
    return _lib.load().ivb_l2norm_rows_fwd(p["x"], 1, D, M, D, p["out"], D, p["inv"], None)


def _l2n_bwd(p, ld):
    return _lib.load().ivb_l2norm_rows_bwd(p["dy"], D, p["xn"], D, p["inv"], M, D, p["dx"], D, None)


def _pool_fwd(p, ld):
    return _lib.load().ivb_pool_attn_fwd(p["q"], p["k"], D, p["v"], D, 2, 417, 16, 88, 0.1, p["out"], p["probs"], None)


def _pool_bwd(p, ld):
    return _lib.load().ivb_pool_attn_bwd(p["q"], p["k"], D, p["v"], D, p["probs"], p["dout"], 2, 417, 16, 88, 0.1,
                                         p["dq"], p["dk"], D, p["dv"], D, None)


def _gather_add(p, ld):
    return _lib.load().ivb_gather_add(p["src"], ld.get("src_bstride", 0), p["table"], p["idx"], 197, -1, 2, 196, D,
                                      p["out"], 1, ld.get("out_bstride", 197 * D), None)


def _scatter_add(p, ld):
    return _lib.load().ivb_scatter_add(p["g"], 0, ld.get("g_bstride", 196 * D), p["idx"], 197, -1, 2, 196, D,
                                       p["table_grad"], None)


def _im2col(p, ld):
    return _lib.load().ivb_im2col_visible(p["video"], p["idx"], 197, 1, 40, 2, 3, 16, 224, 224, 2, 14, 1176, p["cols"],
                                          None)


# entry point: (call, its pointer operands, the row operands among them that must be 16-byte aligned)
ENTRIES = {
    "ivb_norm_fwd": (_norm_fwd, "x weight bias y mean rstd", "x weight bias y"),
    "ivb_norm_bwd": (_norm_bwd, "dy x weight mean rstd dx_in dx_out dweight dbias", "dy x weight dx_in dx_out"),
    "ivb_layerscale_bwd": (_layerscale_bwd, "dx y gamma dy dgamma dcolsum rowscale", "dx y gamma dy"),
    "ivb_colsum_bf16": (_colsum, "x out", "x"),
    "ivb_rmsnorm_pair_fwd": (_pair_fwd, "x w0 w1 y rstd", "x w0 w1 y"),
    "ivb_rmsnorm_pair_bwd": (_pair_bwd, "dy x w0 w1 rstd dx_out dw0 dw1", "dy x w0 w1 dx_out"),
    "ivb_rmsnorm_bwd_layerscale": (_bwd_layerscale,
                                   "dy x weight rstd dx_in dx_out dweight ybr gamma rowscale dyb dgamma dcolsum",
                                   "dy x dx_in dx_out ybr dyb"),
    "ivb_ln_l2_fwd": (_ln_l2_fwd, "z weight bias out stats target loss_sum", "z weight bias out target"),
    "ivb_ln_l2_bwd": (_ln_l2_bwd, "z weight bias stats dout dz dweight dbias", "z weight bias dout dz"),
    "ivb_l2norm_rows_fwd": (_l2n_fwd, "x out inv", "x out"),
    "ivb_l2norm_rows_bwd": (_l2n_bwd, "dy xn inv dx", "dy xn dx"),
    "ivb_pool_attn_fwd": (_pool_fwd, "q k v out probs", "k v"),
    "ivb_pool_attn_bwd": (_pool_bwd, "q k v probs dout dq dk dv", "k v dk dv"),
    "ivb_gather_add": (_gather_add, "src table idx out", "src table out"),
    "ivb_scatter_add": (_scatter_add, "g idx table_grad", "g table_grad"),
    "ivb_im2col_visible": (_im2col, "video idx cols", ""),
}
ROW_OPERANDS = [(e, op) for e, (_, _, ops) in ENTRIES.items() for op in ops.split()]


def _ptrs(entry, **override):
    names = ENTRIES[entry][1].split()
    p = {n: A + (i << 16) for i, n in enumerate(names)}
    p.update(override)
    return p


@cpu_only
@pytest.mark.parametrize("entry,operand", ROW_OPERANDS)
def test_misaligned_row_operand_refused(entry, operand):
    """A view starting at a column that is not a multiple of 8 (bf16) or 4 (fp32) is refused, not read or written
    with misaligned vector accesses."""
    call = ENTRIES[entry][0]
    expect_refusal(call(_ptrs(entry, **{operand: A + 8}), {}), f"{entry}: ")
    assert "aligned" in _lib.load().ivb_last_error().decode()


@cpu_only
@pytest.mark.parametrize("operand", ["weight", "gamma"])
def test_fused_layerscale_weight_gamma_need_8_bytes(operand):
    """The bulk-copy kernel reads weight and gamma 4 bf16 at a time: 8-byte alignment is its rule for them."""
    expect_refusal(_bwd_layerscale(_ptrs("ivb_rmsnorm_bwd_layerscale", **{operand: A + 4}), {}),
                   "weight and gamma 8-byte aligned")


@cpu_only
@pytest.mark.parametrize("operand", ["video", "cols"])
def test_im2col_video_cols_need_4_bytes(operand):
    """im2col_visible reads and writes 2 bf16 at a time: a view starting at an odd element is refused."""
    expect_refusal(_im2col(_ptrs("ivb_im2col_visible", **{operand: A + 2}), {}),
                   "video and cols must be 4-byte aligned")


# the refusal text of each entry point's pitch check (default: the norm and loss kernels')
PITCH_TEXT = {"ivb_gather_add": "src_bstride and out_bstride must be multiples of 8",
              "ivb_scatter_add": "g_bstride must be a multiple of 8"}


@cpu_only
@pytest.mark.parametrize("entry,pitch", [("ivb_norm_bwd", "lddx_in"), ("ivb_norm_bwd", "lddx"),
                                         ("ivb_ln_l2_fwd", "ldo"), ("ivb_ln_l2_fwd", "ldt"),
                                         ("ivb_layerscale_bwd", "ldy"), ("ivb_layerscale_bwd", "lddx"),
                                         ("ivb_norm_fwd", "ldx"), ("ivb_colsum_bf16", "ldx"),
                                         ("ivb_gather_add", "src_bstride"), ("ivb_gather_add", "out_bstride"),
                                         ("ivb_scatter_add", "g_bstride")])
@pytest.mark.parametrize("bad", [D + 4, D + 1])
def test_bad_pitch_refused(entry, pitch, bad):
    call = ENTRIES[entry][0]
    expect_refusal(call(_ptrs(entry), {pitch: bad}), f"{entry}: ")
    assert PITCH_TEXT.get(entry, "/ld must be multiples of 8") in _lib.load().ivb_last_error().decode()


def test_empty_is_a_noop():
    """M = 0 returns 0 before any check or CUDA call."""
    lib = _lib.load()
    assert lib.ivb_norm_fwd(None, 1, 3, None, None, 1e-6, 0, 0, 12, None, 3, None, None, None) == 0
    assert lib.ivb_norm_bwd(None, 3, None, 1, 3, None, None, None, 0, 0, 12, None, 3, None, 1, 3, None, None, None) == 0
    assert lib.ivb_layerscale_bwd(None, 3, None, 3, None, 0, 12, None, 3, None, None, None, None) == 0
    assert lib.ivb_ln_l2_fwd(None, 3, None, None, 1e-5, 0, 12, None, 3, None, None, 0, 3, None, None) == 0
    assert lib.ivb_gather_add(None, 3, None, None, 0, 0, 0, 5, 12, None, 1, 3, None) == 0
    assert lib.ivb_scatter_add(None, 1, 3, None, 0, 0, 0, 5, 12, None, None) == 0
