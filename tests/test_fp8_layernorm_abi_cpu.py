"""FP8 for the LayerNorm towers (InternVideo1's VideoMAE, the MobileCLIP text tower, the stage-2 BERT text layers)
without a GPU.

1. The switches: set_fp8 counts the VideoMAEBlocks and text_modules.TransformerEncoder blocks with the RMSNorm Blocks in
   every scaling, set_fp8_inference also counts BERT's text layers (not its fusion layers), and each class's precision
   comes from modules.block_precision; switching off gives ops.BF16 back.
2. The exclusion rules hold for the new classes as for Block: set_fp8_inference refuses a block in FP8 training mode,
   a block with both switches on refuses to run, FP8 inference refuses a forward that needs a gradient, the
   VideoMAEv2 teacher's head-axis attention and the text tower's causal attention never take the FP8 attention.
3. Every FP8 call these towers make at their recipe shapes passes the C ABI's argument checks: each is called with
   fake device addresses and one argument broken that is checked after every shape rule, so the refusal names that
   argument (and the call never reaches a launch: run only where no CUDA device is visible).
"""
import pytest
import torch

from abi_fake import BASE, cpu_only, expect_refusal
from internvideo_b200 import _lib, ops
from internvideo_b200 import modules as M
from internvideo_b200 import videomae_v1 as v1
from internvideo_b200.bert_modules import BERT_LARGE, BertModel
from internvideo_b200.text_modules import MOBILECLIP_B, TextTransformer, TransformerEncoder

MODES = {"tensor": (dict(scaling="tensor"), ops.FP8_TENSOR), "token": (dict(scaling="token"), ops.FP8_TOKEN),
         "token_wgrad": (dict(scaling="token", wgrad=True), ops.FP8_TOKEN_WGRAD)}


def _iv1():
    return v1.PretrainVisionTransformer(encoder_embed_dim=64, encoder_depth=3, encoder_num_heads=2, decoder_embed_dim=32,
                                        decoder_depth=2, decoder_num_heads=2, decoder_num_classes=1536, qkv_bias=True,
                                        init_values=0.1, img_size=32, patch_size=16)


def _text(layers=3):
    return TextTransformer(dict(MOBILECLIP_B, dim=64, n_heads_per_layer=2, n_transformer_layers=layers,
                                vocab_size=100, context_length=8), 32)


def _bert():
    return BertModel(dict(BERT_LARGE, hidden_size=64, num_attention_heads=2, intermediate_size=128,
                          num_hidden_layers=4, fusion_layer=3, vocab_size=100, max_position_embeddings=16))


# ------------------------------------------------------------------------------------------------ 1. the switches
@pytest.mark.parametrize("mode", sorted(MODES))
def test_set_fp8_counts_and_precision(mode):
    kw, prec = MODES[mode]
    for model, blocks in ((_iv1(), 5), (_text(), 3)):
        assert M.set_fp8(model, True, **kw) == blocks
        fused = [m for m in model.modules() if isinstance(m, M.Fp8Block)]
        assert len(fused) == blocks
        assert all(M.block_precision(b, True) == prec and M.block_precision(b) == prec for b in fused)
        assert all(b._spec(2, 8, **({"causal": True} if isinstance(b, TransformerEncoder) else {}),
                           training=True).precision == prec for b in fused)
        assert M.set_fp8(model, False) == blocks
        assert all(M.block_precision(b, True) == ops.BF16 for b in fused)
    assert M.set_fp8(_bert(), True, **kw) == 0               # BERT has no training path
    # a model holding every tower: all of its fused blocks
    both = torch.nn.ModuleList([_iv1(), _text(2), M.Block(64, 2, 4.0)])
    assert M.set_fp8(both, True, **kw) == 5 + 2 + 1


def test_a_refused_scaling_changes_nothing():
    for model in (_iv1(), _text()):
        for kw in (dict(scaling="tensor", wgrad=True), dict(wgrad=True)):
            with pytest.raises(ValueError, match="wgrad=True needs scaling='token'"):
                M.set_fp8(model, True, **kw)
        with pytest.raises(ValueError, match="scaling must be one of"):
            M.set_fp8(model, True, scaling="block")
        assert all(M.block_precision(b, True) == ops.BF16 for b in model.modules() if isinstance(b, M.Fp8Block))


def test_set_fp8_inference_counts():
    """Off by default; switching on counts the fused blocks and BERT's text layers and quantises their weights (CPU
    tensors cannot be cast, so the counts are taken on the switch's selection alone)."""
    iv1, text, bert = _iv1(), _text(), _bert()
    sel = lambda m: [x for x in m.modules() if isinstance(x, M.Fp8InferenceSwitch) and x._fp8_linears()]  # noqa: E731
    assert len(sel(iv1)) == 5 and len(sel(text)) == 3 and len(sel(bert)) == 3
    assert all(x.fp8_inference is None and not x.fp8_attention for m in (iv1, text, bert) for x in sel(m))
    assert bert.encoder.layer[3]._fp8_linears() == ()        # the fusion layer: never run in text mode
    assert len(bert.encoder.layer[0]._fp8_linears()) == 6
    a, ffn = text.transformer[0].pre_norm_mha[1], text.transformer[0].pre_norm_ffn
    assert text.transformer[0]._fp8_linears() == (a.qkv_proj, a.out_proj, ffn[1], ffn[4])
    for m in (iv1, text, bert):                               # switching off needs no device
        assert M.set_fp8_inference(m, False) == len(sel(m))


# ------------------------------------------------------------------------------------------------ 2. exclusion rules
class _Weights:
    """A stand-in for Fp8InferenceWeights (whose casts need a GPU): get() returns four marker copies."""
    def get(self):
        return tuple((i, i) for i in range(4))


@pytest.mark.parametrize("make", [lambda: _iv1().encoder.blocks[0], lambda: _text().transformer[0]],
                         ids=["VideoMAEBlock", "TransformerEncoder"])
def test_the_two_switches_exclude_each_other(make):
    blk = make()
    M.set_fp8(blk, True, scaling="token")
    with pytest.raises(_lib.IvbError, match="switch that off first"):
        M.set_fp8_inference(blk)
    assert blk.fp8_inference is None
    blk.fp8_inference = _Weights()                            # set_fp8_inference's state, then set_fp8 on top
    with pytest.raises(_lib.IvbError, match="both on"):
        M.block_precision(blk)
    M.set_fp8(blk, False)
    assert M.block_precision(blk) == _Weights().get()
    with pytest.raises(_lib.IvbError, match="has no gradient"):
        M.block_precision(blk, training=True)


def test_fp8_inference_refuses_a_gradient_and_keeps_causal_and_head_axis_attention():
    enc = _text().transformer[0]
    enc.fp8_inference, enc.fp8_attention = _Weights(), True
    with pytest.raises(_lib.IvbError, match="has no gradient"):
        enc._spec(2, 8, True, training=True)
    assert not enc._spec(2, 8, True).attn_fp8                 # causal attention stays bf16
    assert enc._spec(2, 8, False).attn_fp8                    # a non-causal text tower takes the FP8 attention
    blk = _iv1().encoder.blocks[0]
    blk.fp8_inference, blk.fp8_attention = _Weights(), True
    assert blk._spec(2, 8).attn_fp8 and not blk._spec(2, 8, head_axis=True).attn_fp8
    M.set_fp8(blk, True, scaling="token")                     # FP8 training never takes the FP8 attention
    blk.fp8_inference = None
    assert not blk._spec(2, 8, training=True).attn_fp8 and not blk._spec(2, 8, head_axis=True).attn_fp8


# ------------------------------------------------------------------------------------------------ 3. recipe shapes
def _pad16(n):
    return (n + 15) // 16 * 16


# (tower, tokens M, width D, MLP width, set_fp8 trains it): the shapes of the tools/ln_fp8_table.py workloads
TOWERS = [
    ("iv1_base_encoder", 32 * 157, 768, 3072, True), ("iv1_base_decoder", 32 * 1568, 384, 1536, True),
    ("iv1_large_encoder", 32 * 157, 1024, 4096, True), ("iv1_large_decoder", 32 * 1568, 512, 2048, True),
    ("mobileclip_b_text", 128 * 77, 512, 2048, True), ("bert_large_text", 1024 * 40, 1024, 4096, False),
]
A, W, Q, S, R = BASE, BASE + 0x1000000, BASE + 0x2000000, BASE + 0x3000000, BASE + 0x4000000


def _gemm_fp8(M_, N, K, epi, flags=0, out1=False, aux=False, bias=True, gamma=False):
    """Every rule of ivb_gemm_fp8 passes; the tile_n 64 checked last is what is refused."""
    ld0 = N
    return _lib.load().ivb_gemm_fp8(A, 0, _pad16(K), 0, S, W, 0, _pad16(K), S + 0x100000, M_, N, K, epi,
                                    flags | 64, Q, ld0, Q + 0x4000000 if out1 else None, N,
                                    R if bias else None, R + 0x10000 if gamma else None,
                                    R + 0x100000 if aux else None, N, None, 64, None)


@cpu_only
@pytest.mark.parametrize("tower, Mt, D, Hd, trains", TOWERS, ids=[t[0] for t in TOWERS])
def test_recipe_shapes_pass_every_argument_check(tower, Mt, D, Hd, trains):
    lib = _lib.load()
    tile = "ivb_gemm_fp8: tile_n must be 0, 128 or 192"
    # the norms: E4M3 rows (inference) and E4M3 + bf16 rows with statistics (training; BERT's post-LN norms)
    for x_f32 in (1, 0):
        expect_refusal(lib.ivb_norm_fwd_fp8(A, x_f32, D, W, W + 0x10000, 1e-6, 1, Mt, D, Q, _pad16(D), S + 2, None),
                       "ivb_norm_fwd_fp8: row_scale_inv must be 4-byte aligned")
        expect_refusal(lib.ivb_norm_fwd_fp8_train(A, x_f32, D, W, W + 0x10000, 1e-6, 1, Mt, D, Q, _pad16(D), S, R, D,
                                                  S + 0x100000, S + 0x200002, None),
                       "ivb_norm_fwd_fp8_train: row_scale_inv, mean and rstd must be 4-byte aligned")
    # the four forward GEMMs with their epilogues: qkv (bias), proj (residual, gamma), fc1 (GELU), fc2 (residual)
    expect_refusal(_gemm_fp8(Mt, 3 * D, D, 0), tile)
    expect_refusal(_gemm_fp8(Mt, D, D, 3, out1=True, aux=True, gamma=True), tile)
    expect_refusal(_gemm_fp8(Mt, Hd, D, 2, out1=True), tile)
    expect_refusal(_gemm_fp8(Mt, D, Hd, 3, out1=True, aux=True, gamma=True), tile)
    # the row casts of a and g (and of the gradients), and the per-channel weight casts
    for K in (D, Hd, 3 * D):
        expect_refusal(lib.ivb_fp8_quantize_rows(A, K, Mt, K, Q, _pad16(K), S + 2, None),
                       "ivb_fp8_quantize_rows: row_scale_inv must be 4-byte aligned")
    for N, K in ((3 * D, D), (D, D), (Hd, D), (D, Hd)):
        expect_refusal(lib.ivb_fp8_quantize_rows(A, K, N, K, Q, _pad16(K), S + 2, None),
                       "ivb_fp8_quantize_rows: row_scale_inv must be 4-byte aligned")
        expect_refusal(lib.ivb_fp8_quantize_cols_t(A, K, N, K, Q, _pad16(N), S, S + 0x100002, None),
                       "ivb_fp8_quantize_cols_t: col_amax and col_scale_inv must be 4-byte aligned")
    if not trains:
        # BERT: the three N = D qkv GEMMs with bias, the two residual sums accumulated in place in bf16
        expect_refusal(_gemm_fp8(Mt, D, D, 0), tile)
        expect_refusal(_gemm_fp8(Mt, D, D, 0, flags=2), tile)
        expect_refusal(_gemm_fp8(Mt, D, Hd, 0, flags=2), tile)
        return
    # the input-gradient GEMMs: dh (GELU' epilogue), dn2, da, dn1
    expect_refusal(_gemm_fp8(Mt, Hd, D, 4, aux=True, bias=False), tile)
    for N, K in ((D, Hd), (D, D), (D, 3 * D)):
        expect_refusal(_gemm_fp8(Mt, N, K, 0, bias=False), tile)
    # the FP8 weight gradients: the block-scaled transposing casts and the wgrad GEMM over the Mt tokens
    nkb = (Mt + 127) // 128
    for C in (D, Hd, 3 * D):
        expect_refusal(lib.ivb_fp8_quantize_blocks_t(A, C, Mt, C, Q, _pad16(Mt), S + 2, None),
                       "ivb_fp8_quantize_blocks_t: scale_inv and rowscale must be 4-byte aligned")
    for Mo, No in ((3 * D, D), (D, D), (Hd, D), (D, Hd)):
        expect_refusal(lib.ivb_gemm_fp8_wgrad(A, _pad16(Mt), S, W, _pad16(Mt), S + 16 * nkb * Mo, Mo, No, Mt, 1, 2,
                                              Q + 8, No, None, None),
                       "ivb_gemm_fp8_wgrad: out0 must be 16-byte aligned")
