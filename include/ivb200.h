/* ivb200.h — C ABI of libivb200.so: the H100 (sm_90a) compute path for InternVideo2 pre-training.
 *
 * The reference (OpenGVLab/InternVideo) has no FFI of its own: its "operator interface" for this
 * path is the nn.Module surface of
 *   InternVideo2/single_modality/models/internvideo2_pretrain.py   (PatchEmbed :300, RMSNorm :117,
 *     LayerScale :131, Attention :149, Mlp :220, Block :247, Linear_Decoder :334, MLP_Decoder :368,
 *     PretrainInternVideo2.forward :629)
 *   InternVideo2/single_modality/models/flash_attention_class.py:27   (FlashAttention.forward)
 *   InternVideo2/multi_modality/models/criterions.py:15,65,200        (get_sim, vtc_loss, get_mask)
 *   InternVideo2/multi_modality/models/utils.py:193                   (AllGather)
 *   InternVideo1/Pretrain/VideoMAE/engine_for_pretraining.py:66-106   (pixel target + MSE)
 * and the third-party kernels those modules call (cuBLAS Linear, cuDNN Conv3d, FA2
 * flash_attn_varlen_qkvpacked_func / fused_dense / dropout_layer_norm).  Each entry point below
 * names the reference call it stands in for.  internvideo_b200/ops.py binds these with ctypes and
 * wraps them in torch.autograd.Function; INTEGRATION.md shows the stub a maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; tensors are row-major;
 *     "ld" arguments are row pitches in ELEMENTS; bf16 = __nv_bfloat16 bit pattern.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream).
 *   - return value: 0 = ok, non-zero = error; ivb_last_error() returns the text.  No exceptions
 *     cross this boundary.  The library allocates nothing persistent; all buffers are borrowed.
 *   - there is no CPU fallback: without a CUDA device of compute capability 9.0 every compute
 *     entry point returns an error.
 *   - parameter gradients (ivb_norm_bwd, ivb_rmsnorm_pair_bwd, ivb_rmsnorm_bwd_layerscale, ivb_layerscale_bwd,
 *     ivb_colsum_bf16, ivb_ln_l2_bwd, ivb_prenorm_wgrad), the losses (ivb_ln_l2_fwd with a target, ivb_vtc_loss_fwd, ivb_mse_loss) and
 *     dtemp (ivb_vtc_loss_bwd) are summed in a fixed order through a per-device scratch of the library, so the same
 *     inputs give the same bits on every run.  That scratch holds one reduction at a time: these entry points must
 *     not be called concurrently from two streams of the same device (the package runs them on one compute stream).
 *   - the row kernels (ivb_norm_fwd, ivb_norm_bwd, ivb_rmsnorm_pair_*, ivb_rmsnorm_bwd_layerscale, ivb_layerscale_bwd,
 *     ivb_colsum_bf16, ivb_ln_l2_*, ivb_l2norm_rows_*, ivb_pool_attn_*, ivb_gather_add, ivb_scatter_add) move each row
 *     in 16-byte vectors: the row width and every pitch (and clip stride) are multiples of 8 elements (the fp32
 *     pitches of ivb_rmsnorm_bwd_layerscale: of 4), and every row or vector operand is 16-byte aligned (weight and
 *     gamma of ivb_rmsnorm_bwd_layerscale: 8-byte).  ivb_im2col_visible moves 4-byte words: video and cols are 4-byte
 *     aligned.  Per-row and per-column scalars (mean, rstd, stats, parameter gradients) and index lists need only
 *     their type's alignment.  A call that breaks one of these rules is refused before any CUDA call.
 */
#ifndef IVB200_H_
#define IVB200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define IVB_VERSION 100

/* GEMM epilogues (ivb_gemm_bf16) */
#define IVB_EPI_BF16 0      /* out0(bf16) = acc (+bias) (+out0 if IVB_FLAG_ACCUM)                  */
#define IVB_EPI_F32 1       /* out0(f32)  = acc (+bias) (+out0 if IVB_FLAG_ACCUM)                  */
#define IVB_EPI_BIAS_GELU 2 /* h = acc+bias; out1(bf16)=h (opt); out0(bf16)=gelu(h)                */
#define IVB_EPI_RESID 3     /* y = acc+bias; out1(bf16)=y (opt); out0(f32)=aux(f32)+rowscale[m]*gamma*y
                               (rowscale: optional fp32 [M], the per-sample DropPath keep/scale factor) */
#define IVB_EPI_GELU_BWD 4  /* out0(bf16) = acc * gelu'(aux(bf16))                                 */
#define IVB_EPI_SWIGLU 5    /* LLaMA's SwiGLU MLP: B = [gate; up], one K-major bf16 [N = 2I, K] operand (rows [0, I)
                               the gate weight, [I, 2I) the up weight; I a multiple of 8); out0(bf16) [M, I] (pitch ld0)
                               = silu(x gate^T) * (x up^T), both products from the fp32 accumulators, one rounding.
                               The kernels load B's rows interleaved in groups of 8 (gate 8g..8g+7, then up 8g..8g+7)
                               through a 4-D TMA map: no copy of the weight.  Single-CTA bf16 kernels only (cooperative
                               or ping-pong, any tile_n); refused: an MN-major B, bias, out1, IVB_FLAG_ACCUM,
                               IVB_FLAG_2CTA, a DropPath plan, and FP8 (ivb_gemm_fp8).                                */

#define IVB_FLAG_GELU_TANH 1 /* tanh-approx GELU (FA2 FusedMLP) instead of erf (nn.GELU)           */
/* IVB_FLAG_GELU_QUICK (128, below): QuickGELU x * sigmoid(1.702 x) (OpenAI-CLIP blocks, ViCLIP) instead of erf; for
   IVB_EPI_BIAS_GELU and IVB_EPI_GELU_BWD, with or without IVB_FLAG_GELU_SAVE_GRAD.  Excludes IVB_FLAG_GELU_TANH.  */
#define IVB_FLAG_ACCUM 2     /* accumulate into out0                                               */
#define IVB_FLAG_1CTA 4      /* force the cooperative single-CTA kernel (128-row tiles, both MMA warpgroups on one tile) */
#define IVB_FLAG_2CTA 8      /* force the CTA-pair kernel (cluster of 2, 256-row tiles, B tile TMA-multicast)     */
#define IVB_FLAG_GELU_SAVE_GRAD 16 /* EPI_BIAS_GELU: out1 receives gelu'(h) instead of h; EPI_GELU_BWD: aux IS
                                     that saved derivative (out0 = acc * aux) — the backward epilogue then has
                                     no transcendental work (the training path; h itself is never needed)   */
#define IVB_FLAG_PINGPONG 32 /* force the ping-pong kernel (one 128 x 128 tile per MMA warpgroup, each tile's epilogue
                                under the other warpgroup's MMAs); tile_n must be 0 or 128.  For tests and tools:
                                the library picks ping-pong or cooperative by itself                                 */

/* ---- status ---------------------------------------------------------------------------------- */
const char* ivb_last_error(void);
int ivb_version(void);
/* 0 if the current CUDA device can run this library (compute capability 9.0), else error. */
int ivb_device_check(void);
/* number of kernels this library has launched since the last reset (bench.py "gpu_launches"). */
long ivb_launch_count(void);
void ivb_reset_launch_count(void);

/* ---- wgmma GEMM -------------------------------------------------------------------------------
 * D[M,N] = epilogue( sum_k A(m,k) * B(n,k) ), bf16 operands, fp32 accumulate.
 *   a_mn_major = 0: A is stored [M,K] row-major (pitch lda);  1: stored [K,M] row-major.
 *   b_mn_major = 0: B is stored [N,K] row-major (pitch ldb);  1: stored [K,N] row-major.
 * Supported (A,B) majors: (0,0) forward y = x W^T; (0,1) dgrad dx = dy W; (1,1) wgrad dW = dy^T x.
 * Stands in for nn.Linear / F.linear (cuBLAS) at internvideo2_pretrain.py:61-77,195,211,239-242,
 * 356,394 and FA2 fused_dense (FusedMLP :269).  tile_n: 0 = auto, or one of 128/176/192/256.
 * The fused epilogue moves every row of out0 / out1 / aux and the bias / gamma vectors in 16-byte vectors, so:
 * N, lda, ldb, ld0 and (when out1 is given) ld1 are multiples of 8 elements; ldaux (when aux is given) is a multiple
 * of 8 bf16 elements, or of 4 for the fp32 aux of IVB_EPI_RESID; out0, out1, aux, bias and gamma are 16-byte aligned.
 * A call that breaks one of these rules is refused before any CUDA call.                          */
/* process-wide default for problems with M >= 512: 1 = CTA-pair kernel, 0 = single-CTA kernel. */
void ivb_set_default_2cta(int enable);
int ivb_gemm_bf16(const void* A, int a_mn_major, long lda, const void* B, int b_mn_major, long ldb,
                  int M, int N, int K, int epilogue, int flags, void* out0, long ld0, void* out1,
                  long ld1, const void* bias, const void* gamma, const void* aux, long ldaux,
                  const float* rowscale, int tile_n, void* stream);

/* ---- DropPath plans (stochastic depth: skip the work of the rows a draw drops) ----------------------------------
 * ivb_droppath_plan: for each of `branches` rows b of DropPath factors rowscale [branches, M] (pitch ld_rs >= M; the
 * EPI_RESID rowscale of one block branch each), writes the int32 plan [b, 0 .. ivb_droppath_plan_ints(M)) (pitch
 * ld_plan): a row is live when its factor is not 0, a 128-row tile or 64-row k-block when one of its rows is.
 *   plan[0 .. nm)               the nm = ceil(M/128) row tiles: the live ones ascending, then the dead ones ascending
 *   plan[nm]                    the number of live row tiles                         (plan + 0: the M plan)
 *   plan[nm+1 .. nm+1+c)        the c live k-blocks of the nk = ceil(M/64), ascending
 *   plan[nm+1+nk]               c                                                    (plan + nm + 1: the K plan)
 * One stream-ordered kernel; nothing is read by the host, so it is capturable in a CUDA graph.
 * ivb_gemm_bf16_plan: ivb_gemm_bf16 with an M plan over its M rows and / or a K plan over its K (either may be NULL:
 * ivb_gemm_bf16 itself).  The results are those of ivb_gemm_bf16 wherever a plan's dead rows hold DropPath factor 0:
 *   M plan: a dead row tile runs no MMA.  Its rows get IVB_EPI_RESID out0 = aux (with rowscale 0 the sum is the
 *     residual itself) and out1 = 0; every other epilogue writes 0 (IVB_EPI_GELU_BWD does not read aux).  Live tiles are
 *     computed as ivb_gemm_bf16 computes them.  Not with IVB_FLAG_ACCUM.
 *   K plan (A and B MN-major, the weight gradient over tokens): only the listed k-blocks are summed, in ascending order,
 *     so when the left-out rows of dy are zero the result has ivb_gemm_bf16's bits; with none listed the sum is 0.
 *     Epilogue IVB_EPI_BF16 or IVB_EPI_F32 (IVB_FLAG_ACCUM allowed), no bias.
 * A plan runs on the single-CTA kernels: IVB_FLAG_2CTA is refused, the ivb_set_default_2cta default does not apply.
 * The per-token FP8 GEMM takes an M plan (ivb_gemm_fp8_plan), and attention the factors themselves (ivb_attn_fwd_plan,
 * ivb_attn_bwd_plan).                                                                                       */
long ivb_droppath_plan_ints(int M);
int ivb_droppath_plan(const float* rowscale, long ld_rs, int branches, int M, int* plan, long ld_plan, void* stream);
int ivb_gemm_bf16_plan(const void* A, int a_mn_major, long lda, const void* B, int b_mn_major, long ldb,
                       int M, int N, int K, int epilogue, int flags, void* out0, long ld0, void* out1,
                       long ld1, const void* bias, const void* gamma, const void* aux, long ldaux,
                       const float* rowscale, int tile_n, const int* m_plan, const int* k_plan, void* stream);

/* ---- FP8 (opt-in FP8 mode of the ViT block) ---------------------------------------------------
 * Formats: IVB_FP8_E4M3 (4 exponent, 3 mantissa bits, max 448: activations and weights) and IVB_FP8_E5M2 (max 57 344:
 * gradients).  Per-tensor current scaling: the scale comes from the tensor's own amax in the same call.
 *
 * ivb_fp8_quantize: x bf16 [M, K] (pitch ldx, a multiple of 8) ->
 *   *amax      = max |x| (fp32, device; exact: the max of the bf16 magnitudes, the same bits on every run)
 *   scale      = 2^floor(log2(fmax / amax)), fmax = 448 or 57 344; 1 when amax = 0 (exponent clamped to [-126, 126])
 *   out        = round-to-nearest-even(x * scale) in `format`, [M, K] row-major, pitch ldo (a multiple of 16)
 *   out_t      = out^T, [K, M] row-major, pitch ldt (a multiple of 16), optional (NULL: not written)
 *   *scale_inv = 1 / scale (fp32, device), or NaN when amax is Inf or NaN, so that a GEMM reading it gives NaN
 * amax and scale_inv are device floats; amax is also the kernels' workspace (the call zeroes it first).  Columns
 * K .. ldo of out (and M .. ldt of out_t) are not written.  x, out, out_t are 16-byte aligned.  Three stream-ordered
 * operations (a 4-byte memset and two kernels); capturable in a CUDA graph.                          */
#define IVB_FP8_E4M3 0
#define IVB_FP8_E5M2 1
int ivb_fp8_quantize(const void* x, long ldx, int M, int K, int format, void* out, long ldo, void* out_t, long ldt,
                     float* amax, float* scale_inv, void* stream);
/* D[M,N] = epilogue( a_scale_inv * b_scale_inv * sum_k A(m,k) * B(n,k) ), fp8 operands, fp32 accumulate.
 * A: [M,K] row-major in a_format (E4M3 or E5M2); B: [N,K] row-major, E4M3.  Both operands K-major (a_mn_major =
 * b_mn_major = 0; fp8 wgmma has no transposed form): y = x W^T takes W's E4M3 copy, dx = dy W takes the E4M3 copy of W^T
 * (ivb_fp8_quantize's out_t).  lda, ldb: multiples of 16 elements.  a_scale_inv / b_scale_inv: device fp32 scalars
 * (ivb_fp8_quantize's), read by the kernel, never by the host.  Epilogue, flags and their operand rules as for
 * ivb_gemm_bf16, except: no IVB_FLAG_2CTA; tile_n is 0 (auto), 128 or 192.  IVB_FLAG_PINGPONG forces the ping-pong
 * kernel, which accumulates in the tensor core; IVB_FLAG_1CTA forces the cooperative kernel, which adds each 128-element
 * k-block's partial sum to an fp32 accumulator on the CUDA cores.  By default the library picks between them as
 * ivb_gemm_bf16 picks between its ping-pong and cooperative kernels.  A call that breaks one of these rules is refused
 * before any CUDA call.                                                                            */
int ivb_gemm_fp8(const void* A, int a_mn_major, long lda, int a_format, const float* a_scale_inv, const void* B,
                 int b_mn_major, long ldb, const float* b_scale_inv, int M, int N, int K, int epilogue, int flags,
                 void* out0, long ld0, void* out1, long ld1, const void* bias, const void* gamma, const void* aux,
                 long ldaux, const float* rowscale, int tile_n, void* stream);

/* ---- FP8 with per-row scales (FP8 inference of frozen towers) ----------------------------------
 * Each row gets its own power-of-two scale, chosen from the row's amax by the ivb_fp8_quantize rule (E4M3, fmax 448):
 *   scale_r = 2^floor(log2(448 / amax_r)); 1 when amax_r = 0; row_scale_inv[r] = 1 / scale_r, or NaN when the row
 *   holds an Inf or NaN.  out[r, :] = round-to-nearest-even(row * scale_r) in E4M3.
 * Dequantisation (q * scale_inv) is exact, and a row's grid refines the whole tensor's, so no element's cast error
 * exceeds the per-tensor cast's.  The same bits on every run (no atomics).  One stream-ordered kernel per call;
 * capturable in a CUDA graph.  Columns D (or K) .. ldo of out are not written.  A call that breaks a rule below is
 * refused before any CUDA call.
 *
 * ivb_fp8_quantize_rows: x bf16 [M, K] (pitch ldx, a multiple of 8; K <= IVB_FP8_ROWS_MAX_K) -> out E4M3 [M, K]
 *   (pitch ldo, a multiple of 16) and row_scale_inv fp32 [M].  Weights take it with rows = output channels (the
 *   per-channel scales of the GEMM's B operand).  x and out are 16-byte aligned.
 * ivb_norm_fwd_fp8: y = norm(x) * weight (+ bias) as ivb_norm_fwd computes it (fp32 statistics; x fp32 or bf16,
 *   pitch ldx a multiple of 8), written only as E4M3 [M, D] (pitch ldo, a multiple of 16) plus row_scale_inv [M]: each
 *   row is read once and no bf16 copy is written.  D a multiple of 8, D <= IVB_NORM_FP8_MAX_D.  x, weight, bias and
 *   out are 16-byte aligned.
 * ivb_gemm_fp8 with IVB_FLAG_FP8_VECTOR_SCALES: a_scale_inv points at M floats and b_scale_inv at N floats, and the
 *   accumulator (m, n) is multiplied by a_scale_inv[m] * b_scale_inv[n] before the epilogue.  A must be E4M3 and both
 *   vectors 8-byte aligned; the flag with IVB_FLAG_2CTA or a null vector is refused.                                              */
#define IVB_FLAG_FP8_VECTOR_SCALES 64
#define IVB_FLAG_GELU_QUICK 128   /* QuickGELU in the GELU epilogues (documented beside IVB_FLAG_GELU_TANH) */
#define IVB_FP8_ROWS_MAX_K 16384
#define IVB_NORM_FP8_MAX_D 4096
int ivb_fp8_quantize_rows(const void* x, long ldx, int M, int K, void* out, long ldo, float* row_scale_inv,
                          void* stream);
int ivb_norm_fwd_fp8(const void* x, int x_is_f32, long ldx, const void* weight, const void* bias, float eps,
                     int is_layernorm, int M, int D, void* out, long ldo, float* row_scale_inv, void* stream);

/* ---- FP8 training with per-token scales (opt-in per-token FP8 mode of the ViT block) ---------------------------
 * Activations and gradients are cast row by row (ivb_fp8_quantize_rows, E4M3 for both), weights with one scale per
 * output channel for the forward and one per input channel for the input-gradient GEMM; every scale follows the
 * ivb_fp8_quantize_rows rule for its row or column.  Same bits on every run; capturable in a CUDA graph.  A call that
 * breaks a rule below is refused before any CUDA call.
 *
 * ivb_norm_fwd_fp8_train: ivb_norm_fwd_fp8 (same operand rules, same out and row_scale_inv bits) that also writes, from
 *   the same single read of each row, the bf16 row y [M, D] (pitch ldy, a multiple of 8; 16-byte aligned), rstd [M]
 *   and, for LayerNorm, mean [M]: the bits ivb_norm_fwd writes.  y, rstd and (LayerNorm) mean are required; mean,
 *   rstd and row_scale_inv are 4-byte aligned.  One stream-ordered kernel.
 * ivb_fp8_quantize_cols_t: x bf16 [M, K] (pitch ldx, a multiple of 8; a weight [N_out, K_in]) -> out_t E4M3 [K, M]
 *   = (x * col_scale)^T (pitch ldt, a multiple of 16 and >= M) and col_scale_inv fp32 [K], one power-of-two scale per
 *   column of x from the column's amax (NaN when the column holds an Inf or NaN).  out_t is the B operand of the
 *   input-gradient GEMM dx = dy W with IVB_FLAG_FP8_VECTOR_SCALES, col_scale_inv its per-output-channel vector.
 *   col_amax fp32 [K] is the call's workspace (zeroed first; afterwards the columns' amax).  x and out_t are 16-byte
 *   aligned, col_amax and col_scale_inv 4-byte.  Columns M .. ldt of out_t are not written.  Three stream-ordered
 *   operations (a memset of col_amax and two kernels).                                                             */
int ivb_norm_fwd_fp8_train(const void* x, int x_is_f32, long ldx, const void* weight, const void* bias, float eps,
                           int is_layernorm, int M, int D, void* out, long ldo, float* row_scale_inv, void* y, long ldy,
                           float* mean, float* rstd, void* stream);
int ivb_fp8_quantize_cols_t(const void* x, long ldx, int M, int K, void* out_t, long ldt, float* col_amax,
                            float* col_scale_inv, void* stream);
/* ivb_gemm_fp8_plan: ivb_gemm_fp8 with the M plan of a DropPath plan over its M rows (ivb_droppath_plan; NULL:
 *   ivb_gemm_fp8 itself), with ivb_gemm_bf16_plan's M-plan rules: a dead row tile loads nothing and runs no MMA, its
 *   rows get IVB_EPI_RESID out0 = aux and out1 = 0 and every other epilogue writes 0; live tiles get ivb_gemm_fp8's
 *   values, on the kernel form it would pick (the cooperative one at tile_n 128: tile_n 192 is refused).  A plan needs
 *   IVB_FLAG_FP8_VECTOR_SCALES (per-row scales are untouched by the other rows' values; a per-tensor scale is not) and
 *   excludes IVB_FLAG_ACCUM.                                                                                      */
int ivb_gemm_fp8_plan(const void* A, int a_mn_major, long lda, int a_format, const float* a_scale_inv, const void* B,
                      int b_mn_major, long ldb, const float* b_scale_inv, int M, int N, int K, int epilogue, int flags,
                      void* out0, long ld0, void* out1, long ld1, const void* bias, const void* gamma, const void* aux,
                      long ldaux, const float* rowscale, int tile_n, const int* m_plan, void* stream);

/* ---- FP8 weight gradients with per-(128-token block, channel) scales (set_fp8 with wgrad=True) -------------------
 * The weight gradient dW = dy^T act sums over tokens, so per-token scales cannot be factored out of it, and fp8 wgmma
 * reads only K-major operands.  Both operands are therefore cast transposed, with one power-of-two scale per channel
 * per 128-token block (the DeepSeek-V3 technical report's 1 x 128 tiles, 3.3), and the GEMM applies the scales of each
 * 128-token k-block as it adds that k-block's partial sum to its fp32 accumulator.  Same bits on every run; capturable
 * in a CUDA graph.  A call that breaks a rule below is refused before any CUDA call.
 *
 * ivb_fp8_quantize_blocks_t: x bf16 [M, C] (M tokens; pitch ldx, a multiple of 8; C a multiple of 8) -> out_t E4M3
 *   [C, M] (pitch ldt, a multiple of 16 and >= M; row c holds channel c over all tokens) and scale_inv fp32
 *   [ceil(M/128), C] (block-major: one k-block's scales are contiguous).  Block b's scale of channel c follows the
 *   ivb_fp8_quantize_rows rule on amax(|x[128b : 128b + 128, c]|) (the last block may be partial: its own rows): a
 *   power of two, 1 when the amax is 0, scale_inv NaN when the block holds an Inf or NaN.  Columns M .. ldt of out_t
 *   are not written.  x and out_t are 16-byte aligned, scale_inv 4-byte.  One stream-ordered kernel.
 * ivb_fp8_quantize_blocks_t_plan: the same with the DropPath factors rowscale fp32 [M] of the branch (required): a
 *   token whose factor is 0 is cast as 0.  Its gradient row is 0, so it adds nothing to the weight gradient, and with
 *   it zeroed no scale depends on values a DropPath plan may or may not have computed (ivb_attn_fwd_plan writes 0 where
 *   ivb_attn_fwd writes the attention output).
 * ivb_gemm_fp8_wgrad: out0[M, N] = sum_kb sum_{k in kb} A_t[m, k] B_t[n, k] * a_scale_inv[kb, m] * b_scale_inv[kb, n]
 *   (+ out0 under IVB_FLAG_ACCUM) over the 128-element k-blocks kb.  A_t: E4M3 [M, K] (dy^T; pitch lda), B_t: E4M3
 *   [N, K] (act^T; pitch ldb), both ivb_fp8_quantize_blocks_t outputs; lda, ldb multiples of 16 and >= K.
 *   a_scale_inv [ceil(K/128), M] and b_scale_inv [ceil(K/128), N], 16-byte aligned.  M and N multiples of 8; epilogue
 *   IVB_EPI_BF16 or IVB_EPI_F32 (out0 16-byte aligned, ld0 a multiple of 8), no bias; flags 0 or IVB_FLAG_ACCUM.  One
 *   kernel form: the cooperative kernel (128 x 128 tiles) that promotes each k-block to fp32 on the CUDA cores.
 *   k_plan (optional, NULL: every k-block): the 128-token k-blocks to sum, ascending, then their count at
 *   k_plan[ceil(K/128)]: the M plan of a DropPath plan over the tokens (ivb_droppath_plan, plan + 0) as it is.  When
 *   the left-out rows of dy are zero the result has the unplanned call's bits; with none listed the sum is 0.        */
int ivb_fp8_quantize_blocks_t(const void* x, long ldx, int M, int C, void* out_t, long ldt, float* scale_inv,
                              void* stream);
int ivb_fp8_quantize_blocks_t_plan(const void* x, long ldx, int M, int C, void* out_t, long ldt, float* scale_inv,
                                   const float* rowscale, void* stream);
int ivb_gemm_fp8_wgrad(const void* A_t, long lda, const float* a_scale_inv, const void* B_t, long ldb,
                       const float* b_scale_inv, int M, int N, int K, int epilogue, int flags, void* out0, long ld0,
                       const int* k_plan, void* stream);

/* ---- RMSNorm / LayerNorm (row reductions, HBM-bound) -------------------------------------------
 * y(bf16) = norm(x) * weight (+ bias).  is_layernorm=0: RMSNorm (internvideo2_pretrain.py:117-128,
 * FA2 DropoutAddRMSNorm :467; eps 1e-6); 1: nn.LayerNorm (eps 1e-5, :525,:532).
 * x is fp32 (x_is_f32=1, the fp32 residual stream) or bf16.  rstd[M] (and mean[M] for LayerNorm)
 * are written for the backward pass.  bias, mean and rstd may be NULL.                            */
int ivb_norm_fwd(const void* x, int x_is_f32, long ldx, const void* weight, const void* bias,
                 float eps, int is_layernorm, int M, int D, void* y, long ldy, float* mean,
                 float* rstd, void* stream);
/* dx = d norm / dx (+ dx_in, fp32, pitch lddx_in, optional); dweight/dbias: fp32 [D], ACCUMULATED
 * (summed in a fixed order) — zero them first, or NULL.  mean is NULL for RMSNorm.  dx_out is fp32 or bf16.
 * In-place dx_out == dy is allowed.                                                              */
int ivb_norm_bwd(const void* dy, long lddy, const void* x, int x_is_f32, long ldx,
                 const void* weight, const float* mean, const float* rstd, int is_layernorm, int M,
                 int D, const float* dx_in, long lddx_in, void* dx_out, int dx_out_is_f32,
                 long lddx, float* dweight, float* dbias, void* stream);

/* q-norm AND k-norm of a block in one launch (internvideo2_pretrain.py:198-206: RMSNorm over the flattened H*d of q and
 * of k, weights [D] each): the two [M, D] column slices at x and x + x_pair_off of a bf16 [M, ldx] buffer.  D <= 1536.
 * rstd: fp32 [M][2] (token-major).  The backward writes dx in place of / next to dy with the same pairing. */
int ivb_rmsnorm_pair_fwd(const void* x, long ldx, long x_pair_off, const void* w0, const void* w1, float eps, int M,
                         int D, void* y, long ldy, long y_pair_off, float* rstd, void* stream);
int ivb_rmsnorm_pair_bwd(const void* dy, long lddy, long dy_pair_off, const void* x, long ldx, long x_pair_off,
                         const void* w0, const void* w1, const float* rstd, int M, int D, void* dx_out, long lddx,
                         long dx_pair_off, float* dweight0, float* dweight1, void* stream);
/* RMSNorm backward on the fp32 residual stream FUSED with the LayerScale backward that consumes its result in Block.backward
 * (internvideo2_pretrain.py:284-291 differentiated): dx_out = rmsnorm_bwd(dy, x, w, rstd) + dx_in (fp32 [M,D]);
 * dyb (bf16) = rowscale[m] * gamma * dx_out; dgamma += sum_m rowscale*dx_out*ybr; dcolsum += gamma * sum_m rowscale*dx_out;
 * dweight += RMSNorm weight gradient.  rowscale (DropPath factors), dx_in, dweight, dgamma and dcolsum are optional. */
int ivb_rmsnorm_bwd_layerscale(const void* dy, long lddy, const float* x, long ldx, const void* weight, const float* rstd,
                               int M, int D, const float* dx_in, long lddx_in, float* dx_out, long lddx, float* dweight,
                               const void* ybr, long ldyb, const void* gamma, const float* rowscale, void* dyb, long lddyb,
                               float* dgamma, float* dcolsum, void* stream);
/* ---- LayerScale backward (internvideo2_pretrain.py:131-146 + residual :284-291) -----------------
 * dx' = rowscale[m] * dx (rowscale optional: DropPath); dy(bf16) = gamma * dx' ;
 * dgamma[j] += sum_m dx'*y ; dcolsum[j] += gamma[j] * sum_m dx'  (= the branch Linear's bias gradient).
 * gamma may be NULL (no LayerScale: dy = dx'); y, dgamma and dcolsum may be NULL.                 */
int ivb_layerscale_bwd(const float* dx, long lddx, const void* y, long ldy, const void* gamma,
                       int M, int D, void* dy, long lddy, float* dgamma, float* dcolsum,
                       const float* rowscale, void* stream);
/* out[j] += sum_m x[m,j]   (bf16 in, fp32, summed in a fixed order) — bias gradients. */
int ivb_colsum_bf16(const void* x, long ldx, int M, int N, float* out, void* stream);

/* ---- attention (wgmma, flash-style)  -----------------------------------------------------------
 * out[b,q,h,:] = softmax(scale * q k^T) v, non-causal, no dropout.  q/k/v are [B*n, ld*] projection
 * buffers; `q` points at (token 0, head 0, dim 0) of its slot, heads are contiguous (h d), so the
 * packed qkv[B,S,3,H,d] layout of FlashAttention.forward (flash_attention_class.py:27-50) is passed
 * as q=qkv, k=qkv+H*d, v=qkv+2*H*d with ld=3*H*d.  lse2[B,H,n] (optional) = log2-domain logsumexp
 * of the scaled scores, consumed by ivb_attn_bwd.  head_dim: multiple of 8 in [16, 128] (the model
 * uses 64/88/128); every pitch a multiple of 8.  B = 0 or n = 0 is a no-op.                           */
int ivb_attn_fwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                 void* out, long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                 void* stream);
/* Head-axis attention of the VideoMAEv2 teacher exactly as the reference executes it (videomae.py:94-97 passes [B,H,N,d]
 * tensors to flash_attn_func, whose layout is [B,seqlen,nheads,d]: the softmax runs over the H heads of each token).
 * qkv: bf16 [B*N, ld] rows (q | k | v, each H*d); out: bf16 [B, H, N, d] contiguous (the caller reshapes it to [B, N, H*d]
 * the way the reference's `.reshape(B, N, -1)` does).  H <= 32. */
int ivb_headaxis_attn_fwd(const void* qkv, long ld, int B, int N, int H, int d, float softmax_scale, void* out,
                          void* stream);
/* Backward of ivb_attn_fwd (autograd of FlashAttention.forward / _naive_attn).  `out`, `dout` are
 * [B*n, ld] with heads contiguous; lse2 from the forward; delta_ws: 16-byte aligned fp32 workspace of
 * ivb_attn_bwd_workspace_floats(B, n, H) elements (padded lse2 + rowsum(dO*O));
 * dq/dk/dv are written (not accumulated), bf16, same head layout as q/k/v (typically the three
 * slots of one [B*n, 3*H*d] gradient buffer).                                                       */
long ivb_attn_bwd_workspace_floats(int B, int n, int H);
int ivb_attn_bwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                 const void* out, long ldo, const void* dout, long lddo, const float* lse2,
                 float* delta_ws, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv,
                 int B, int n, int H, int d, float softmax_scale, void* stream);
/* ivb_attn_fwd_plan / ivb_attn_bwd_plan: ivb_attn_fwd / ivb_attn_bwd that skip the clips a DropPath draw drops.
 * rowscale: the attention branch's DropPath factors, fp32 [B*n] (required; the EPI_RESID rowscale of proj), one
 * factor per clip repeated over its rows: clip b is dead when rowscale[b*n] is 0.  A dead clip's CTAs load nothing and
 * run no MMA.  The forward writes its out rows 0 and its lse2 rows 0 (finite); the backward writes its dq, dk and dv
 * rows 0, and its delta_ws entries as ivb_attn_bwd does.  Live clips get ivb_attn_fwd's / ivb_attn_bwd's bits.
 * Those are the results of the plain calls wherever they matter: proj multiplies a dead clip's attention output by
 * 0, so its gradient rows, and with them dq, dk and dv, are zero there too.                                        */
int ivb_attn_fwd_plan(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                      void* out, long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                      const float* rowscale, void* stream);
int ivb_attn_bwd_plan(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                      const void* out, long ldo, const void* dout, long lddo, const float* lse2,
                      float* delta_ws, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv,
                      int B, int n, int H, int d, float softmax_scale, const float* rowscale, void* stream);
/* ivb_attn_fwd_causal / ivb_attn_bwd_causal: ivb_attn_fwd / ivb_attn_bwd with a causal mask, key index > query index
 * masked out (the additive -inf upper triangle of the MobileCLIP text tower, text_encoder.py:149-158, 185-191), with
 * the same operands, operand rules and workspace.  Every row keeps its own key, so no row is empty.  The forward and
 * the dQ pass stream the key tiles up to the one that holds the CTA's last query, the dK/dV pass the query tiles from
 * the one that holds the CTA's first key; only the tiles that cross the diagonal are masked element by element.  There
 * is no causal form of the DropPath plans or of the FP8 forward.                                                      */
int ivb_attn_fwd_causal(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                        void* out, long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                        void* stream);
int ivb_attn_bwd_causal(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                        const void* out, long ldo, const void* dout, long lddo, const float* lse2,
                        float* delta_ws, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv,
                        int B, int n, int H, int d, float softmax_scale, void* stream);
/* ivb_attn_fwd_keylen: ivb_attn_fwd with a key-padding mask given as per-clip key lengths, with the same operands and
 * operand rules.  kv_len: int32 [B] (device, required): in clip b every key >= kv_len[b] is masked out for every query
 * (the additive -10000 of right-padded BERT captions, xbert.py:1099-1119, underflows to the same 0 in fp32).  All n
 * query rows are computed and written, padded ones included.  A clip's CTAs stream only the ceil(kv_len[b] / 64) key
 * tiles that hold its keys.  kv_len is read on the device, never by the host, so the call is capturable in a CUDA
 * graph.  An entry outside [1, n] makes that clip's out rows (and lse2 rows) NaN; the call still returns 0.  A null
 * kv_len is refused before any CUDA call.  There is no backward, causal, DropPath-plan or FP8 form.                 */
int ivb_attn_fwd_keylen(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                        void* out, long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                        const int* kv_len, void* stream);
/* ---- FP8 attention forward (FP8 inference of frozen towers; no lse, no backward) ------------------------------------
 * Every scale is a power of two chosen from an amax by the ivb_fp8_quantize_rows rule (E4M3; 1 when the amax is 0,
 * scale_inv NaN when the amax is Inf or NaN), so dequantisation is exact.  Same bits on every run; one stream-ordered
 * kernel per call; capturable in a CUDA graph.  head_dim d: a multiple of 8 in [16, 128] (the model uses 64 / 88 / 128).
 * B = 0 or n = 0 is a no-op.  A call that breaks a rule below is refused before any CUDA call.
 *
 * ivb_attn_fp8_pack: q, k, v as ivb_attn_fwd takes them (bf16 [B*n, H*d] views; ldq, ldk, ldv multiples of 8; 16-byte
 *   aligned) ->
 *   q8, k8 E4M3 [B*n, H*dp], dp = round_up(d, 32): head h in columns h*dp .. h*dp + d, then dp - d zero columns
 *     (pitch ld8, a multiple of 16 and >= H*dp; columns H*dp .. ld8 are not written), one scale per (token, head) from
 *     the amax of that head's d columns of the row: q_scale_inv, k_scale_inv fp32 [B, H, ns] with
 *     ns = ivb_attn_fp8_scale_pitch(n) (n rounded up to 64; entries n .. ns are written 0), 16-byte aligned;
 *   vt8 E4M3 [B, H, d, ldvt] = V^T per (clip, head) (ldvt a multiple of 16 and >= round_up(n, 16); keys n ..
 *     round_up(n, 16) are written 0, later ones are not written), one scale per (clip, head, channel) from the amax over
 *     the clip's n tokens: v_scale_inv fp32 [B, H, d].
 *   q8, k8 and vt8 are 16-byte aligned.
 * ivb_attn_fwd_fp8: out[b,q,h,:] = softmax(scale q k^T) v (bf16; pitch ldo, a multiple of 8; 4-byte aligned) from the
 *   pack's outputs, on the FP8 tensor cores: S = q_scale_inv k_scale_inv (q8 k8^T), P = exp2(S scale log2e - max) cast
 *   to E4M3 as P * 2^8, O = (P vt8^T) v_scale_inv / rowsum(P).  The operand rules are the pack's: ld8 and ldvt as above
 *   (a vt8 pitch below round_up(n, 16) is refused); q8, k8, vt8, q_scale_inv and k_scale_inv 16-byte aligned,
 *   v_scale_inv 8-byte.                                                                                           */
int ivb_attn_fp8_scale_pitch(int n);
int ivb_attn_fp8_pack(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, int B, int n, int H,
                      int d, void* q8, void* k8, long ld8, float* q_scale_inv, float* k_scale_inv, void* vt8, long ldvt,
                      float* v_scale_inv, void* stream);
int ivb_attn_fwd_fp8(const void* q8, const void* k8, long ld8, const float* q_scale_inv, const float* k_scale_inv,
                     const void* vt8, long ldvt, const float* v_scale_inv, void* out, long ldo, int B, int n, int H,
                     int d, float softmax_scale, void* stream);

/* ---- token front-end (tubelet embed as visible-only gather-GEMM) --------------------------------
 * idx[b, 0..n_keep) = ascending positions where mask[b, :] == 0 — the order of `x[~mask]`
 * (internvideo2_pretrain.py:659); bit-exact.  *err_flag is set to 1+b if clip b does not keep
 * exactly n_keep tokens.  mask is uint8/bool [B, N].                                               */
int ivb_visible_indices(const void* mask_u8, int B, int N, int n_keep, int* idx, int* err_flag,
                        void* stream);
/* im2col rows (bf16, K padded to Kpad with zeros) of patch tokens idx[b, j0 .. j0+rows_per_clip)
 * (token t >= 1 is patch t-1 in (frame, py, px) order); K axis ordered like the Conv3d weight
 * [D, C, tubelet, p, p] (PatchEmbed, internvideo2_pretrain.py:320-331).  video: bf16 [B,C,T,H,W].  */
int ivb_im2col_visible(const void* video, const int* idx, int idx_stride, int j0, int rows_per_clip,
                       int B, int C, int T, int H, int W, int tubelet, int patch, int Kpad,
                       void* cols, void* stream);
/* ivb_im2col_visible's rows, each normalised by the RMSNorm that InternVideo-Next's patch embed applies to a patch's
 * K = C*t*p*p pixels before the Conv3d (`norm_before`, InternVideo_next.py:302-342): per row
 * r = rsqrt(mean_k a_k^2 + eps) in fp32, cols[row, k] = bf16(weight[pi(k)] * bf16(a_k * r)), zeros for K <= k < Kpad,
 * and rstd[row] = r (fp32 [B*rows_per_clip], for ivb_prenorm_wgrad).  weight: bf16 [K] in the reference's
 * (t hp wp c) order; pi maps the column (c, dt, dy, dx) to ((dt*p + dy)*p + dx)*C + c.  Kpad <= 1536; video, idx,
 * cols and rstd 4-byte aligned, weight 2-byte aligned.                                                              */
int ivb_im2col_prenorm(const void* video, const int* idx, int idx_stride, int j0, int rows_per_clip, int B, int C,
                       int T, int H, int W, int tubelet, int patch, int Kpad, const void* weight, float eps, void* cols,
                       float* rstd, void* stream);
/* Weight gradient of that RMSNorm: dweight[pi(k)] += sum over rows of dcols[row, k] * bf16(a_k * rstd[row]) (fp32 [K]),
 * the normalised pixels recomputed from the video and ivb_im2col_prenorm's rstd; summed in a fixed order (see
 * Conventions).  dcols: bf16 [B*rows_per_clip, lddc], the gradient of the im2col rows (lddc a multiple of 8, >= Kpad).
 * Same row selection and limits as ivb_im2col_prenorm; dcols and dweight 4-byte aligned.                          */
int ivb_prenorm_wgrad(const void* video, const int* idx, int idx_stride, int j0, int rows_per_clip, int B, int C,
                      int T, int H, int W, int tubelet, int patch, int Kpad, const float* rstd, const void* dcols,
                      long lddc, float* dweight, void* stream);
/* out[b,j,:] = src[b*src_bstride + j*D + :] (fp32, optional) + table[idx[b*idx_bstride + j] + idx_off]
 * (bf16 table, optional; idx NULL means j).  cls/pos-embed adds :635-656, decoder pos adds :712-737. */
int ivb_gather_add(const float* src, long src_bstride, const void* table, const int* idx,
                   int idx_bstride, int idx_off, int B, int rows, int D, void* out, int out_is_f32,
                   long out_bstride, void* stream);
/* table_grad[idx[b,j] + idx_off, :] += g[b,j,:]  (fp32) — backward of ivb_gather_add (idx NULL means j).  Clips are
 * added in order; when idx[b,:] has no repeats within a clip the result is the same on every run. */
int ivb_scatter_add(const void* g, int g_is_f32, long g_bstride, const int* idx, int idx_bstride,
                    int idx_off, int B, int rows, int D, float* table_grad, void* stream);

/* ---- text-tower token embedding (MobileCLIP TextTransformer.forward_embedding, text_encoder.py:131-147) ------------
 * ivb_token_embed_fwd: out[b*L + l, :] = table[ids[b, l]] + pos[l] in fp32 (the residual stream; pitch ldo).  ids:
 *   int64 [B, L] (8-byte aligned); table: bf16 [V, D]; pos: bf16 [L, D].  An id outside [0, V) sets *err_flag (int32,
 *   device) to 1 + its row and reads table row 0 instead; nothing is read by the host.
 * ivb_token_embed_bwd: dtable[v] = sum of g[p] over the positions p with ids[p] == v, in position order, for every id
 *   present (the other rows of dtable are not written: zero them first); dpos[l] = sum over b = 0 .. B-1 of
 *   g[b*L + l].  g fp32 [B*L, D] (pitch ldg), dtable fp32 [V, D], dpos fp32 [L, D], all written, not accumulated.  No
 *   float atomics: the positions are sorted by id in ws (int32, ivb_token_embed_bwd_workspace_ints(V, B, L) elements),
 *   so the same inputs give the same bits on every run.  Out-of-range ids count as id 0, as in the forward.
 * D, ldo and ldg are multiples of 8; table, pos, out, g, dtable and dpos are 16-byte aligned.  Stream-ordered;
 *   capturable in a CUDA graph.  A call that breaks a rule is refused before any CUDA call.                          */
int ivb_token_embed_fwd(const long long* ids, int B, int L, const void* table, int V, const void* pos, int D,
                        float* out, long ldo, int* err_flag, void* stream);
long ivb_token_embed_bwd_workspace_ints(int V, int B, int L);
int ivb_token_embed_bwd(const long long* ids, int B, int L, const float* g, long ldg, int V, int D, float* dtable,
                        float* dpos, int* ws, void* stream);

/* ---- rotary position embedding (LLaMA's apply_rotary_pos_emb with rotate_half, transformers modeling_llama; the
 * InternVideo2-CLIP text tower, backbones/internvideo2/internvideo2_clip_text.py) ---------------------------------
 * ivb_rope_qk: rotates heads h = 0 .. H-1 of the q and k rows of B clips of L tokens in place; row r = b*L + l is at
 *   q + r*ldq and k + r*ldk (bf16; q and k may be column slots of one qkv buffer), its head h at columns h*d .. h*d + d.
 *   With half = d/2 and c, s = cos_t[l, j], sin_t[l, j] (fp32 [L, half], contiguous; l the position in the clip):
 *     x_j' = x_j c - x_{j+half} s,   x_{j+half}' = x_{j+half} c + x_j s   (j < half),
 *   in fp32, each result rounded to bf16 once.  d a multiple of 16 in [16, 128]; ldq, ldk multiples of 8 and >= H*d;
 *   q, k, cos_t and sin_t 16-byte aligned.  B = 0 or L = 0 is a no-op.  One stream-ordered kernel; capturable in a
 *   CUDA graph.  A call that breaks a rule is refused before any CUDA call.                                          */
int ivb_rope_qk(void* q, long ldq, void* k, long ldk, int B, int L, int H, int d, const float* cos_t,
                const float* sin_t, void* stream);

/* ---- decoder heads: LayerNorm(1e-5) -> x/||x|| (+ optional fused (2-2<out,tgt>) loss sum) --------
 * Linear_Decoder / MLP_Decoder.forward tail (internvideo2_pretrain.py:356-359, 394-397) and the
 * alignment loss (engines/engine_for_pretraining.py:131-136).  stats: fp32 [M,3] = mean, rstd, 1/||y||.
 * out may be NULL when only the loss is wanted; target NULL when only the features are wanted.      */
int ivb_ln_l2_fwd(const void* z, long ldz, const void* weight, const void* bias, float eps, int M,
                  int C, void* out, long ldo, float* stats, const void* target, int target_is_f32,
                  long ldt, float* loss_sum, void* stream);
/* d_out = (gscale_host * *gscale_dev) * dout (gscale_dev NULL: 1).  For the fused loss pass dout = target and
 * gscale_host = -2/rows.  Writes dz (bf16); accumulates dweight/dbias (fp32, optional).          */
int ivb_ln_l2_bwd(const void* z, long ldz, const void* weight, const void* bias, const float* stats,
                  int M, int C, const void* dout, int dout_is_f32, long lddo, float gscale_host,
                  const float* gscale_dev, void* dz, long lddz, float* dweight, float* dbias,
                  void* stream);

/* ---- video-text contrastive loss (criterions.py:15-55, 65-103, 200-216) --------------------------
 * cos_v2t [G,G] fp32 = normalize(v) @ normalize(t)^T over the GATHERED batch; idx int64 [G].
 * *loss += 1/2 (CE_v2t + CE_t2v) with soft targets (idx==idx^T)/rowsum.  lse_row/lse_col: fp32 [G].
 * The loss sums one partial per row and per column in the library's scratch: G <= 3 145 728.         */
/* temp_dev (optional, device fp32[1]) overrides `temp`: the learnable temperature stays on the device
 * (internvideo2_clip_small.py:45,96-99), no host read per step, valid inside a captured CUDA graph.  */
int ivb_vtc_loss_fwd(const float* cos_v2t, const long long* idx, int G, float temp,
                     const float* temp_dev, float* lse_row, float* lse_col, float* loss, void* stream);
/* dcos (bf16 [G,G]) = d loss / d cos_v2t * gscale; *dtemp += d loss / d temp * gscale, with gscale = gscale_host *
 * *gscale_dev (gscale_dev optional).                                                                */
int ivb_vtc_loss_bwd(const float* cos_v2t, const long long* idx, int G, float temp,
                     const float* temp_dev, const float* lse_row, const float* lse_col, float gscale_host,
                     const float* gscale_dev, void* dcos_bf16, float* dtemp, void* stream);
/* F.normalize(x, dim=-1) (eps 1e-12) -> bf16 rows + 1/norm; and its backward. */
int ivb_l2norm_rows_fwd(const void* x, int x_is_f32, long ldx, int M, int C, void* out, long ldo,
                        float* inv_norm, void* stream);
int ivb_l2norm_rows_bwd(const float* dy, long lddy, const void* xn, long ldxn, const float* inv_norm,
                        int M, int C, float* dx, long lddx, void* stream);

/* ---- IV1 VideoMAE pixel-reconstruction target + MSE (engine_for_pretraining.py:66-106) -----------
 * labels fp32 [B*n_mask, tubelet*p*p*C] ('b n (p c)'), per-patch per-channel (x-mean)/(sqrt(var_unbiased)+1e-6)
 * of the un-normalised video (x*std+mean).  masked_idx: int32 [B*n_mask] patch indices.              */
int ivb_pixel_targets(const void* video, const int* masked_idx, int n_mask, int B, int C, int T,
                      int H, int W, int tubelet, int patch, int normalize, const float* mean3,
                      const float* std3, float* labels, void* stream);
/* *loss_sum += sum (pred-label)^2 ; dpred (bf16, optional) = gscale * 2 (pred-label), gscale = gscale_host *
 * *gscale_dev.  loss_sum and gscale_dev are optional.                                               */
int ivb_mse_loss(const void* pred_bf16, const float* label, long n, float* loss_sum,
                 float gscale_host, const float* gscale_dev, void* dpred_bf16, void* stream);

/* ---- single-query attention pooling (AttentionPoolingBlock / CrossAttention with 1 query per clip,
 * internvideo2_pretrain.py:61-76,107-114).  q: bf16 [B, H*d]; k, v: bf16 [B*n, ld]; out: bf16 [B, H*d];
 * probs: fp32 [B,H,n] (saved for the backward).  dq/dk/dv are written, not accumulated.  The scores of
 * one (clip, head) live in 48 KB of shared memory: n <= 12280 - d (forward), n <= 12280 - 2d (backward). */
int ivb_pool_attn_fwd(const void* q, const void* k, long ldk, const void* v, long ldv, int B, int n,
                      int H, int d, float scale, void* out, float* probs, void* stream);
int ivb_pool_attn_bwd(const void* q, const void* k, long ldk, const void* v, long ldv,
                      const float* probs, const void* dout, int B, int n, int H, int d, float scale,
                      void* dq, void* dk, long lddk, void* dv, long lddv, void* stream);

/* ---- InternVideo-MM global extractor: position conv + key LayerNorm (clip_vit_only_global.py:203-231, 147) ----------
 * ivb_dpe_ln_fwd: x holds one extractor tap of the backbone stream, N clips of T frames of 1 + H*W rows each: row
 *   (n*T + t)*(1 + H*W) + l, l = 0 the frame's cls row, l = 1 + h*W + w its patch (h, w).  x is fp32 (x_is_f32 = 1,
 *   the residual stream) or bf16, pitch ldx.  y bf16 (pitch ldy), the same rows:
 *     patch row:  y = LN(x + conv_b + sum_{dt,dh,dw in {-1,0,1}} conv_w[c, dt, dh, dw] * x[n, t+dt, h+dh, w+dw, c])
 *     cls row:    y = LN(x)
 *   with zero padding at the edges of the T x H x W grid (the depthwise Conv3d `dpe`, kernel 3, padding 1, bias, added
 *   to the patch tokens, then `ln_3`).  LN: LayerNorm over C with ln_w, ln_b and eps.  conv_w: bf16 [C, 1, 3, 3, 3] as
 *   the reference stores it (2-byte aligned); conv_b, ln_w, ln_b: bf16 [C].  Every sum in fp32, one bf16 rounding of y;
 *   the same bits on every run (no atomics).  T, H, W >= 1 (T = 1: only the centre temporal tap contributes); C a
 *   multiple of 8 in [8, 4096]; ldx, ldy multiples of 8 and >= C; x, conv_b, ln_w, ln_b and y 16-byte aligned; y must
 *   not overlap x (a CTA reads the neighbour rows that other CTAs write).  N = 0
 *   is a no-op.  One stream-ordered kernel; capturable in a CUDA graph.  A call that breaks a rule is refused before
 *   any CUDA call.                                                                                                  */
int ivb_dpe_ln_fwd(const void* x, int x_is_f32, long ldx, const void* conv_w, const void* conv_b, const void* ln_w,
                   const void* ln_b, float eps, int N, int T, int H, int W, int C, void* y, long ldy, void* stream);

/* ---- flat AdamW (decoupled weight decay; fp32 master/moments, bf16 model copy) --------------------
 * torch.optim.AdamW semantics (optim_factory.py:141-142; DeepSpeed adam_w_mode utils.py:821-834).
 * Gradients are multiplied by grad_scale * (*grad_scale_dev) first (1/world_size, clip coefficient; grad_scale_dev
 * optional). */
int ivb_adamw_step(float* master, float* exp_avg, float* exp_avg_sq, const void* grad,
                   int grad_is_f32, void* param_bf16, long n, float lr, float beta1, float beta2,
                   float eps, float weight_decay, int step, float grad_scale,
                   const float* grad_scale_dev, const float* dyn_lr_step, void* stream);
/* dyn_lr_step (optional): device float[2] = {lr, step}; when given it overrides the host lr/step so a
 * captured CUDA graph of the training step stays valid while the schedule advances.               */

/* ---- in-switch (NVLS) gradient all-reduce over an NVLink multicast mapping --------------------------
 * Replaces the reference's DDP / DeepSpeed gradient all-reduce (run_pretraining.py:378 DistributedDataParallel,
 * utils.py:814-834 deepspeed.initialize) for the flat bf16 gradient buffer.  Elements
 * [elem_off, elem_off + numel) of a symmetric buffer — the same allocation on every rank, mapped by all of them
 * through the multicast address mc_base — become the sum over ranks on EVERY rank (fp32 accumulation inside the
 * switch, one bf16 rounding; bit-identical on all ranks).  flag_ptrs_dev: device array of `world` pointers, entry p
 * = rank p's peer-mapped, zero-initialised flag array of ivb_nvls_flag_words() uint32.  Every rank must launch the
 * same sequence of these calls (collective).  elem_off and numel must be multiples of 8.             */
int ivb_nvls_allreduce_bf16(void* mc_base, long elem_off, long numel, const void* flag_ptrs_dev, int rank,
                            int world, int nblocks, void* stream);
int ivb_nvls_flag_words(void);

#ifdef __cplusplus
}
#endif
#endif /* IVB200_H_ */
