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
 *     ivb_colsum_bf16, ivb_ln_l2_bwd) are summed over rows in a fixed order through a per-device scratch of the
 *     library, so the same inputs give the same bits on every run.  That scratch holds one reduction at a time:
 *     these entry points must not be called concurrently from two streams of the same device.
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

#define IVB_FLAG_GELU_TANH 1 /* tanh-approx GELU (FA2 FusedMLP) instead of erf (nn.GELU)           */
#define IVB_FLAG_ACCUM 2     /* accumulate into out0                                               */
#define IVB_FLAG_1CTA 4      /* force the single-CTA kernel (128-row tiles)                                      */
#define IVB_FLAG_2CTA 8      /* force the CTA-pair kernel (cluster of 2, 256-row tiles, B tile TMA-multicast)     */
#define IVB_FLAG_GELU_SAVE_GRAD 16 /* EPI_BIAS_GELU: out1 receives gelu'(h) instead of h; EPI_GELU_BWD: aux IS
                                     that saved derivative (out0 = acc * aux) — the backward epilogue then has
                                     no transcendental work (the training path; h itself is never needed)   */

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
 * 356,394 and FA2 fused_dense (FusedMLP :269).  tile_n: 0 = auto, or one of 128/176/192/256.     */
/* process-wide default for problems with M >= 512: 1 = CTA-pair kernel, 0 = single-CTA kernel. */
void ivb_set_default_2cta(int enable);
int ivb_gemm_bf16(const void* A, int a_mn_major, long lda, const void* B, int b_mn_major, long ldb,
                  int M, int N, int K, int epilogue, int flags, void* out0, long ld0, void* out1,
                  long ld1, const void* bias, const void* gamma, const void* aux, long ldaux,
                  const float* rowscale, int tile_n, void* stream);

/* ---- RMSNorm / LayerNorm (row reductions, HBM-bound) -------------------------------------------
 * y(bf16) = norm(x) * weight (+ bias).  is_layernorm=0: RMSNorm (internvideo2_pretrain.py:117-128,
 * FA2 DropoutAddRMSNorm :467; eps 1e-6); 1: nn.LayerNorm (eps 1e-5, :525,:532).
 * x is fp32 (x_is_f32=1, the fp32 residual stream) or bf16.  rstd[M] (and mean[M] for LayerNorm)
 * are written for the backward pass.                                                              */
int ivb_norm_fwd(const void* x, int x_is_f32, long ldx, const void* weight, const void* bias,
                 float eps, int is_layernorm, int M, int D, void* y, long ldy, float* mean,
                 float* rstd, void* stream);
/* dx = d norm / dx (+ dx_in, fp32, pitch lddx_in, optional); dweight/dbias: fp32 [D], ACCUMULATED
 * (summed in a fixed order) — zero them first.  dx_out is fp32 or bf16.  In-place dx_out == dy is allowed.      */
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
 * dweight += RMSNorm weight gradient.  rowscale (DropPath factors) and dx_in are optional. */
int ivb_rmsnorm_bwd_layerscale(const void* dy, long lddy, const float* x, long ldx, const void* weight, const float* rstd,
                               int M, int D, const float* dx_in, long lddx_in, float* dx_out, long lddx, float* dweight,
                               const void* ybr, long ldyb, const void* gamma, const float* rowscale, void* dyb, long lddyb,
                               float* dgamma, float* dcolsum, void* stream);
/* ---- LayerScale backward (internvideo2_pretrain.py:131-146 + residual :284-291) -----------------
 * dx' = rowscale[m] * dx (rowscale optional: DropPath); dy(bf16) = gamma * dx' ;
 * dgamma[j] += sum_m dx'*y ; dcolsum[j] += gamma[j] * sum_m dx'  (= the branch Linear's bias gradient).
 * gamma may be NULL (no LayerScale: dy = dx').                                                     */
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
 * of the scaled scores, consumed by ivb_attn_bwd.  head_dim: multiple of 8, <= 128 (64/88/128).   */
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
/* out[b,j,:] = src[b*src_bstride + j*D + :] (fp32, optional) + table[idx[b*idx_bstride + j] + idx_off]
 * (bf16 table, optional; idx NULL means j).  cls/pos-embed adds :635-656, decoder pos adds :712-737. */
int ivb_gather_add(const float* src, long src_bstride, const void* table, const int* idx,
                   int idx_bstride, int idx_off, int B, int rows, int D, void* out, int out_is_f32,
                   long out_bstride, void* stream);
/* table_grad[idx[b,j] + idx_off, :] += g[b,j,:]  (fp32) — backward of ivb_gather_add.  Clips are added in order;
 * when idx[b,:] has no repeats within a clip the result is the same on every run. */
int ivb_scatter_add(const void* g, int g_is_f32, long g_bstride, const int* idx, int idx_bstride,
                    int idx_off, int B, int rows, int D, float* table_grad, void* stream);

/* ---- decoder heads: LayerNorm(1e-5) -> x/||x|| (+ optional fused (2-2<out,tgt>) loss sum) --------
 * Linear_Decoder / MLP_Decoder.forward tail (internvideo2_pretrain.py:356-359, 394-397) and the
 * alignment loss (engines/engine_for_pretraining.py:131-136).  stats: fp32 [M,3] = mean, rstd, 1/||y||.
 * out may be NULL when only the loss is wanted; target NULL when only the features are wanted.      */
int ivb_ln_l2_fwd(const void* z, long ldz, const void* weight, const void* bias, float eps, int M,
                  int C, void* out, long ldo, float* stats, const void* target, int target_is_f32,
                  long ldt, float* loss_sum, void* stream);
/* d_out = (gscale_host * *gscale_dev) * dout.  For the fused loss pass dout = target and
 * gscale_host = -2/rows.  Writes dz (bf16); accumulates dweight/dbias (fp32).                    */
int ivb_ln_l2_bwd(const void* z, long ldz, const void* weight, const void* bias, const float* stats,
                  int M, int C, const void* dout, int dout_is_f32, long lddo, float gscale_host,
                  const float* gscale_dev, void* dz, long lddz, float* dweight, float* dbias,
                  void* stream);

/* ---- video-text contrastive loss (criterions.py:15-55, 65-103, 200-216) --------------------------
 * cos_v2t [G,G] fp32 = normalize(v) @ normalize(t)^T over the GATHERED batch; idx int64 [G].
 * *loss += 1/2 (CE_v2t + CE_t2v) with soft targets (idx==idx^T)/rowsum.  lse_row/lse_col: fp32 [G]. */
/* temp_dev (optional, device fp32[1]) overrides `temp`: the learnable temperature stays on the device
 * (internvideo2_clip_small.py:45,96-99), no host read per step, valid inside a captured CUDA graph.  */
int ivb_vtc_loss_fwd(const float* cos_v2t, const long long* idx, int G, float temp,
                     const float* temp_dev, float* lse_row, float* lse_col, float* loss, void* stream);
/* dcos (bf16 [G,G]) = d loss / d cos_v2t * gscale; *dtemp += d loss / d temp * gscale.              */
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
/* *loss_sum += sum (pred-label)^2 ; dpred (bf16, optional) = gscale * 2 (pred-label).               */
int ivb_mse_loss(const void* pred_bf16, const float* label, long n, float* loss_sum,
                 float gscale_host, const float* gscale_dev, void* dpred_bf16, void* stream);

/* ---- single-query attention pooling (AttentionPoolingBlock / CrossAttention with 1 query per clip,
 * internvideo2_pretrain.py:61-76,107-114).  q: bf16 [B, H*d]; k, v: bf16 [B*n, ld]; out: bf16 [B, H*d];
 * probs: fp32 [B,H,n] (saved for the backward).  dq/dk/dv are written, not accumulated.               */
int ivb_pool_attn_fwd(const void* q, const void* k, long ldk, const void* v, long ldv, int B, int n,
                      int H, int d, float scale, void* out, float* probs, void* stream);
int ivb_pool_attn_bwd(const void* q, const void* k, long ldk, const void* v, long ldv,
                      const float* probs, const void* dout, int B, int n, int H, int d, float scale,
                      void* dq, void* dk, long lddk, void* dv, long lddv, void* stream);

/* ---- flat AdamW (decoupled weight decay; fp32 master/moments, bf16 model copy) --------------------
 * torch.optim.AdamW semantics (optim_factory.py:141-142; DeepSpeed adam_w_mode utils.py:821-834).
 * Gradients are multiplied by grad_scale * (*grad_scale_dev) first (1/world_size, clip coefficient). */
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
