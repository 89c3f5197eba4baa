// ivb_loss.cu — contrastive loss, L2 row normalisation, pixel targets + MSE, the flat AdamW step and single-query
// attention pooling: HBM-bound kernels with warp-shuffle row reductions.  The decoder heads' LN -> L2 alignment loss
// is in ivb_norm.cu.
//
//   video-text contrastive       InternVideo2/multi_modality/models/criterions.py:15-55,65-103,200-216
//   pixel-reconstruction target  InternVideo1/Pretrain/VideoMAE/engine_for_pretraining.py:66-98 + MSE :43,106
#include <math.h>

#include "ivb_internal.h"
#include "ivb_ptx.cuh"
#include "ivb_rows.cuh"

namespace ivb {

// ---------------------------------------------------------------- flat AdamW (fp32 master, bf16 model copy)
template <bool G_F32>
__global__ void adamw_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v,
                             const void* __restrict__ grad, __nv_bfloat16* __restrict__ param_bf16,
                             long n, float lr, float beta1, float beta2, float eps, float wd,
                             float step, float grad_scale_host,
                             const float* __restrict__ grad_scale_dev, const float* __restrict__ dyn) {
  const long i = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  if (dyn != nullptr) {  // device-resident {lr, step}: keeps a captured CUDA graph valid across steps
    lr = dyn[0];
    step = dyn[1];
  }
  // The bias corrections are computed here for a host step too, so the two give the same bits.
  const float bc1 = 1.f - powf(beta1, step);
  const float bc2 = 1.f - powf(beta2, step);
  const float gs_dev = grad_scale_dev ? *grad_scale_dev : 1.f;
  // a device scale that is not a positive finite number marks a bad step (NaN/Inf global gradient norm:
  // engine.step(check_finite) — engine_for_pretraining.py:151-161 aborts there): leave every state untouched
  if (!(gs_dev > 0.f) || gs_dev > 3.0e38f) return;
  const float grad_scale = grad_scale_host * gs_dev;
  float g[4], p[4], mm[4], vv[4];
  const int cnt = (n - i) >= 4 ? 4 : static_cast<int>(n - i);
  // 16-byte vector path when the 4-element group is whole and every base pointer is 16 B aligned
  const bool vec = cnt == 4 &&
                   ((reinterpret_cast<uintptr_t>(master) | reinterpret_cast<uintptr_t>(m) |
                     reinterpret_cast<uintptr_t>(v)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(grad) & (G_F32 ? 15 : 7)) == 0 &&
                   (reinterpret_cast<uintptr_t>(param_bf16) & 7) == 0;
  if (vec) {
    const float4 p4 = *reinterpret_cast<const float4*>(master + i);
    const float4 m4 = *reinterpret_cast<const float4*>(m + i);
    const float4 v4 = *reinterpret_cast<const float4*>(v + i);
    p[0] = p4.x; p[1] = p4.y; p[2] = p4.z; p[3] = p4.w;
    mm[0] = m4.x; mm[1] = m4.y; mm[2] = m4.z; mm[3] = m4.w;
    vv[0] = v4.x; vv[1] = v4.y; vv[2] = v4.z; vv[3] = v4.w;
    if (G_F32) {
      const float4 g4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(grad) + i);
      g[0] = g4.x; g[1] = g4.y; g[2] = g4.z; g[3] = g4.w;
    } else {
      const uint2 gb = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(grad) + i);
      const float2 a = unpack_bf16(gb.x), b = unpack_bf16(gb.y);
      g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] *= grad_scale;
  } else {
    for (int k = 0; k < cnt; ++k) {
      g[k] = (G_F32 ? reinterpret_cast<const float*>(grad)[i + k]
                    : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(grad)[i + k])) * grad_scale;
      p[k] = master[i + k]; mm[k] = m[i + k]; vv[k] = v[i + k];
    }
  }
  const float inv_bc1 = 1.f / bc1, inv_bc2 = 1.f / bc2, decay = 1.f - lr * wd;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k < cnt) {
      p[k] *= decay;
      mm[k] = beta1 * mm[k] + (1.f - beta1) * g[k];
      vv[k] = beta2 * vv[k] + (1.f - beta2) * g[k] * g[k];
      p[k] -= lr * (mm[k] * inv_bc1) / (sqrtf(vv[k] * inv_bc2) + eps);
    }
  }
  if (vec) {
    *reinterpret_cast<float4*>(master + i) = make_float4(p[0], p[1], p[2], p[3]);
    *reinterpret_cast<float4*>(m + i) = make_float4(mm[0], mm[1], mm[2], mm[3]);
    *reinterpret_cast<float4*>(v + i) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    uint2 pb;
    pb.x = pack_bf16(p[0], p[1]); pb.y = pack_bf16(p[2], p[3]);
    *reinterpret_cast<uint2*>(param_bf16 + i) = pb;
  } else {
    for (int k = 0; k < cnt; ++k) {
      master[i + k] = p[k]; m[i + k] = mm[k]; v[i + k] = vv[k];
      param_bf16[i + k] = __float2bfloat16(p[k]);
    }
  }
}

// ---------------------------------------------------------------- contrastive loss (video-text)
// cosv2t [G,G] fp32 = vn @ tn^T (wgmma GEMM).  S = cos / temp.  idx int64 [G].
// row pass: lse_r[i], tsum_r[i] = sum_j tg[i,j] S[i,j] ; col pass: lse_c[i], tsum_c[i] = sum_j tg[i,j] S[j,i]
// loss = 1/(2G) sum_i [(lse_r[i] - tsum_r[i]) + (lse_c[i] - tsum_c[i])]          (criterions.py:93-102)
// Each CTA stores its term in loss_part[blockIdx.x]; scalar_finish adds them into the loss in slot order.
__global__ void __launch_bounds__(256)
vtc_stats_kernel(const float* __restrict__ cosm, const long long* __restrict__ idx, int G, float inv_temp,
                 const float* __restrict__ temp_dev,
                 float* __restrict__ lse_r, float* __restrict__ lse_c, float* __restrict__ loss_part) {
  // a device-resident temperature (the learnable `temp` parameter) overrides the host value: no D2H
  // sync per step and a captured CUDA graph follows the parameter as it trains
  if (temp_dev != nullptr) inv_temp = 1.f / *temp_dev;
  // blocks [0, G): row i ; blocks [G, 2G): column i
  const int which = blockIdx.x / G;
  const int i = blockIdx.x % G;
  const long long my = idx[i];
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < G; j += blockDim.x) {
    const float s = (which == 0 ? cosm[static_cast<long>(i) * G + j] : cosm[static_cast<long>(j) * G + i]) * inv_temp;
    mx = fmaxf(mx, s);
  }
  __shared__ float red[3 * 8];
  mx = block_reduce<true>(mx, red);
  float sums[3] = {0.f, 0.f, 0.f};   // sum exp(S - mx), sum of the target entries' S, their count
  for (int j = threadIdx.x; j < G; j += blockDim.x) {
    const float s = (which == 0 ? cosm[static_cast<long>(i) * G + j] : cosm[static_cast<long>(j) * G + i]) * inv_temp;
    sums[0] += __expf(s - mx);
    if (idx[j] == my) { sums[1] += s; sums[2] += 1.f; }
  }
  block_reduce(sums, red);
  if (threadIdx.x == 0) {
    const float lse = mx + __logf(sums[0]);
    (which == 0 ? lse_r : lse_c)[i] = lse;
    loss_part[blockIdx.x] = (lse - sums[1] / sums[2]) * (0.5f / G);
  }
}

// dS[a,b] = gs/(2G) * [ exp(S-lse_r[a]) + exp(S-lse_c[b]) - 2*tg[a,b] ] ; written as bf16 d(cos) = dS/temp
// and row a's share of dtemp = sum dS * (-S/temp) stored in dtemp_part[a] (null: not wanted).
__global__ void __launch_bounds__(256)
vtc_grad_kernel(const float* __restrict__ cosm, const long long* __restrict__ idx, int G, float inv_temp,
                const float* __restrict__ temp_dev,
                const float* __restrict__ lse_r, const float* __restrict__ lse_c, float gscale_host,
                const float* __restrict__ gscale_dev, __nv_bfloat16* __restrict__ dcos,
                float* __restrict__ dtemp_part) {
  if (temp_dev != nullptr) inv_temp = 1.f / *temp_dev;
  const int a = blockIdx.x;
  const float gs = gscale_host * (gscale_dev ? *gscale_dev : 1.f) * (0.5f / G);
  const long long my = idx[a];
  float cnt = 0.f;
  for (int j = threadIdx.x; j < G; j += blockDim.x) cnt += (idx[j] == my) ? 1.f : 0.f;
  __shared__ float red[8];
  const float inv_cnt = 1.f / block_reduce(cnt, red);
  const float la = lse_r[a];
  float dt = 0.f;
  for (int b = threadIdx.x; b < G; b += blockDim.x) {
    const float s = cosm[static_cast<long>(a) * G + b] * inv_temp;
    const float tg = (idx[b] == my) ? inv_cnt : 0.f;
    const float ds = gs * (__expf(s - la) + __expf(s - lse_c[b]) - 2.f * tg);
    dcos[static_cast<long>(a) * G + b] = __float2bfloat16(ds * inv_temp);
    dt += ds * (-s * inv_temp);
  }
  dt = block_reduce(dt, red);
  if (threadIdx.x == 0 && dtemp_part) dtemp_part[a] = dt;
}

// F.normalize(x, dim=-1) rows (eps 1e-12): out bf16, inv_norm saved.   x fp32 or bf16.
template <bool XF32>
__global__ void l2norm_rows_kernel(const void* __restrict__ x, long ldx, int M, int C,
                                   __nv_bfloat16* __restrict__ out, long ldo, float* __restrict__ inv_norm) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float ss = 0.f;
  for (int c = lane * 8; c < C; c += 256) { float v[8]; load8<XF32>(x, row * ldx + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) ss += v[k] * v[k]; }
  ss = warp_sum(ss);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  for (int c = lane * 8; c < C; c += 256) { float v[8], o[8]; load8<XF32>(x, row * ldx + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = v[k] * inv;
    store8<false>(out, row * ldo + c, o); }
  if (lane == 0 && inv_norm) inv_norm[row] = inv;
}
// backward of F.normalize: dx = inv * (dy - xn * <dy, xn>)   (dy fp32, xn bf16) -> dx fp32
__global__ void l2norm_rows_bwd_kernel(const float* __restrict__ dy, long lddy, const __nv_bfloat16* __restrict__ xn,
                                       long ldxn, const float* __restrict__ inv_norm, int M, int C,
                                       float* __restrict__ dx, long lddx) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float dot = 0.f;
  for (int c = lane * 8; c < C; c += 256) { float g[8], v[8]; load8<true>(dy, row * lddy + c, g); load8<false>(xn, row * ldxn + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) dot += g[k] * v[k]; }
  dot = warp_sum(dot);
  const float inv = inv_norm[row];
  for (int c = lane * 8; c < C; c += 256) { float g[8], v[8], o[8]; load8<true>(dy, row * lddy + c, g); load8<false>(xn, row * ldxn + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = inv * (g[k] - v[k] * dot);
    store8<true>(dx, row * lddx + c, o); }
}

// ---------------------------------------------------------------- IV1 pixel targets + MSE
// One CTA (C warps) per masked patch: warp c normalises channel c over the tub*P*P pixels
// (mean / unbiased variance, +1e-6 on the std), labels layout 'b n (p c)'.
// The sums run over u - pivot, the pivot being the channel's first pixel of the patch: a flat patch then sums to
// exactly 0 and gets the label 0, where raw sums of u leave a rounding residue that the 1e-6 guard amplifies ~10^6
// times; a near-flat patch keeps its small differences instead of losing them to the cancellation of large sums.
__global__ void pixel_target_kernel(const __nv_bfloat16* __restrict__ video, const int* __restrict__ midx,
                                    int n_mask, int B, int C, int T, int H, int W, int tub, int P,
                                    int normalize, const float* __restrict__ mean3, const float* __restrict__ std3,
                                    float* __restrict__ labels) {
  const int row = blockIdx.x;            // b * n_mask + m
  const int b = row / n_mask;
  const int c = threadIdx.x >> 5;        // channel
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const int tok = midx[row];
  const int gw = W / P, gh = H / P;
  const int f = tok / (gh * gw), py = (tok / gw) % gh, px = tok % gw;
  const int npix = tub * P * P;
  const float mu_c = mean3[c], sd_c = std3[c];
  // un-normalised pixel i of the patch: one rounding, the same bits wherever it is evaluated
  auto pixel = [&](int i) {
    const int dx = i % P, dy = (i / P) % P, dt = i / (P * P);
    const long src = (((static_cast<long>(b) * C + c) * T + (f * tub + dt)) * H + (py * P + dy)) * W + (px * P + dx);
    return fmaf(__bfloat162float(video[src]), sd_c, mu_c);
  };
  float* out = labels + static_cast<long>(row) * npix * C;
  if (!normalize) {
    for (int i = lane; i < npix; i += 32) out[static_cast<long>(i) * C + c] = pixel(i);
    return;
  }
  const float pivot = __shfl_sync(0xffffffffu, lane == 0 ? pixel(0) : 0.f, 0);
  float s = 0.f;
  for (int i = lane; i < npix; i += 32) s += pixel(i) - pivot;
  const float mean = warp_sum(s) / npix;        // relative to the pivot
  float ss = 0.f;
  for (int i = lane; i < npix; i += 32) {
    const float d = (pixel(i) - pivot) - mean;
    ss += d * d;
  }
  const float var = warp_sum(ss) / (npix - 1);
  const float inv = 1.f / (sqrtf(var) + 1e-6f);
  for (int i = lane; i < npix; i += 32) out[static_cast<long>(i) * C + c] = ((pixel(i) - pivot) - mean) * inv;
}

// the CTA's sum (pred - label)^2 -> loss_part[blockIdx.x] (null: not wanted) ; dpred(bf16) = gscale * 2 (pred - label)
// (optional)
__global__ void __launch_bounds__(256)
mse_kernel(const __nv_bfloat16* __restrict__ pred, const float* __restrict__ label, long n,
           float* __restrict__ loss_part, float gscale_host, const float* __restrict__ gscale_dev,
           __nv_bfloat16* __restrict__ dpred) {
  const float gs = gscale_host * (gscale_dev ? *gscale_dev : 1.f);
  float acc = 0.f;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const float d = __bfloat162float(pred[i]) - label[i];
    acc += d * d;
    if (dpred) dpred[i] = __float2bfloat16(2.f * gs * d);
  }
  __shared__ float red[8];
  acc = block_reduce(acc, red);
  if (threadIdx.x == 0 && loss_part) loss_part[blockIdx.x] = acc;
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_adamw_step(float* master, float* exp_avg, float* exp_avg_sq, const void* grad,
                              int grad_is_f32, void* param_bf16, long n, float lr, float beta1,
                              float beta2, float eps, float weight_decay, int step, float grad_scale,
                              const float* grad_scale_dev, const float* dyn_lr_step, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n <= 0) return 0;
  const int threads = 256;
  const long blocks = (n + threads * 4 - 1) / (threads * 4);
  return launch("adamw_kernel", grad_is_f32 ? adamw_kernel<true> : adamw_kernel<false>, (unsigned)blocks, threads, 0,
                stream, NO_PDL, master, exp_avg, exp_avg_sq, grad, reinterpret_cast<__nv_bfloat16*>(param_bf16), n, lr,
                beta1, beta2, eps, weight_decay, static_cast<float>(step), grad_scale, grad_scale_dev, dyn_lr_step);
}

extern "C" int ivb_vtc_loss_fwd(const float* cos_v2t, const long long* idx, int G, float temp,
                                const float* temp_dev, float* lse_row, float* lse_col, float* loss,
                                void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (G <= 0) return 0;
  if (temp_dev == nullptr && !(temp > 0.f)) return set_error("ivb_vtc_loss_fwd: temp must be > 0");
  float* part = scalar_slots(2L * G, "ivb_vtc_loss_fwd: G too large for the loss scratch");
  if (part == nullptr) return 1;
  if (int rc = launch("vtc_stats_kernel", vtc_stats_kernel, 2 * G, 256, 0, stream, NO_PDL, cos_v2t, idx, G, 1.f / temp,
                      temp_dev, lse_row, lse_col, part))
    return rc;
  return scalar_finish(2 * G, loss, stream);
}

extern "C" int ivb_vtc_loss_bwd(const float* cos_v2t, const long long* idx, int G, float temp,
                                const float* temp_dev,
                                const float* lse_row, const float* lse_col, float gscale_host,
                                const float* gscale_dev, void* dcos_bf16, float* dtemp, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (G <= 0) return 0;
  float* part = nullptr;
  if (dtemp != nullptr && (part = scalar_slots(G, "ivb_vtc_loss_bwd: G too large for the dtemp scratch")) == nullptr)
    return 1;
  if (int rc = launch("vtc_grad_kernel", vtc_grad_kernel, G, 256, 0, stream, NO_PDL, cos_v2t, idx, G, 1.f / temp,
                      temp_dev, lse_row, lse_col, gscale_host, gscale_dev, reinterpret_cast<__nv_bfloat16*>(dcos_bf16),
                      part))
    return rc;
  return scalar_finish(G, dtemp, stream);
}

extern "C" int ivb_l2norm_rows_fwd(const void* x, int x_is_f32, long ldx, int M, int C, void* out,
                                   long ldo, float* inv_norm, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (ldx & 7) || (ldo & 7)) return set_error("ivb_l2norm_rows_fwd: C/ld must be multiples of 8");
  if (misaligned(16, x, out)) return set_error("ivb_l2norm_rows_fwd: x and out must be 16-byte aligned");
  const int wpb = 8;
  const unsigned grid = (M + wpb - 1) / wpb;
  return launch("l2norm_rows_kernel", x_is_f32 ? l2norm_rows_kernel<true> : l2norm_rows_kernel<false>, grid, wpb * 32, 0,
                stream, NO_PDL, x, ldx, M, C, reinterpret_cast<__nv_bfloat16*>(out), ldo, inv_norm);
}

extern "C" int ivb_l2norm_rows_bwd(const float* dy, long lddy, const void* xn, long ldxn,
                                   const float* inv_norm, int M, int C, float* dx, long lddx,
                                   void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (lddy & 7) || (ldxn & 7) || (lddx & 7)) return set_error("ivb_l2norm_rows_bwd: C/ld must be multiples of 8");
  if (misaligned(16, dy, xn, dx)) return set_error("ivb_l2norm_rows_bwd: dy, xn and dx must be 16-byte aligned");
  const int wpb = 8;
  return launch("l2norm_rows_bwd_kernel", l2norm_rows_bwd_kernel, (M + wpb - 1) / wpb, wpb * 32, 0, stream, NO_PDL, dy,
                lddy, reinterpret_cast<const __nv_bfloat16*>(xn), ldxn, inv_norm, M, C, dx, lddx);
}

extern "C" int ivb_pixel_targets(const void* video, const int* masked_idx, int n_mask, int B, int C,
                                 int T, int H, int W, int tubelet, int patch, int normalize,
                                 const float* mean3, const float* std3, float* labels, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || n_mask <= 0) return 0;
  if (C > 8) return set_error("ivb_pixel_targets: at most 8 channels");
  return launch("pixel_target_kernel", pixel_target_kernel, B * n_mask, C * 32, 0, stream, NO_PDL,
                reinterpret_cast<const __nv_bfloat16*>(video), masked_idx, n_mask, B, C, T, H, W, tubelet, patch,
                normalize, mean3, std3, labels);
}

extern "C" int ivb_mse_loss(const void* pred_bf16, const float* label, long n, float* loss_sum,
                            float gscale_host, const float* gscale_dev, void* dpred_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n <= 0) return 0;
  const int grid = persistent_grid(n, 256, 8);
  float* part = nullptr;
  if (loss_sum != nullptr && (part = scalar_slots(grid, "ivb_mse_loss: too many CTAs for the loss scratch")) == nullptr)
    return 1;
  if (int rc = launch("mse_kernel", mse_kernel, grid, 256, 0, stream, NO_PDL,
                      reinterpret_cast<const __nv_bfloat16*>(pred_bf16), label, n, part, gscale_host, gscale_dev,
                      reinterpret_cast<__nv_bfloat16*>(dpred_bf16)))
    return rc;
  return scalar_finish(grid, loss_sum, stream);
}

// ---------------------------------------------------------------- single-query attention pooling
// AttentionPoolingBlock / CrossAttention with ONE query per clip (internvideo2_pretrain.py:61-76, 107-114):
//   s_j = scale * <q_h, k_{j,h}> ; p = softmax_j(s) ; o_h = sum_j p_j v_{j,h}.   One CTA per (head, clip).
namespace ivb {

__global__ void __launch_bounds__(128)
pool_attn_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, long ldk,
                     const __nv_bfloat16* __restrict__ v, long ldv, int n, int H, int d, float scale,
                     __nv_bfloat16* __restrict__ out, float* __restrict__ probs) {
  extern __shared__ float sm[];          // [d] q_h | [n] scores/probs | [4] red
  float* sq = sm;
  float* sp = sm + d;
  float* red = sp + n;
  const int h = blockIdx.x, b = blockIdx.y, D = H * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) sq[i] = __bfloat162float(q[static_cast<long>(b) * D + h * d + i]) * scale;
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const __nv_bfloat16* kr = k + (static_cast<long>(b) * n + j) * ldk + h * d;
    float s = 0.f;
    for (int c = 0; c < d; c += 8) {
      float kv[8];
      load8<false>(kr, c, kv);
#pragma unroll
      for (int t = 0; t < 8; ++t) s += kv[t] * sq[c + t];
    }
    sp[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_reduce<true>(mx, red);
  float se = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) { const float e = __expf(sp[j] - mx); sp[j] = e; se += e; }
  se = block_reduce(se, red);
  const float inv = 1.f / se;
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float pj = sp[j] * inv;
    sp[j] = pj;
    probs[(static_cast<long>(b) * H + h) * n + j] = pj;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float o = 0.f;
    const __nv_bfloat16* vc = v + static_cast<long>(b) * n * ldv + h * d + c;
    for (int j = 0; j < n; ++j) o += sp[j] * __bfloat162float(vc[static_cast<long>(j) * ldv]);
    out[static_cast<long>(b) * D + h * d + c] = __float2bfloat16(o);
  }
}

__global__ void __launch_bounds__(128)
pool_attn_bwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, long ldk,
                     const __nv_bfloat16* __restrict__ v, long ldv, const float* __restrict__ probs,
                     const __nv_bfloat16* __restrict__ dout, int n, int H, int d, float scale,
                     __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dk, long lddk,
                     __nv_bfloat16* __restrict__ dv, long lddv) {
  extern __shared__ float sm[];          // [d] q_h*scale | [d] do_h | [n] ds | [4] red
  float* sq = sm;
  float* sdo = sm + d;
  float* sds = sdo + d;
  float* red = sds + n;
  const int h = blockIdx.x, b = blockIdx.y, D = H * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    sq[i] = __bfloat162float(q[static_cast<long>(b) * D + h * d + i]) * scale;
    sdo[i] = __bfloat162float(dout[static_cast<long>(b) * D + h * d + i]);
  }
  __syncthreads();
  const float* pr = probs + (static_cast<long>(b) * H + h) * n;
  float acc = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const __nv_bfloat16* vr = v + (static_cast<long>(b) * n + j) * ldv + h * d;
    float dp = 0.f;
    for (int c = 0; c < d; c += 8) {
      float vv[8];
      load8<false>(vr, c, vv);
#pragma unroll
      for (int t = 0; t < 8; ++t) dp += vv[t] * sdo[c + t];
    }
    sds[j] = dp;
    acc += pr[j] * dp;
  }
  acc = block_reduce(acc, red);
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float pj = pr[j];
    const float ds = pj * (sds[j] - acc);
    sds[j] = ds;
    __nv_bfloat16* dkr = dk + (static_cast<long>(b) * n + j) * lddk + h * d;
    __nv_bfloat16* dvr = dv + (static_cast<long>(b) * n + j) * lddv + h * d;
    for (int c = 0; c < d; c += 8) {
      float a[8], bb[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) { a[t] = ds * sq[c + t]; bb[t] = pj * sdo[c + t]; }
      store8<false>(dkr, c, a);
      store8<false>(dvr, c, bb);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float g = 0.f;
    const __nv_bfloat16* kc = k + static_cast<long>(b) * n * ldk + h * d + c;
    for (int j = 0; j < n; ++j) g += sds[j] * __bfloat162float(kc[static_cast<long>(j) * ldk]);
    dq[static_cast<long>(b) * D + h * d + c] = __float2bfloat16(g * scale);
  }
}

}  // namespace ivb

extern "C" int ivb_pool_attn_fwd(const void* q, const void* k, long ldk, const void* v, long ldv, int B,
                                 int n, int H, int d, float scale, void* out, float* probs, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0) return 0;
  if ((d & 7) || (ldk & 7) || (ldv & 7)) return set_error("ivb_pool_attn_fwd: d/ld must be multiples of 8");
  if (misaligned(16, k, v)) return set_error("ivb_pool_attn_fwd: k and v must be 16-byte aligned");
  const size_t smem = (static_cast<size_t>(d) + n + 8) * sizeof(float);
  if (smem > 48 * 1024) return set_error("ivb_pool_attn_fwd: sequence too long for the single-query kernel");
  return launch("pool_attn_fwd_kernel", pool_attn_fwd_kernel, dim3(H, B), 128, smem, stream, NO_PDL,
                reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k), ldk,
                reinterpret_cast<const __nv_bfloat16*>(v), ldv, n, H, d, scale, reinterpret_cast<__nv_bfloat16*>(out),
                probs);
}

extern "C" int ivb_pool_attn_bwd(const void* q, const void* k, long ldk, const void* v, long ldv,
                                 const float* probs, const void* dout, int B, int n, int H, int d,
                                 float scale, void* dq, void* dk, long lddk, void* dv, long lddv,
                                 void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0) return 0;
  if ((d & 7) || (ldk & 7) || (ldv & 7) || (lddk & 7) || (lddv & 7)) return set_error("ivb_pool_attn_bwd: d/ld must be multiples of 8");
  if (misaligned(16, k, v, dk, dv)) return set_error("ivb_pool_attn_bwd: k, v, dk and dv must be 16-byte aligned");
  const size_t smem = (2 * static_cast<size_t>(d) + n + 8) * sizeof(float);
  if (smem > 48 * 1024) return set_error("ivb_pool_attn_bwd: sequence too long for the single-query kernel");
  return launch("pool_attn_bwd_kernel", pool_attn_bwd_kernel, dim3(H, B), 128, smem, stream, NO_PDL,
                reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k), ldk,
                reinterpret_cast<const __nv_bfloat16*>(v), ldv, probs, reinterpret_cast<const __nv_bfloat16*>(dout), n,
                H, d, scale, reinterpret_cast<__nv_bfloat16*>(dq), reinterpret_cast<__nv_bfloat16*>(dk), lddk,
                reinterpret_cast<__nv_bfloat16*>(dv), lddv);
}
