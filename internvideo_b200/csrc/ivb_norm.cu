// ivb_norm.cu — HBM-bound row/column reduction kernels of the ViT block:
//   RMSNorm / LayerNorm forward + backward   (internvideo2_pretrain.py:117-128; FA2 DropoutAddRMSNorm
//                                             :467 incl. the q/k-norm over the full C :198-206;
//                                             nn.LayerNorm of the pooling block / decoders :525,:532)
//   LayerScale backward                      (internvideo2_pretrain.py:131-146)
//   bias-gradient column sums
//   decoder head: LayerNorm -> L2-normalise  (Linear_Decoder / MLP_Decoder.forward internvideo2_pretrain.py:355-365,
//                 and the (2 - 2 <out, tgt>).mean() loss   393-403; engines/engine_for_pretraining.py:131-136)
// One warp per row, 16-byte vector loads, warp-shuffle reductions; parameter gradients are
// accumulated per warp in shared memory, stored as one partial per column per CTA and summed in a fixed
// order by colred_finish (ivb_colred.cuh).
// The forward has two kernels: norm_fwd_kernel streams the row (LayerNorm, and RMSNorm above D = 1536, to bf16), and
// norm_rows_kernel holds it in registers and writes it as bf16 (RMSNorm, the q/k pair), as E4M3 with a per-row
// scale (FP8 inference), or as both (FP8 training), all launched by launch_norm_fwd.
// The backward has two kernels too, norm_bwd_kernel (streamed) and norm_bwd_rows_kernel (held in registers), both
// launched by launch_norm_bwd; each also runs the decoder head's LN -> L2 backward, a LayerNorm backward whose dy is
// formed from the upstream gradient.
#include <stdio.h>
#include <stdlib.h>
#include <type_traits>

#include "ivb_colred.cuh"
#include "ivb_fp8.cuh"
#include "ivb_internal.h"
#include "ivb_ptx.cuh"
#include "ivb_rows.cuh"

namespace ivb {

// ------------------------------------------------------------------ forward
template <bool XF32, bool LN>
__global__ void __launch_bounds__(256)
norm_fwd_kernel(const void* __restrict__ x, long ldx, const __nv_bfloat16* __restrict__ w,
                const __nv_bfloat16* __restrict__ b, float eps, int M, int D,
                __nv_bfloat16* __restrict__ y, long ldy, float* __restrict__ mean_out,
                float* __restrict__ rstd_out) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int nch = D >> 3;
  const float invD = 1.0f / static_cast<float>(D);
  for (long row = (long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < M;
       row += (long)gridDim.x * warps_per_block) {
    const long xo = row * ldx;
    float mean = 0.f;
    if (LN) {
      float s = 0.f;
      for (int c = lane; c < nch; c += 32) {
        float v[8];
        load8<XF32>(x, xo + c * 8, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[j];
      }
      mean = warp_sum(s) * invD;
    }
    float ss = 0.f;
    for (int c = lane; c < nch; c += 32) {
      float v[8];
      load8<XF32>(x, xo + c * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[j] - mean; ss += d * d; }
    }
    const float rstd = rsqrtf(warp_sum(ss) * invD + eps);
    for (int c = lane; c < nch; c += 32) {
      float v[8], wv[8], o[8];
      load8<XF32>(x, xo + c * 8, v);
      load8<false>(w, c * 8, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[j] - mean) * rstd * wv[j];
      if (LN && b != nullptr) {
        float bv[8];
        load8<false>(b, c * 8, bv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += bv[j];
      }
      store8<false>(y, row * ldy + c * 8, o);
    }
    if (lane == 0) {
      if (rstd_out) rstd_out[row] = rstd;
      if (LN && mean_out) mean_out[row] = mean;
    }
  }
}

// ------------------------------------------------------------------ decoder head: LayerNorm + L2 normalise
// out = y / ||y||,  y = LN(z) * w + b.   stats[row] = {mean, rstd, 1/||y||}.
// If tgt != nullptr and want_loss, also stores the CTA's sum over its rows of (2 - 2 <out, tgt>)  (engine :131-136)
// in colred slot blockIdx.x, for colred_finish to add into the loss.
template <bool TGT_F32>
__global__ void __launch_bounds__(256)
ln_l2_fwd_kernel(const __nv_bfloat16* __restrict__ z, long ldz, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ bsh, float eps, int M, int C,
                 __nv_bfloat16* __restrict__ out, long ldo, float* __restrict__ stats,
                 const void* __restrict__ tgt, long ldt, bool want_loss) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const float invC = 1.f / C;
  float loss_acc = 0.f;
  for (long row = static_cast<long>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < M;
       row += static_cast<long>(gridDim.x) * wpb) {
    const __nv_bfloat16* zr = z + row * ldz;
    float s = 0.f;
    for (int c = lane * 8; c < C; c += 256) { float v[8]; load8<false>(zr, c, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) s += v[k]; }
    const float mean = warp_sum(s) * invC;
    float ss = 0.f;
    for (int c = lane * 8; c < C; c += 256) { float v[8]; load8<false>(zr, c, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) { const float d = v[k] - mean; ss += d * d; } }
    const float rstd = rsqrtf(warp_sum(ss) * invC + eps);
    float n2 = 0.f, dot = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
      float v[8], wv[8], bv[8];
      load8<false>(zr, c, v); load8<false>(w, c, wv); load8<false>(bsh, c, bv);
      float t[8];
      if (tgt) load8<TGT_F32>(tgt, row * ldt + c, t);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float y = (v[k] - mean) * rstd * wv[k] + bv[k];
        n2 += y * y;
        if (tgt) dot += y * t[k];
      }
    }
    n2 = warp_sum(n2);
    const float inv_n = rsqrtf(n2);
    if (tgt) { dot = warp_sum(dot); loss_acc += 2.f - 2.f * dot * inv_n; }   // the same in every lane
    if (out) {
      for (int c = lane * 8; c < C; c += 256) {
        float v[8], wv[8], bv[8], o[8];
        load8<false>(zr, c, v); load8<false>(w, c, wv); load8<false>(bsh, c, bv);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = ((v[k] - mean) * rstd * wv[k] + bv[k]) * inv_n;
        store8<false>(out, row * ldo + c, o);
      }
    }
    if (lane == 0 && stats) { stats[row * 3 + 0] = mean; stats[row * 3 + 1] = rstd; stats[row * 3 + 2] = inv_n; }
  }
  if (tgt && want_loss) {
    __shared__ float red[8];
    loss_acc = block_reduce(lane == 0 ? loss_acc : 0.f, red);
    if (threadIdx.x == 0) colred_put(0, gridDim.x, blockIdx.x, 1, 0, loss_acc);
  }
}

// ------------------------------------------------------------------ backward
// RMSNorm (LN = false: mean = 0, s1 = 0) / LayerNorm backward of 8 columns of a row; g = dy, xh = normalised x.
// Sweep 1: s1 += g*w, s2 += g*w*xh.
template <bool LN>
__device__ __forceinline__ void norm_bwd_sums8(const float g[8], const float wv[8], const float xh[8], float& s1,
                                               float& s2) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float gj = g[j] * wv[j];
    if (LN) s1 += gj;
    s2 += gj * xh[j];
  }
}
// Sweep 2 (s1, s2 now row means): dx = rstd * (g*w - s1 - xh*s2) (+ dx_in); the warp's colred rows at acc (null: no
// weight gradient) get dweight += g*xh and, for LN, dbias += g.
template <bool LN, bool DXF32>
__device__ __forceinline__ void norm_bwd_dx8(const float g[8], const float wv[8], const float xh[8], float rstd,
                                             float s1, float s2, const float* dx_in, long in_off, void* dx_out,
                                             long out_off, float* acc, int D) {
  float o[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = LN ? rstd * (g[j] * wv[j] - s1 - xh[j] * s2) : rstd * (g[j] * wv[j] - xh[j] * s2);
  if (dx_in != nullptr) {   // its own rounding, as these gradients have always been computed: __fadd_rn keeps
                            // the compiler from contracting the add into the multiply above where it inlines this
    float r[8];
    load8<true>(dx_in, in_off, r);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __fadd_rn(o[j], r[j]);
  }
  store8<DXF32>(dx_out, out_off, o);
  if (acc != nullptr) {
    colred_add<8>(acc, g, xh);
    if (LN) colred_add<8>(acc + D, g);
  }
}

// The decoder head's LN -> L2 backward (the L2 forms) is the LayerNorm backward of dy = inv_n * (g*gs - out*a), where
// out = (xh*w + b) * inv_n is the forward's output, g*gs the gradient reaching it and a = <g*gs, out> over the row:
// ln_l2_dot8 sums a over 8 columns (v = z), and ln_l2_dy8 turns g into dy and sets xh = (z - mean) * rstd.
__device__ __forceinline__ void ln_l2_dot8(const float v[8], const float g[8], const float wv[8], const float bv[8],
                                           float mean, float rstd, float inv_n, float gs, float& a) {
#pragma unroll
  for (int k = 0; k < 8; ++k) a += g[k] * gs * ((v[k] - mean) * rstd * wv[k] + bv[k]) * inv_n;
}
__device__ __forceinline__ void ln_l2_dy8(const float v[8], float g[8], const float wv[8], const float bv[8], float mean,
                                          float rstd, float inv_n, float gs, float a, float xh[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    xh[k] = (v[k] - mean) * rstd;
    const float o = (xh[k] * wv[k] + bv[k]) * inv_n;
    g[k] = inv_n * (g[k] * gs - o * a);
  }
}

// dy and dx_out of the norm forms may be one buffer (the in-place q-norm backward); the LN -> L2 gradient and dz never
// alias, and are declared so.
template <bool NOALIAS>
using GradIn = std::conditional_t<NOALIAS, const __nv_bfloat16* __restrict__, const __nv_bfloat16*>;
template <bool NOALIAS> using GradOut = std::conditional_t<NOALIAS, void* __restrict__, void*>;

// dynamic smem: colred rows [warps][LN ? 2 : 1][D]
// L2 (LN, bf16 x = z and dx, no dx_in): dy is the upstream gradient g, fp32 with GF32, scaled by gscale_host *
// *gscale_dev; mean_in is the forward's stats[M][3] = {mean, rstd, inv_n}, and rstd_in is not read.
template <bool XF32, bool LN, bool DXF32, bool L2, bool GF32>
__global__ void __launch_bounds__(256)
norm_bwd_kernel(GradIn<L2> dy, long lddy, const void* __restrict__ x, long ldx, const __nv_bfloat16* __restrict__ w,
                const __nv_bfloat16* __restrict__ b, const float* __restrict__ mean_in,
                const float* __restrict__ rstd_in, int M, int D, const float* __restrict__ dx_in, long lddx_in,
                GradOut<L2> dx_out, long lddx, float* __restrict__ dweight, float* __restrict__ dbias, float gscale_host,
                const float* __restrict__ gscale_dev) {
  if constexpr (!L2) {   // the L2 forms are launched without PDL
    pdl_wait();
    pdl_launch_dependents();
  }
  extern __shared__ float acc_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  const int nch = D >> 3;
  const float invD = 1.0f / static_cast<float>(D);
  const float gs = L2 ? gscale_host * (gscale_dev ? *gscale_dev : 1.f) : 1.f;
  const bool want_dw = dweight != nullptr;
  float* acc = want_dw ? colred_zero(acc_smem, LN ? 2 : 1, D) : nullptr;
  for (long row = (long)blockIdx.x * warps_per_block + warp; row < M;
       row += (long)gridDim.x * warps_per_block) {
    const long xo = row * ldx;
    const long go = row * lddy;
    float mean = 0.f, rstd, inv_n = 0.f;
    if constexpr (L2) {
      mean = mean_in[row * 3]; rstd = mean_in[row * 3 + 1]; inv_n = mean_in[row * 3 + 2];
    } else {
      rstd = rstd_in[row];
      if (LN) mean = mean_in[row];
    }
    // f(c) for the row's 8-column chunks c = lane, lane + 32, ... in order.  The L2 forms count the loop in columns:
    // counted in chunks, the bf16 form takes 64 registers instead of 48, and counted in columns, the norm forms' code
    // changes.
    auto each_chunk = [&](auto f) {
      if constexpr (L2) {
        for (int col = lane * 8; col < D; col += 256) f(col >> 3);
      } else {
        for (int c = lane; c < nch; c += 32) f(c);
      }
    };
    float a = 0.f;
    if (L2) {
      each_chunk([&](int c) {
        float v[8], g[8], wv[8], bv[8];
        load8<XF32>(x, xo + c * 8, v);
        load8<GF32>(dy, go + c * 8, g);
        load8<false>(w, c * 8, wv);
        load8<false>(b, c * 8, bv);
        ln_l2_dot8(v, g, wv, bv, mean, rstd, inv_n, gs, a);
      });
      a = warp_sum(a);
    }
    // chunk c's dy, weights and normalised x, for each of the two sweeps
    auto chunk = [&](int c, float g[8], float wv[8], float xh[8]) {
      float v[8];
      load8<XF32>(x, xo + c * 8, v);
      load8<GF32>(dy, go + c * 8, g);
      load8<false>(w, c * 8, wv);
      if (L2) {
        float bv[8];
        load8<false>(b, c * 8, bv);
        ln_l2_dy8(v, g, wv, bv, mean, rstd, inv_n, gs, a, xh);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) xh[j] = (v[j] - mean) * rstd;
      }
    };
    float s1 = 0.f, s2 = 0.f;  // sum dy*w, sum dy*w*xhat
    each_chunk([&](int c) {
      float g[8], wv[8], xh[8];
      chunk(c, g, wv, xh);
      norm_bwd_sums8<LN>(g, wv, xh, s1, s2);
    });
    s1 = LN ? warp_sum(s1) * invD : 0.f;
    s2 = warp_sum(s2) * invD;
    each_chunk([&](int c) {
      float g[8], wv[8], xh[8];
      chunk(c, g, wv, xh);
      norm_bwd_dx8<LN, DXF32>(g, wv, xh, rstd, s1, s2, L2 ? nullptr : dx_in, row * lddx_in + c * 8, dx_out,
                              row * lddx + c * 8, want_dw ? acc + c * 8 : nullptr, D);
    });
  }
  if (want_dw) {
    __syncthreads();
    colred_flush<LN ? 2 : 1>(acc_smem, warps_per_block, D, dbias != nullptr ? 3u : 1u);
  }
}

// ------------------------------------------------------------------ LayerScale backward / column sums
// CTA = 8 warps; CTA handles a 256-column strip x 64 rows; lane owns 8 columns.
template <bool HAS_Y>
__global__ void __launch_bounds__(256)
layerscale_bwd_kernel(const float* __restrict__ dx, long lddx, const __nv_bfloat16* __restrict__ y,
                      long ldy, const __nv_bfloat16* __restrict__ gamma, int M, int D,
                      __nv_bfloat16* __restrict__ dy, long lddy, float* __restrict__ dgamma,
                      float* __restrict__ dcolsum, int nstrips, const float* __restrict__ rowscale) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[2][8][256];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int strip = blockIdx.x % nstrips;
  const int rb = blockIdx.x / nstrips;
  const int col = strip * 256 + lane * 8;
  const bool col_ok = col < D;
  float ag[8], as[8], gm[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { ag[j] = 0.f; as[j] = 0.f; gm[j] = 1.f; }
  if (col_ok && gamma != nullptr) load8<false>(gamma, col, gm);
  if (col_ok) {
    for (int r = rb * 64 + warp; r < min(M, rb * 64 + 64); r += 8) {
      float d[8], o[8];
      load8<true>(dx, (long)r * lddx + col, d);
      if (rowscale != nullptr) {
        const float rs = rowscale[r];
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] *= rs;
      }
      if (HAS_Y) {
        float yv[8];
        load8<false>(y, (long)r * ldy + col, yv);
#pragma unroll
        for (int j = 0; j < 8; ++j) ag[j] += d[j] * yv[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { as[j] += d[j]; o[j] = d[j] * gm[j]; }
      store8<false>(dy, (long)r * lddy + col, o);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { red[0][warp][lane * 8 + j] = ag[j]; red[1][warp][lane * 8 + j] = as[j]; }
  __syncthreads();
  const int c = threadIdx.x;  // 256 columns of the strip
  if (strip * 256 + c < D) {
    float sg = 0.f, ss = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { sg += red[0][k][c]; ss += red[1][k][c]; }
    const int nrb = gridDim.x / nstrips;
    if (HAS_Y && dgamma != nullptr) colred_put(0, nrb, rb, D, strip * 256 + c, sg);
    // bias gradient of the branch Linear: d/db [gamma * (acc + b)] = gamma * sum_m dx'
    if (dcolsum != nullptr)
      colred_put(1, nrb, rb, D, strip * 256 + c, gamma != nullptr ? ss * __bfloat162float(gamma[strip * 256 + c]) : ss);
  }
}

__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M, int N,
                   float* __restrict__ out, int nstrips, int rows_per_cta) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[8][256];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int strip = blockIdx.x % nstrips;
  const int rb = blockIdx.x / nstrips;
  const int col = strip * 256 + lane * 8;
  float a[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = 0.f;
  if (col < N) {
    const int r1 = min(M, (rb + 1) * rows_per_cta);
    for (int r = rb * rows_per_cta + warp; r < r1; r += 8) {
      float v[8];
      load8<false>(x, (long)r * ldx + col, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = a[j];
  __syncthreads();
  const int c = threadIdx.x;
  if (strip * 256 + c < N) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k][c];
    colred_put(0, gridDim.x / nstrips, rb, N, strip * 256 + c, s);
  }
}


// ------------------------------------------------------------------ register-resident rows (D <= 256*NCH)
// norm_fwd_kernel streams every row twice (statistics pass + output pass, the second from L1/L2).  Where the row fits
// in registers (the block norms, D = 384..1536, and the FP8 forms up to IVB_NORM_FP8_MAX_D) one warp holds it: one HBM
// read per operand, and the row's amax, and with it the row's power-of-two E4M3 scale (fp8_scale), is known before the
// first byte is stored.  The statistics and y = (x - mean) * rstd * w (+ b) are the fp32 expressions of
// norm_fwd_kernel (RMSNorm: mean = 0, and v - 0.f == v exactly), so every form holds the row ivb_norm_fwd rounds to bf16.
// OUT is what the row becomes:
//   NORM_Y   the bf16 row y, and rstd and (LN) mean where their pointers are non-null (ivb_norm_fwd, RMSNorm);
//   NORM_Q   only the E4M3 row q and its scale_inv: the frozen towers' FP8 inference writes no bf16 row;
//   NORM_QY  both, for FP8 training with per-token scales: the weight gradient reads the bf16 row y, the norm backward
//            mean and rstd.
// PAIR (NORM_Y only): the q-norm and the k-norm of a block in ONE launch (internvideo2_pretrain.py:198-206).  Virtual
// row r covers token r>>1, part r&1; part p reads/writes at column offset p*pair_off of its token's row and uses weight
// w / w1.  rstd_out is indexed by the virtual row ([M][2]).  (Two 37 MB launches were each ~3x off the HBM time.)
enum NormOut { NORM_Y, NORM_Q, NORM_QY };

template <bool XF32, bool LN, int NCH, NormOut OUT, bool PAIR>
__global__ void __launch_bounds__(256)
norm_rows_kernel(const void* __restrict__ x, long ldx, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ b, float eps, int M, int D, __nv_bfloat16* __restrict__ y, long ldy,
                 float* __restrict__ mean_out, float* __restrict__ rstd_out, uint8_t* __restrict__ q, long ldq,
                 float* __restrict__ q_scale_inv, const __nv_bfloat16* __restrict__ w1, long x_pair_off,
                 long y_pair_off) {
  static_assert(!PAIR || OUT == NORM_Y, "norm_rows_kernel: PAIR writes bf16 rows only");
  constexpr bool kQ = OUT != NORM_Y, kY = OUT != NORM_Q;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int nch = D >> 3;
  const float invD = 1.0f / static_cast<float>(D);
  for (long row = (long)blockIdx.x * wpb + (threadIdx.x >> 5); row < M; row += (long)gridDim.x * wpb) {
    const long tok = PAIR ? (row >> 1) : row;
    const int part = PAIR ? static_cast<int>(row & 1) : 0;
    const long xo = tok * ldx + part * x_pair_off;
    // y's offset is formed at the store: held from here, it cost the E4M3 + bf16 form two registers
    auto yo = [&](int c) { return tok * ldy + part * y_pair_off + c * 8; };
    const __nv_bfloat16* wp = (PAIR && part) ? w1 : w;
    // The bf16 RMSNorm sums the squares as its chunks arrive, the other forms once the row is loaded: the same sums in
    // the same order, and each form keeps its schedule.  The other order costs the bf16 NCH-6 form 4 registers, and
    // the E4M3 RMSNorm of bf16 rows at D = 3200 1.6 % of its time (73.7 against 72.5 us at M = 13344; H100 SXM 80 GB,
    // 700 W power limit).
    constexpr bool kSumAtLoad = !kQ && !LN;
    float v[NCH][8];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i)
      if (lane + 32 * i < nch) {
        load8<XF32>(x, xo + (lane + 32 * i) * 8, v[i]);
        if (kSumAtLoad) {
#pragma unroll
          for (int j = 0; j < 8; ++j) ss += v[i][j] * v[i][j];
        }
      }
    float mean = 0.f;
    if (LN) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NCH; ++i)
        if (lane + 32 * i < nch) {
#pragma unroll
          for (int j = 0; j < 8; ++j) s += v[i][j];
        }
      mean = warp_sum(s) * invD;
    }
    if (!kSumAtLoad) {
#pragma unroll
      for (int i = 0; i < NCH; ++i)
        if (lane + 32 * i < nch) {
#pragma unroll
          for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; ss += d * d; }
        }
    }
    const float rstd = rsqrtf(warp_sum(ss) * invD + eps);
    unsigned m = 0;   // fp32 magnitude bits: NaN > Inf > every finite value
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float wv[8], t[8];
        float* o = kQ ? v[i] : t;   // the E4M3 forms keep the row in v until its scale is known
        load8<false>(wp, c * 8, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * wv[j];
        if (LN && b != nullptr) {
          float bv[8];
          load8<false>(b, c * 8, bv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += bv[j];
        }
        if constexpr (kQ) {
#pragma unroll
          for (int j = 0; j < 8; ++j) m = max(m, __float_as_uint(o[j]) & 0x7fffffffu);
        } else {
          store8<false>(y, yo(c), o);
        }
      }
    }
    if constexpr (kQ) {
      m = __reduce_max_sync(0xffffffffu, m);
      float scale, sinv;
      fp8_scale(m, 8, scale, sinv);
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const int c = lane + 32 * i;
        if (c < nch) {
          *reinterpret_cast<uint2*>(q + row * ldq + c * 8) = cvt_e4m3x8(v[i], scale);
          if constexpr (kY) store8<false>(y, yo(c), v[i]);
        }
      }
      if (lane == 0) q_scale_inv[row] = sinv;
    }
    if (kY && lane == 0) {   // NORM_QY: the caller guarantees rstd_out and (LN) mean_out
      if (kQ || rstd_out) rstd_out[row] = rstd;
      if (LN && (kQ || mean_out)) mean_out[row] = mean;
    }
  }
}

// The backward over rows held in registers (D <= 256*NCH): RMSNorm, the q/k pair and, with L2, the LN -> L2 backward
// (operands as in norm_bwd_kernel).  Each row is read from HBM once, all its loads in flight together.
// dynamic smem: colred rows [warps][L2 ? 2 : 1][D] (only when dweight != nullptr)
// PAIR: virtual row r covers token r>>1, part r&1; part p reads and writes at column offset p*pair_off of its token's
// rows and uses weight w / w1; its weight gradient is the pair's second colred output.
template <bool XF32, bool DXF32, int NCH, bool PAIR, bool L2>
__global__ void __launch_bounds__(L2 ? 128 : 256, 2)
norm_bwd_rows_kernel(GradIn<L2> dy, long lddy, const void* __restrict__ x, long ldx, const __nv_bfloat16* __restrict__ w,
                     const __nv_bfloat16* __restrict__ b, const float* __restrict__ mean_in,
                     const float* __restrict__ rstd_in, int M, int D, const float* __restrict__ dx_in, long lddx_in,
                     GradOut<L2> dx_out, long lddx, float* __restrict__ dweight, float* __restrict__ dbias, float gscale_host,
                     const float* __restrict__ gscale_dev, const __nv_bfloat16* __restrict__ w1, long x_pair_off,
                     long dy_pair_off, long dx_pair_off) {
  // What a row is held as.  RMSNorm and the pair hold the normalised row in fp32 (8*NCH registers) and dy as the raw
  // packed bf16 it was loaded as (4*NCH): keeping dy*w in fp32 as well pushed the kernel to 150 registers / 1 CTA per
  // SM and made it 2x slower.  LN -> L2 holds z and g packed and forms xh and dy again in each sweep: its 13-chunk rows
  // at C = 3200 do not fit in registers as fp32.
  constexpr bool kHoldXh = !L2;
  if constexpr (!L2) {   // the L2 form is launched without PDL
    pdl_wait();
    pdl_launch_dependents();
  }
  extern __shared__ float acc_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int nch = D >> 3;
  const float invD = 1.0f / static_cast<float>(D);
  const float gs = L2 ? gscale_host * (gscale_dev ? *gscale_dev : 1.f) : 1.f;
  const bool want_dw = dweight != nullptr;
  float* acc = want_dw ? colred_zero(acc_smem, L2 ? 2 : 1, D) : nullptr;
  // PAIR: the virtual-row stride gridDim.x * wpb is even (wpb = 8), so a warp only ever sees ONE part
  // (row parity == warp parity): its accumulator belongs to that part's weight gradient.
  for (long row = (long)blockIdx.x * wpb + warp; row < M; row += (long)gridDim.x * wpb) {
    const long tok = PAIR ? (row >> 1) : row;
    const int part = PAIR ? static_cast<int>(row & 1) : 0;
    const long xo = tok * ldx + part * x_pair_off;
    const long go = tok * lddy + part * dy_pair_off;
    const long oo = tok * lddx + part * dx_pair_off;
    const __nv_bfloat16* wp = (PAIR && part) ? w1 : w;
    float mean = 0.f, rstd = L2 ? 0.f : rstd_in[row], inv_n = 0.f;   // L2: read after the row is in flight
    float xh[kHoldXh ? NCH : 1][8];
    uint4 zq[kHoldXh ? 1 : NCH], gq[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        if constexpr (kHoldXh) load8<XF32>(x, xo + c * 8, xh[i]);
        else zq[i] = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(x) + xo + c * 8);
        gq[i] = *reinterpret_cast<const uint4*>(dy + go + c * 8);
      }
    }
    float a = 0.f;
    if constexpr (L2) {
      mean = mean_in[row * 3]; rstd = mean_in[row * 3 + 1]; inv_n = mean_in[row * 3 + 2];
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const int c = lane + 32 * i;
        if (c < nch) {
          float v[8], g[8], wv[8], bv[8];
          unpack8(zq[i], v);
          unpack8(gq[i], g);
          load8<false>(w, c * 8, wv);
          load8<false>(b, c * 8, bv);
          ln_l2_dot8(v, g, wv, bv, mean, rstd, inv_n, gs, a);
        }
      }
      a = warp_sum(a);
    }
    // chunk i's dy and weights; returns its normalised x, held or formed in xl
    auto chunk = [&](int i, float g[8], float wv[8], float xl[8]) -> const float* {
      const int c = lane + 32 * i;
      if constexpr (kHoldXh) {
        load8<false>(wp, c * 8, wv);
        unpack8(gq[i], g);
        return xh[i];
      } else {
        float v[8], bv[8];
        unpack8(zq[i], v);
        unpack8(gq[i], g);
        load8<false>(w, c * 8, wv);
        load8<false>(b, c * 8, bv);
        ln_l2_dy8(v, g, wv, bv, mean, rstd, inv_n, gs, a, xl);
        return xl;
      }
    };
    float s1 = 0.f, s2 = 0.f;  // s1 stays 0 (RMSNorm)
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      if (lane + 32 * i < nch) {
        float g[8], wv[8], xl[8];
        const float* xhi = chunk(i, g, wv, xl);
        if constexpr (kHoldXh) {
#pragma unroll
          for (int j = 0; j < 8; ++j) xh[i][j] *= rstd;
        }
        norm_bwd_sums8<L2>(g, wv, xhi, s1, s2);
      }
    }
    s1 = L2 ? warp_sum(s1) * invD : 0.f;
    s2 = warp_sum(s2) * invD;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float g[8], wv[8], xl[8];
        const float* xhi = chunk(i, g, wv, xl);
        norm_bwd_dx8<L2, DXF32>(g, wv, xhi, rstd, s1, s2, L2 ? nullptr : dx_in, row * lddx_in + c * 8, dx_out,
                                oo + c * 8, want_dw ? acc + c * 8 : nullptr, D);
      }
    }
  }
  if (want_dw) {
    __syncthreads();
    colred_flush<L2 ? 2 : 1, PAIR ? 2 : 1>(acc_smem, wpb, D, PAIR || dbias != nullptr ? 3u : 1u);
  }
}

// ------------------------------------------------------------------ bulk-copy (TMA) row pipeline
// Every warp owns a ring of TMA_NBUF row slots in shared memory that lane 0 keeps full with cp.async.bulk (1-D bulk
// copies completing on per-slot mbarriers); the arithmetic reads the row from shared memory (conflict-free 16-byte
// lanes), so four input rows per token cost no registers.  It is used where it removes a whole kernel: the backward
// fused with the LayerScale backward.

// RMSNorm backward on the fp32 stream FUSED with the LayerScale backward that follows it in the block
// (Block.backward: dx = rmsnorm_bwd(dy, x) + dx_in is the gradient of the residual stream, which the preceding branch's
// LayerScale consumes at once: dyb = rs * gamma * dx, dgamma += sum rs*dx*ybr, dcolsum += gamma * sum rs*dx):
//   inputs per row: dy bf16 [D], x fp32 [D], dx_in fp32 [D] (optional), ybr bf16 [D]
//   outputs: dx fp32 [D], dyb bf16 [D]
// The separate layerscale_bwd kernel re-read dx (4 D bytes/row) and ran at 0.62 of the HBM rate; fused, the
// gradient of the stream never makes that extra round trip.
constexpr int TMA_NW = 4, TMA_NBUF = 2;   // 8 rows in flight per SM

// smem: row slots [warp][TMA_NBUF][slot] + colred rows [warp][3][D] fp32 (dweight, dgamma, dcolsum) + mbarriers
static size_t rms_bwd_tma_smem(int D, bool has_in) {
  const size_t slot = static_cast<size_t>(D) * (4 + 2 + (has_in ? 4 : 0) + 2);
  return TMA_NW * TMA_NBUF * slot + static_cast<size_t>(TMA_NW) * 3 * D * 4 + TMA_NW * TMA_NBUF * 8;
}

__global__ void __launch_bounds__(128, 1)
rms_bwd_tma_kernel(const __nv_bfloat16* __restrict__ dy, long lddy, const float* __restrict__ x, long ldx,
                   const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd_in, int M, int D,
                   const float* __restrict__ dx_in, long lddx_in, float* __restrict__ dx_out, long lddx,
                   float* __restrict__ dweight,
                   const __nv_bfloat16* __restrict__ ybr, long ldyb, const __nv_bfloat16* __restrict__ gamma,
                   const float* __restrict__ rowscale, __nv_bfloat16* __restrict__ dyb, long lddyb,
                   float* __restrict__ dgamma, float* __restrict__ dcolsum) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(128) uint8_t rt_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool has_in = dx_in != nullptr;
  const uint32_t by_dy = static_cast<uint32_t>(D) * 2u, by_x = static_cast<uint32_t>(D) * 4u;
  const uint32_t slot = by_x + by_dy + (has_in ? by_x : 0u) + by_dy;      // bytes per buffered row
  uint8_t* base = rt_smem + static_cast<long>(warp) * TMA_NBUF * slot;
  float* accs = reinterpret_cast<float*>(rt_smem + static_cast<long>(TMA_NW) * TMA_NBUF * slot);
  uint64_t* bars = reinterpret_cast<uint64_t*>(rt_smem + static_cast<long>(TMA_NW) * TMA_NBUF * slot +
                                               static_cast<long>(TMA_NW) * 3 * D * 4) + warp * TMA_NBUF;
  const long W = static_cast<long>(gridDim.x) * TMA_NW;
  const long gw = static_cast<long>(blockIdx.x) * TMA_NW + warp;
  auto fill = [&](int b, long row) {
    uint8_t* s0 = base + static_cast<long>(b) * slot;
    mbar_expect_tx(&bars[b], slot);
    bulk_load_1d(s0, x + row * ldx, by_x, &bars[b]);
    bulk_load_1d(s0 + by_x, dy + row * lddy, by_dy, &bars[b]);
    uint32_t off = by_x + by_dy;
    if (has_in) { bulk_load_1d(s0 + off, dx_in + row * lddx_in, by_x, &bars[b]); off += by_x; }
    bulk_load_1d(s0 + off, ybr + row * ldyb, by_dy, &bars[b]);
  };
  float* acc = colred_zero(accs, 3, D);
  if (lane == 0) {
#pragma unroll
    for (int b = 0; b < TMA_NBUF; ++b) mbar_init(&bars[b], 1);
    fence_mbar_init();
#pragma unroll
    for (int b = 0; b < TMA_NBUF; ++b) {
      const long row = gw + b * W;
      if (row < M) fill(b, row);
    }
  }
  __syncwarp();
  const int nq = D >> 2;
  const float invD = 1.0f / static_cast<float>(D);
  long it = 0;
  for (long row = gw; row < M; row += W, ++it) {
    const int b = static_cast<int>(it % TMA_NBUF);
    mbar_wait(&bars[b], static_cast<uint32_t>((it / TMA_NBUF) & 1));
    const uint8_t* s0 = base + static_cast<long>(b) * slot;
    const float4* xs = reinterpret_cast<const float4*>(s0);
    const uint2* gs = reinterpret_cast<const uint2*>(s0 + by_x);
    const float4* rs_in = reinterpret_cast<const float4*>(s0 + by_x + by_dy);
    const uint2* ys = reinterpret_cast<const uint2*>(s0 + by_x + by_dy + (has_in ? by_x : 0u));
    const float rstd = rstd_in[row];
    float s2 = 0.f;
    for (int g = lane; g < nq; g += 32) {
      const float4 a = xs[g];
      const uint2 gq = gs[g], wq = *reinterpret_cast<const uint2*>(w + g * 4);
      const float2 g0 = unpack_bf16(gq.x), g1 = unpack_bf16(gq.y), w0 = unpack_bf16(wq.x), w1 = unpack_bf16(wq.y);
      s2 += g0.x * w0.x * a.x + g0.y * w0.y * a.y + g1.x * w1.x * a.z + g1.y * w1.y * a.w;
    }
    s2 = warp_sum(s2) * rstd * invD;             // mean(g*w*xhat), xhat = x*rstd
    const float rsc = rowscale ? rowscale[row] : 1.f;
    float* dxr = dx_out + row * lddx;
    for (int g = lane; g < nq; g += 32) {
      const float4 a = xs[g];
      const uint2 gq = gs[g], wq = *reinterpret_cast<const uint2*>(w + g * 4);
      const float2 g0 = unpack_bf16(gq.x), g1 = unpack_bf16(gq.y), w0 = unpack_bf16(wq.x), w1 = unpack_bf16(wq.y);
      const float gv[4] = {g0.x, g0.y, g1.x, g1.y};
      const float xh[4] = {a.x * rstd, a.y * rstd, a.z * rstd, a.w * rstd};
      float4 o;
      o.x = rstd * (g0.x * w0.x - xh[0] * s2); o.y = rstd * (g0.y * w0.y - xh[1] * s2);
      o.z = rstd * (g1.x * w1.x - xh[2] * s2); o.w = rstd * (g1.y * w1.y - xh[3] * s2);
      if (has_in) {   // its own rounding, as this gradient has always been computed: __fadd_rn keeps the
                      // compiler's copy of the loop for has_in from contracting the add into the multiply above
        const float4 r = rs_in[g];
        o.x = __fadd_rn(o.x, r.x); o.y = __fadd_rn(o.y, r.y); o.z = __fadd_rn(o.z, r.z); o.w = __fadd_rn(o.w, r.w);
      }
      *reinterpret_cast<float4*>(dxr + g * 4) = o;
      colred_add<4>(acc + g * 4, gv, xh);
      const uint2 yq = ys[g], gmq = *reinterpret_cast<const uint2*>(gamma + g * 4);
      const float2 y0 = unpack_bf16(yq.x), y1 = unpack_bf16(yq.y), m0 = unpack_bf16(gmq.x), m1 = unpack_bf16(gmq.y);
      const float yv[4] = {y0.x, y0.y, y1.x, y1.y};
      const float d[4] = {o.x * rsc, o.y * rsc, o.z * rsc, o.w * rsc};
      uint2 ob;
      ob.x = pack_bf16(d[0] * m0.x, d[1] * m0.y); ob.y = pack_bf16(d[2] * m1.x, d[3] * m1.y);
      *reinterpret_cast<uint2*>(dyb + row * lddyb + g * 4) = ob;
      colred_add<4>(acc + D + g * 4, d, yv);
      colred_add<4>(acc + 2 * D + g * 4, d);
    }
    __syncwarp();
    const long nxt = row + static_cast<long>(TMA_NBUF) * W;
    if (lane == 0 && nxt < M) fill(b, nxt);
  }
  __syncthreads();
  colred_flush<3>(accs, TMA_NW, D, (dweight ? 1u : 0u) | (dgamma ? 2u : 0u) | (dcolsum ? 4u : 0u), gamma);
}

static int launch_rms_bwd_tma(const void* dy, long lddy, const void* x, long ldx, const void* w, const float* rstd, int M,
                              int D, const float* dx_in, long lddx_in, void* dx_out, long lddx, float* dweight,
                              const void* ybr, long ldyb, const void* gamma, const float* rowscale, void* dyb, long lddyb,
                              float* dgamma, float* dcolsum, cudaStream_t stream) {
  if (int rc = raise_smem_limit<rms_bwd_tma_kernel>(226 * 1024, "cudaFuncSetAttribute(rms_bwd_tma)")) return rc;
  const int grid = persistent_grid(M, TMA_NW, 1);
  if (colred_check(3, grid, D, "rms_bwd_tma: gradient scratch too small")) return 1;
  if (int rc = launch("rms_bwd_tma_kernel", rms_bwd_tma_kernel, grid, TMA_NW * 32, rms_bwd_tma_smem(D, dx_in != nullptr),
                      stream, ALLOW_PDL,
                      reinterpret_cast<const __nv_bfloat16*>(dy), lddy, reinterpret_cast<const float*>(x), ldx,
                      reinterpret_cast<const __nv_bfloat16*>(w), rstd, M, D, dx_in, lddx_in,
                      reinterpret_cast<float*>(dx_out), lddx, dweight,
                      reinterpret_cast<const __nv_bfloat16*>(ybr), ldyb,
                      reinterpret_cast<const __nv_bfloat16*>(gamma), rowscale,
                      reinterpret_cast<__nv_bfloat16*>(dyb), lddyb, dgamma, dcolsum))
    return rc;
  return colred_finish(3, grid, D, dweight, dgamma, dcolsum, stream);
}

// Runtime flags and row widths to template arguments: f(std::bool_constant<b>{}), and f(NCH) for the
// register-resident row kernels, whose rows hold NCH 256-column chunks: pick_nch<L...> picks the first L with
// D <= 256 * L, else the last.
template <typename F>
static auto pick_bool(bool b, F f) { return b ? f(std::true_type{}) : f(std::false_type{}); }
template <int L, int... Ls, typename F>
static int pick_nch(int D, F f) {
  if constexpr (sizeof...(Ls) == 0) return f(std::integral_constant<int, L>{});
  else return D <= 256 * L ? f(std::integral_constant<int, L>{}) : pick_nch<Ls...>(D, f);
}

// The operands of one norm forward; outputs that are null are not written.  q: the E4M3 row (NORM_Q / NORM_QY);
// w1 and the pair offsets: the second part of a PAIR launch.
struct NormFwd {
  const void* x; long ldx; bool x_f32;
  const void* w; const void* b; float eps; bool ln; int M; int D;
  void* y; long ldy; float* mean; float* rstd;
  void* q = nullptr; long ldq = 0; float* q_scale_inv = nullptr;
  const void* w1 = nullptr; long x_pair_off = 0, y_pair_off = 0;
};

// The one forward launch path.  NORM_Y: RMSNorm rows up to D = 1536 (and every PAIR launch) on the register-resident
// kernel, read from HBM exactly once; LayerNorm and wider RMSNorm rows on the streaming norm_fwd_kernel.  The E4M3
// forms always hold the row in registers.
template <NormOut OUT, bool PAIR = false>
static int launch_norm_fwd(const NormFwd& a, cudaStream_t stream) {
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(a.w);
  const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(a.b);
  __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(a.y);
  const long rows = PAIR ? 2L * a.M : a.M;
  const int blocks = persistent_grid(rows, 8, 8);
  auto in_registers = [&](auto xf, auto ln) {
    // bf16 rows up to D = 1536, the E4M3 forms up to IVB_NORM_FP8_MAX_D = 4096
    return pick_nch<2, 4, 6, OUT == NORM_Y ? 6 : 16>(a.D, [&](auto nch) {
      return launch("norm_rows_kernel", norm_rows_kernel<xf, ln, nch, OUT, PAIR>, blocks, 256, 0, stream, ALLOW_PDL,
                    a.x, a.ldx, w, b, a.eps, (int)rows, a.D, y, a.ldy, a.mean, a.rstd,
                    reinterpret_cast<uint8_t*>(a.q), a.ldq, a.q_scale_inv,
                    reinterpret_cast<const __nv_bfloat16*>(a.w1), a.x_pair_off, a.y_pair_off);
    });
  };
  if constexpr (PAIR) {   // the q/k norms: RMSNorm of bf16 rows
    return in_registers(std::false_type{}, std::false_type{});
  } else {
    return pick_bool(a.x_f32, [&](auto xf) {
      if constexpr (OUT == NORM_Y) {
        if (!a.ln && a.D <= 1536) return in_registers(xf, std::false_type{});
        return pick_bool(a.ln, [&](auto ln) {
          return launch("norm_fwd_kernel", norm_fwd_kernel<xf, ln>, blocks, 256, 0, stream, ALLOW_PDL, a.x, a.ldx, w, b,
                        a.eps, a.M, a.D, y, a.ldy, a.mean, a.rstd);
        });
      } else {
        return pick_bool(a.ln, [&](auto ln) { return in_registers(xf, ln); });
      }
    });
  }
}

// The operands of one norm backward; dw and db may be null.  l2: the decoder head's LN -> L2 backward (see
// norm_bwd_kernel); gs and gs_dev scale its gradient dy.  w1, dw1 and the pair offsets: the second part of a PAIR launch.
struct NormBwd {
  const void* dy; long lddy; bool dy_f32;
  const void* x; long ldx; bool x_f32;
  const void* w; const void* b; const float* mean; const float* rstd; bool ln; int M; int D;
  const float* dx_in; long lddx_in; void* dx; long lddx; bool dx_f32;
  float* dw; float* db;
  bool l2 = false; float gs = 1.f; const float* gs_dev = nullptr;
  const void* w1 = nullptr; float* dw1 = nullptr; long x_pair_off = 0, dy_pair_off = 0, dx_pair_off = 0;
};

// Launches Kern, first raising its shared-memory limit to `limit` where smem passes the default 48 KB.
template <auto Kern, typename... Args>
static int launch_smem(const char* name, int limit, int grid, int threads, size_t smem, cudaStream_t stream,
                       LaunchPdl pdl, Args... args) {
  if (smem > 48 * 1024)
    if (int rc = raise_smem_limit<Kern>(limit, "cudaFuncSetAttribute(norm_bwd)")) return rc;
  return launch(name, Kern, grid, threads, smem, stream, pdl, args...);
}

// The one backward launch path.  norm_bwd_rows_kernel reads each row from HBM once: RMSNorm rows up to D = 1536, every
// PAIR launch, and LN -> L2 rows of a bf16 gradient up to C = 3328; norm_bwd_kernel streams the rest.  The weight and
// bias gradients are summed per warp in shared memory (nacc rows of D per warp) and then across CTAs by colred_finish.
template <bool PAIR = false>
static int launch_norm_bwd(const NormBwd& a, cudaStream_t stream) {
  const bool in_registers = PAIR || (!a.ln && a.D <= 1536) || (a.l2 && !a.dy_f32 && a.D <= 256 * 13);
  const long rows = PAIR ? 2L * a.M : a.M;
  const int nacc = a.ln ? 2 : 1;
  int wpb = in_registers && a.l2 ? 4 : 8;
  size_t smem = a.dw ? static_cast<size_t>(nacc) * wpb * a.D * sizeof(float) : 0;
  while (smem > 200 * 1024 && wpb > 1) { wpb /= 2; smem /= 2; }   // streaming rows only: the register forms need <= 104 KB
  // >= 2 rows per warp so the shared-memory flush amortises.  The register forms run 2 CTAs per SM, one persistent
  // wave; the streaming one keeps ~32 warps/SM in flight: it is pure HBM streaming and latency-bound below that
  // (measured 2.8x off the HBM time with 1.4 CTAs/SM).
  const int grid = in_registers ? persistent_grid(rows, 2 * wpb, 2) : persistent_grid(a.M, 2 * wpb, smem > 96 * 1024 ? 2 : 4);
  if (colred_check(2, grid, a.D, a.l2 ? "ln_l2_bwd: gradient scratch too small" : "norm_bwd: gradient scratch too small"))
    return 1;
  const LaunchPdl pdl = a.l2 ? NO_PDL : ALLOW_PDL;
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(a.w);
  const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(a.b);
  const __nv_bfloat16* dy = reinterpret_cast<const __nv_bfloat16*>(a.dy);   // or fp32 (L2 with dy_f32)
  auto streamed = [&](auto xf, auto ln, auto dxf, auto l2, auto gf) {
    return launch_smem<norm_bwd_kernel<xf, ln, dxf, l2, gf>>(
        "norm_bwd_kernel", 220 * 1024, grid, wpb * 32, smem, stream, pdl, dy, a.lddy, a.x, a.ldx, w, b, a.mean, a.rstd,
        a.M, a.D, a.dx_in, a.lddx_in, a.dx, a.lddx, a.dw, a.db, a.gs, a.gs_dev);
  };
  auto in_regs = [&](auto xf, auto dxf, auto nch, auto l2) {
    return launch_smem<norm_bwd_rows_kernel<xf, dxf, nch, PAIR, l2>>(
        "norm_bwd_rows_kernel", 110 * 1024, grid, wpb * 32, smem, stream, pdl, dy, a.lddy, a.x, a.ldx, w, b, a.mean,
        a.rstd, (int)rows, a.D, a.dx_in, a.lddx_in, a.dx, a.lddx, a.dw, a.db, a.gs, a.gs_dev,
        reinterpret_cast<const __nv_bfloat16*>(a.w1), a.x_pair_off, a.dy_pair_off, a.dx_pair_off);
  };
  constexpr std::false_type F{};
  constexpr std::true_type T{};
  int rc;
  if constexpr (PAIR) {   // the q/k norms: RMSNorm of bf16 rows
    rc = pick_nch<2, 4, 6>(a.D, [&](auto nch) { return in_regs(F, F, nch, F); });
  } else if (a.l2) {   // LayerNorm of bf16 z to bf16 dz
    rc = in_registers ? pick_nch<3, 6, 13>(a.D, [&](auto nch) { return in_regs(F, F, nch, T); })
                      : pick_bool(a.dy_f32, [&](auto gf) { return streamed(F, T, F, T, gf); });
  } else {
    rc = pick_bool(a.x_f32, [&](auto xf) {
      return pick_bool(a.dx_f32, [&](auto dxf) {
        if (in_registers) return pick_nch<2, 4, 6>(a.D, [&](auto nch) { return in_regs(xf, dxf, nch, F); });
        return pick_bool(a.ln, [&](auto ln) { return streamed(xf, ln, dxf, F, F); });
      });
    });
  }
  float* out1 = PAIR ? a.dw1 : a.ln ? a.db : nullptr;   // the second gradient: the pair's second weight, or the bias
  if (rc != 0 || a.dw == nullptr) return rc;
  return colred_finish(out1 ? 2 : 1, grid, a.D, a.dw, out1, nullptr, stream);
}

// Sets the error text "<fn>: <what>"; returns set_error's status.
static int fail(const char* fn, const char* what) {
  char msg[128];
  snprintf(msg, sizeof(msg), "%s: %s", fn, what);
  return set_error(msg);
}

// The checks of ivb_norm_fwd_fp8 and, with train, of ivb_norm_fwd_fp8_train (which also needs y, rstd and the
// LayerNorm mean); fn names the entry point in messages.
static int check_norm_fwd_fp8(const char* fn, bool train, const NormFwd& a) {
  if (a.M <= 0) return fail(fn, "empty tensor");
  if (a.D <= 0 || a.D > IVB_NORM_FP8_MAX_D || (a.D & 7))
    return fail(fn, "D must be a multiple of 8 in [8, IVB_NORM_FP8_MAX_D]");
  if ((a.ldx & 7) || a.ldx < a.D) return fail(fn, "ldx must be a multiple of 8 elements and >= D");
  if ((a.ldq & 15) || a.ldq < a.D) return fail(fn, "ldo must be a multiple of 16 elements and >= D");
  if (train && ((a.ldy & 7) || a.ldy < a.D)) return fail(fn, "ldy must be a multiple of 8 elements and >= D");
  if (a.x == nullptr || a.w == nullptr || a.q == nullptr || a.q_scale_inv == nullptr ||
      (train && (a.y == nullptr || a.rstd == nullptr || (a.ln && a.mean == nullptr))))
    return fail(fn, train ? "x, weight, out, row_scale_inv, y, rstd or (LayerNorm) mean is null"
                          : "x, weight, out or row_scale_inv is null");
  if (misaligned(16, a.x, a.w, a.b, a.q, a.y))
    return fail(fn, train ? "x, weight, bias, out and y must be 16-byte aligned"
                          : "x, weight, bias and out must be 16-byte aligned");
  if (misaligned(4, a.q_scale_inv, a.mean, a.rstd))
    return fail(fn, train ? "row_scale_inv, mean and rstd must be 4-byte aligned" : "row_scale_inv must be 4-byte aligned");
  return 0;
}

float* scalar_slots(long n, const char* who) {
  if (colred_check(1, n, 1, who)) return nullptr;
  static float* base[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  const bool tracked = dev >= 0 && dev < 64;
  if (tracked && base[dev] != nullptr) return base[dev];
  void* p = nullptr;
  const cudaError_t e = cudaGetSymbolAddress(&p, g_colred);
  if (e != cudaSuccess) {
    set_error_cuda(who, e);
    return nullptr;
  }
  if (tracked) base[dev] = static_cast<float*>(p);
  return static_cast<float*>(p);
}

int scalar_finish(int n, float* dst, cudaStream_t stream) {
  return colred_finish(1, n, 1, dst, nullptr, nullptr, stream);
}

float* colred_cols(long n, int D, const char* who) {
  return scalar_slots(n * D, who);
}

int colred_cols_finish(int n, int D, float* dst, cudaStream_t stream) {
  return colred_finish(1, n, D, dst, nullptr, nullptr, stream);
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_norm_fwd(const void* x, int x_is_f32, long ldx, const void* weight,
                            const void* bias, float eps, int is_layernorm, int M, int D, void* y,
                            long ldy, float* mean, float* rstd, void* stream_) {
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (ldy & 7)) return set_error("ivb_norm_fwd: D/ld must be multiples of 8");
  if (misaligned(16, x, weight, bias, y)) return set_error("ivb_norm_fwd: x, weight, bias and y must be 16-byte aligned");
  return launch_norm_fwd<NORM_Y>({x, ldx, x_is_f32 != 0, weight, bias, eps, is_layernorm != 0, M, D, y, ldy, mean, rstd},
                                 reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int ivb_norm_fwd_fp8(const void* x, int x_is_f32, long ldx, const void* weight, const void* bias, float eps,
                                int is_layernorm, int M, int D, void* out, long ldo, float* row_scale_inv,
                                void* stream_) {
  const NormFwd a{x, ldx, x_is_f32 != 0, weight, bias, eps, is_layernorm != 0, M, D, nullptr, 0, nullptr, nullptr,
                  out, ldo, row_scale_inv};
  if (int rc = check_norm_fwd_fp8("ivb_norm_fwd_fp8", false, a)) return rc;
  return launch_norm_fwd<NORM_Q>(a, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int ivb_norm_fwd_fp8_train(const void* x, int x_is_f32, long ldx, const void* weight, const void* bias,
                                      float eps, int is_layernorm, int M, int D, void* out, long ldo,
                                      float* row_scale_inv, void* y, long ldy, float* mean, float* rstd,
                                      void* stream_) {
  const NormFwd a{x, ldx, x_is_f32 != 0, weight, bias, eps, is_layernorm != 0, M, D, y, ldy, mean, rstd,
                  out, ldo, row_scale_inv};
  if (int rc = check_norm_fwd_fp8("ivb_norm_fwd_fp8_train", true, a)) return rc;
  return launch_norm_fwd<NORM_QY>(a, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int ivb_norm_bwd(const void* dy, long lddy, const void* x, int x_is_f32, long ldx,
                            const void* weight, const float* mean, const float* rstd,
                            int is_layernorm, int M, int D, const float* dx_in, long lddx_in,
                            void* dx_out, int dx_out_is_f32, long lddx, float* dweight,
                            float* dbias, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (lddy & 7) || (lddx & 7) || (lddx_in & 7))
    return set_error("ivb_norm_bwd: D/ld must be multiples of 8");
  if (misaligned(16, dy, x, weight, dx_in, dx_out))
    return set_error("ivb_norm_bwd: dy, x, weight, dx_in and dx_out must be 16-byte aligned");
  if (is_layernorm && mean == nullptr) return set_error("ivb_norm_bwd: LayerNorm needs mean");
  return launch_norm_bwd({dy, lddy, false, x, ldx, x_is_f32 != 0, weight, nullptr, mean, rstd, is_layernorm != 0, M, D,
                          dx_in, lddx_in, dx_out, lddx, dx_out_is_f32 != 0, dweight, dbias},
                         stream);
}

extern "C" int ivb_layerscale_bwd(const float* dx, long lddx, const void* y, long ldy,
                                  const void* gamma, int M, int D, void* dy, long lddy,
                                  float* dgamma, float* dcolsum, const float* rowscale,
                                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (lddx & 7) || (ldy & 7) || (lddy & 7)) return set_error("ivb_layerscale_bwd: D/ld must be multiples of 8");
  if (misaligned(16, dx, y, gamma, dy))
    return set_error("ivb_layerscale_bwd: dx, y, gamma and dy must be 16-byte aligned");
  const int nstrips = (D + 255) / 256;
  const int rbs = (M + 63) / 64;
  const __nv_bfloat16* yy = reinterpret_cast<const __nv_bfloat16*>(y);
  const __nv_bfloat16* gg = reinterpret_cast<const __nv_bfloat16*>(gamma);
  __nv_bfloat16* dyo = reinterpret_cast<__nv_bfloat16*>(dy);
  if (colred_check(2, rbs, D, "ivb_layerscale_bwd: gradient scratch too small")) return 1;
  if (int rc = launch("layerscale_bwd_kernel", y != nullptr ? layerscale_bwd_kernel<true> : layerscale_bwd_kernel<false>,
                      nstrips * rbs, 256, 0, stream, ALLOW_PDL, dx, lddx, yy, ldy, gg, M, D, dyo, lddy, dgamma, dcolsum,
                      nstrips, rowscale))
    return rc;
  return colred_finish(2, rbs, D, y != nullptr ? dgamma : nullptr, dcolsum, nullptr, stream);
}

extern "C" int ivb_colsum_bf16(const void* x, long ldx, int M, int N, float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((N & 7) || (ldx & 7)) return set_error("ivb_colsum_bf16: N/ld must be multiples of 8");
  if (misaligned(16, x)) return set_error("ivb_colsum_bf16: x must be 16-byte aligned");
  const int nstrips = (N + 255) / 256;
  const int rows_per_cta = 128;
  const int rbs = (M + rows_per_cta - 1) / rows_per_cta;
  if (colred_check(1, rbs, N, "ivb_colsum_bf16: gradient scratch too small")) return 1;
  if (int rc = launch("colsum_bf16_kernel", colsum_bf16_kernel, nstrips * rbs, 256, 0, stream, ALLOW_PDL,
                      reinterpret_cast<const __nv_bfloat16*>(x), ldx, M, N, out, nstrips, rows_per_cta))
    return rc;
  return colred_finish(1, rbs, N, out, nullptr, nullptr, stream);
}

// q-norm and k-norm of one block in a single launch: the two [M, D] column slices x and x + pair_off of a
// [M, ldx] bf16 buffer, weights w0 / w1, outputs at y and y + y_pair_off; rstd [M][2] (token-major).
extern "C" int ivb_rmsnorm_pair_fwd(const void* x, long ldx, long x_pair_off, const void* w0, const void* w1,
                                    float eps, int M, int D, void* y, long ldy, long y_pair_off, float* rstd,
                                    void* stream_) {
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (ldy & 7) || (x_pair_off & 7) || (y_pair_off & 7))
    return set_error("ivb_rmsnorm_pair_fwd: D/ld/offsets must be multiples of 8");
  if (D > 1536) return set_error("ivb_rmsnorm_pair_fwd: D > 1536 (use two ivb_norm_fwd calls)");
  if (misaligned(16, x, w0, w1, y)) return set_error("ivb_rmsnorm_pair_fwd: x, w0, w1 and y must be 16-byte aligned");
  NormFwd a{x, ldx, false, w0, nullptr, eps, false, M, D, y, ldy, nullptr, rstd};
  a.w1 = w1;
  a.x_pair_off = x_pair_off;
  a.y_pair_off = y_pair_off;
  return launch_norm_fwd<NORM_Y, true>(a, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int ivb_rmsnorm_pair_bwd(const void* dy, long lddy, long dy_pair_off, const void* x, long ldx,
                                    long x_pair_off, const void* w0, const void* w1, const float* rstd, int M,
                                    int D, void* dx_out, long lddx, long dx_pair_off, float* dweight0,
                                    float* dweight1, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (lddy & 7) || (lddx & 7) || (x_pair_off & 7) || (dy_pair_off & 7) || (dx_pair_off & 7))
    return set_error("ivb_rmsnorm_pair_bwd: D/ld/offsets must be multiples of 8");
  if (D > 1536) return set_error("ivb_rmsnorm_pair_bwd: D > 1536 (use two ivb_norm_bwd calls)");
  if ((dweight0 == nullptr) != (dweight1 == nullptr)) return set_error("ivb_rmsnorm_pair_bwd: give both weight gradients or none");
  if (misaligned(16, dy, x, w0, w1, dx_out))
    return set_error("ivb_rmsnorm_pair_bwd: dy, x, w0, w1 and dx_out must be 16-byte aligned");
  NormBwd a{dy, lddy, false, x, ldx, false, w0, nullptr, nullptr, rstd, false, M, D, nullptr, 0, dx_out, lddx, false,
            dweight0, nullptr};
  a.w1 = w1;
  a.dw1 = dweight1;
  a.x_pair_off = x_pair_off;
  a.dy_pair_off = dy_pair_off;
  a.dx_pair_off = dx_pair_off;
  return launch_norm_bwd<true>(a, stream);
}

// RMSNorm backward (fp32 stream) fused with the LayerScale backward of the branch that produced the stream
// (see rms_bwd_tma_kernel).  dx_out fp32 [M, D] = rmsnorm_bwd(dy, x, w, rstd) + dx_in;
// dyb bf16 = rowscale * gamma * dx_out; dgamma += colsum(rowscale * dx_out * ybr); dcolsum += gamma * colsum(rowscale * dx_out).
extern "C" int ivb_rmsnorm_bwd_layerscale(const void* dy, long lddy, const float* x, long ldx, const void* weight,
                                          const float* rstd, int M, int D, const float* dx_in, long lddx_in,
                                          float* dx_out, long lddx, float* dweight, const void* ybr, long ldyb,
                                          const void* gamma, const float* rowscale, void* dyb, long lddyb,
                                          float* dgamma, float* dcolsum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 3) || (lddy & 7) || (lddx & 3) || (ldyb & 7) || (lddyb & 7) || (lddx_in & 3))
    return set_error("ivb_rmsnorm_bwd_layerscale: D multiple of 8, pitches multiples of 16 bytes");
  if (ybr == nullptr || gamma == nullptr || dyb == nullptr) return set_error("ivb_rmsnorm_bwd_layerscale: ybr, gamma, dyb are required");
  if (misaligned(16, dy, x, dx_in, dx_out, ybr, dyb) || misaligned(8, weight, gamma))
    return set_error("ivb_rmsnorm_bwd_layerscale: dy, x, dx_in, dx_out, ybr and dyb must be 16-byte aligned, weight and "
                     "gamma 8-byte aligned");
  if (rms_bwd_tma_smem(D, dx_in != nullptr) > 226 * 1024)
    return set_error("ivb_rmsnorm_bwd_layerscale: D too large for the shared-memory row ring (use the separate kernels)");
  return launch_rms_bwd_tma(dy, lddy, x, ldx, weight, rstd, M, D, dx_in, lddx_in, dx_out, lddx, dweight, ybr, ldyb, gamma,
                            rowscale, dyb, lddyb, dgamma, dcolsum, stream);
}

extern "C" int ivb_ln_l2_fwd(const void* z, long ldz, const void* weight, const void* bias, float eps,
                             int M, int C, void* out, long ldo, float* stats, const void* target,
                             int target_is_f32, long ldt, float* loss_sum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (ldz & 7) || (ldo & 7) || (ldt & 7)) return set_error("ivb_ln_l2_fwd: C/ld must be multiples of 8");
  if (misaligned(16, z, weight, bias, out, target))
    return set_error("ivb_ln_l2_fwd: z, weight, bias, out and target must be 16-byte aligned");
  const int blocks = persistent_grid(M, 8, 8);
  float* loss = target != nullptr ? loss_sum : nullptr;
  if (loss != nullptr && colred_check(1, blocks, 1, "ivb_ln_l2_fwd: loss scratch too small")) return 1;
  auto zz = reinterpret_cast<const __nv_bfloat16*>(z);
  auto ww = reinterpret_cast<const __nv_bfloat16*>(weight);
  auto bb = reinterpret_cast<const __nv_bfloat16*>(bias);
  auto oo = reinterpret_cast<__nv_bfloat16*>(out);
  if (int rc = launch("ln_l2_fwd_kernel", target_is_f32 ? ln_l2_fwd_kernel<true> : ln_l2_fwd_kernel<false>, blocks,
                      256, 0, stream, NO_PDL, zz, ldz, ww, bb, eps, M, C, oo, ldo, stats, target, ldt, loss != nullptr))
    return rc;
  return colred_finish(1, blocks, 1, loss, nullptr, nullptr, stream);
}

extern "C" int ivb_ln_l2_bwd(const void* z, long ldz, const void* weight, const void* bias,
                             const float* stats, int M, int C, const void* dout, int dout_is_f32,
                             long lddo, float gscale_host, const float* gscale_dev, void* dz, long lddz,
                             float* dweight, float* dbias, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (ldz & 7) || (lddz & 7) || (lddo & 7)) return set_error("ivb_ln_l2_bwd: C/ld must be multiples of 8");
  if (misaligned(16, z, weight, bias, dout, dz))
    return set_error("ivb_ln_l2_bwd: z, weight, bias, dout and dz must be 16-byte aligned");
  NormBwd a{dout, lddo, dout_is_f32 != 0, z, ldz, false, weight, bias, stats, nullptr, true, M, C, nullptr, 0, dz, lddz,
            false, dweight, dbias};
  a.l2 = true;
  a.gs = gscale_host;
  a.gs_dev = gscale_dev;
  return launch_norm_bwd(a, stream);
}
