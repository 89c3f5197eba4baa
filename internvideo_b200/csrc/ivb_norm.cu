// ivb_norm.cu — HBM-bound row/column reduction kernels of the ViT block:
//   RMSNorm / LayerNorm forward + backward   (internvideo2_pretrain.py:117-128; FA2 DropoutAddRMSNorm
//                                             :467 incl. the q/k-norm over the full C :198-206;
//                                             nn.LayerNorm of the pooling block / decoders :525,:532)
//   LayerScale backward                      (internvideo2_pretrain.py:131-146)
//   bias-gradient column sums
// One warp per row, 16-byte vector loads, warp-shuffle reductions; parameter gradients are
// accumulated per warp in shared memory, stored as one partial per column per CTA and summed in a fixed
// order by colred_finish (ivb_colred.cuh).
#include <stdlib.h>

#include "ivb_colred.cuh"
#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

template <bool F32>
__device__ __forceinline__ void load8(const void* base, long elem_off, float v[8]) {
  if (F32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem_off);
    float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(base) + elem_off);
    float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
    v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y; v[4] = f2.x; v[5] = f2.y; v[6] = f3.x; v[7] = f3.y;
  }
}
__device__ __forceinline__ void unpack8(const uint4& u, float v[8]) {
  float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
  v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y; v[4] = f2.x; v[5] = f2.y; v[6] = f3.x; v[7] = f3.y;
}
template <bool F32>
__device__ __forceinline__ void store8(void* base, long elem_off, const float v[8]) {
  if (F32) {
    float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem_off);
    p[0] = make_float4(v[0], v[1], v[2], v[3]);
    p[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint4 u;
    u.x = pack_bf16(v[0], v[1]); u.y = pack_bf16(v[2], v[3]);
    u.z = pack_bf16(v[4], v[5]); u.w = pack_bf16(v[6], v[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(base) + elem_off) = u;
  }
}

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

// ------------------------------------------------------------------ backward
// dynamic smem: float acc[(LN ? 2 : 1)][warps][D]
template <bool XF32, bool LN, bool DXF32>
__global__ void __launch_bounds__(256)
norm_bwd_kernel(const __nv_bfloat16* dy, long lddy, const void* __restrict__ x, long ldx,
                const __nv_bfloat16* __restrict__ w, const float* __restrict__ mean_in,
                const float* __restrict__ rstd_in, int M, int D, const float* __restrict__ dx_in,
                long lddx_in, void* dx_out, long lddx, float* __restrict__ dweight,
                float* __restrict__ dbias) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float acc_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  const int nch = D >> 3;
  const float invD = 1.0f / static_cast<float>(D);
  const bool want_dw = dweight != nullptr;
  float* accw = acc_smem + (long)warp * D;
  float* accb = acc_smem + (long)(warps_per_block + warp) * D;
  if (want_dw) {
    for (int i = lane; i < D; i += 32) {
      accw[i] = 0.f;
      if (LN) accb[i] = 0.f;
    }
  }
  __syncwarp();
  for (long row = (long)blockIdx.x * warps_per_block + warp; row < M;
       row += (long)gridDim.x * warps_per_block) {
    const long xo = row * ldx;
    const long go = row * lddy;
    const float rstd = rstd_in[row];
    const float mean = LN ? mean_in[row] : 0.f;
    float s1 = 0.f, s2 = 0.f;  // sum g, sum g*xhat
    for (int c = lane; c < nch; c += 32) {
      float v[8], g[8], wv[8];
      load8<XF32>(x, xo + c * 8, v);
      load8<false>(dy, go + c * 8, g);
      load8<false>(w, c * 8, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float gj = g[j] * wv[j];
        const float xh = (v[j] - mean) * rstd;
        s1 += gj;
        s2 += gj * xh;
      }
    }
    s1 = LN ? warp_sum(s1) * invD : 0.f;
    s2 = warp_sum(s2) * invD;
    for (int c = lane; c < nch; c += 32) {
      float v[8], g[8], wv[8], o[8];
      load8<XF32>(x, xo + c * 8, v);
      load8<false>(dy, go + c * 8, g);
      load8<false>(w, c * 8, wv);
      float xh[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xh[j] = (v[j] - mean) * rstd;
        o[j] = rstd * (g[j] * wv[j] - s1 - xh[j] * s2);
      }
      if (dx_in != nullptr) {
        float r[8];
        load8<true>(dx_in, row * lddx_in + c * 8, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r[j];
      }
      store8<DXF32>(dx_out, row * lddx + c * 8, o);
      if (want_dw) {
        float4* aw = reinterpret_cast<float4*>(accw + c * 8);
        float4 a0 = aw[0], a1 = aw[1];
        a0.x += g[0] * xh[0]; a0.y += g[1] * xh[1]; a0.z += g[2] * xh[2]; a0.w += g[3] * xh[3];
        a1.x += g[4] * xh[4]; a1.y += g[5] * xh[5]; a1.z += g[6] * xh[6]; a1.w += g[7] * xh[7];
        aw[0] = a0; aw[1] = a1;
        if (LN) {
          float4* ab = reinterpret_cast<float4*>(accb + c * 8);
          float4 b0 = ab[0], b1 = ab[1];
          b0.x += g[0]; b0.y += g[1]; b0.z += g[2]; b0.w += g[3];
          b1.x += g[4]; b1.y += g[5]; b1.z += g[6]; b1.w += g[7];
          ab[0] = b0; ab[1] = b1;
        }
      }
    }
  }
  if (want_dw) {
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      float sw = 0.f, sb = 0.f;
      for (int k = 0; k < warps_per_block; ++k) {
        sw += acc_smem[(long)k * D + i];
        if (LN) sb += acc_smem[(long)(warps_per_block + k) * D + i];
      }
      colred_put(0, gridDim.x, blockIdx.x, D, i, sw);
      if (LN && dbias != nullptr) colred_put(1, gridDim.x, blockIdx.x, D, i, sb);
    }
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


// ------------------------------------------------------------------ register-resident RMSNorm (D <= 256*NCH)
// The generic kernels above stream every row twice (statistics pass + output pass, second pass from L1/L2).
// For the block norms (D = 384..1536) the row fits in registers: one HBM read per operand, period.
// PAIR: the q-norm and the k-norm of a block in ONE launch (internvideo2_pretrain.py:198-206).  Virtual row r covers
// token r>>1, part r&1; part p reads/writes at column offset p*pair_off of its token's row and uses weight w / w1.
// rstd_out is indexed by the virtual row ([M][2]).  (Two 37 MB launches were each ~3x off the HBM time.)
template <bool XF32, int NCH, bool PAIR>
__global__ void __launch_bounds__(256)
rms_fwd_reg_kernel(const void* __restrict__ x, long ldx, const __nv_bfloat16* __restrict__ w, float eps,
                   int M, int D, __nv_bfloat16* __restrict__ y, long ldy, float* __restrict__ rstd_out,
                   const __nv_bfloat16* __restrict__ w1, long x_pair_off, long y_pair_off) {
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
    const long yo = tok * ldy + part * y_pair_off;
    const __nv_bfloat16* wp = (PAIR && part) ? w1 : w;
    float v[NCH][8];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        load8<XF32>(x, xo + c * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += v[i][j] * v[i][j];
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) * invD + eps);
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float wv[8], o[8];
        load8<false>(wp, c * 8, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = v[i][j] * rstd * wv[j];
        store8<false>(y, yo + c * 8, o);
      }
    }
    if (lane == 0 && rstd_out) rstd_out[row] = rstd;
  }
}

// dynamic smem: float acc[warps][D] (only when dweight != nullptr)
// Registers: the normalised row in fp32 (8*NCH) + dy as the raw packed bf16 it was loaded as (4*NCH);
// keeping dy*w in fp32 as well pushed the kernel to 150 registers / 1 CTA per SM and made it 2x slower.
template <bool XF32, bool DXF32, int NCH, bool PAIR>
__global__ void __launch_bounds__(256, 2)
rms_bwd_reg_kernel(const __nv_bfloat16* dy, long lddy, const void* __restrict__ x, long ldx,
                   const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd_in, int M, int D,
                   const float* __restrict__ dx_in, long lddx_in, void* dx_out, long lddx,
                   float* __restrict__ dweight, const __nv_bfloat16* __restrict__ w1,
                   float* __restrict__ dweight1, long x_pair_off, long dy_pair_off, long dx_pair_off) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float acc_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int nch = D >> 3;
  const float invD = 1.0f / static_cast<float>(D);
  const bool want_dw = dweight != nullptr;
  float* accw = acc_smem + (long)warp * D;
  if (want_dw) for (int i = lane; i < D; i += 32) accw[i] = 0.f;
  __syncwarp();
  // PAIR: the virtual-row stride gridDim.x * wpb is even (wpb = 8), so a warp only ever sees ONE part
  // (row parity == warp parity): its accumulator belongs to that part's weight gradient.
  for (long row = (long)blockIdx.x * wpb + warp; row < M; row += (long)gridDim.x * wpb) {
    const long tok = PAIR ? (row >> 1) : row;
    const int part = PAIR ? static_cast<int>(row & 1) : 0;
    const long xo = tok * ldx + part * x_pair_off;
    const long go = tok * lddy + part * dy_pair_off;
    const long oo = tok * lddx + part * dx_pair_off;
    const __nv_bfloat16* wp = (PAIR && part) ? w1 : w;
    const float rstd = rstd_in[row];
    float xh[NCH][8];
    uint4 gq[NCH];
    float s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        load8<XF32>(x, xo + c * 8, xh[i]);
        gq[i] = *reinterpret_cast<const uint4*>(dy + go + c * 8);
      }
    }
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float wv[8], g[8];
        load8<false>(wp, c * 8, wv);
        unpack8(gq[i], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] *= rstd;
          s2 += g[j] * wv[j] * xh[i][j];
        }
      }
    }
    s2 = warp_sum(s2) * invD;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float wv[8], g[8], o[8];
        load8<false>(wp, c * 8, wv);
        unpack8(gq[i], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] * wv[j] - xh[i][j] * s2);
        if (dx_in != nullptr) {
          float r[8];
          load8<true>(dx_in, row * lddx_in + c * 8, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        store8<DXF32>(dx_out, oo + c * 8, o);
        if (want_dw) {
          float4* aw = reinterpret_cast<float4*>(accw + c * 8);
          float4 a0 = aw[0], a1 = aw[1];
          a0.x += g[0] * xh[i][0]; a0.y += g[1] * xh[i][1]; a0.z += g[2] * xh[i][2]; a0.w += g[3] * xh[i][3];
          a1.x += g[4] * xh[i][4]; a1.y += g[5] * xh[i][5]; a1.z += g[6] * xh[i][6]; a1.w += g[7] * xh[i][7];
          aw[0] = a0; aw[1] = a1;
        }
      }
    }
  }
  if (want_dw) {
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      if (PAIR) {
        float s0 = 0.f, s1 = 0.f;
        for (int k = 0; k < wpb; k += 2) { s0 += acc_smem[(long)k * D + i]; s1 += acc_smem[(long)(k + 1) * D + i]; }
        colred_put(0, gridDim.x, blockIdx.x, D, i, s0);
        colred_put(1, gridDim.x, blockIdx.x, D, i, s1);
      } else {
        float sw = 0.f;
        for (int k = 0; k < wpb; ++k) sw += acc_smem[(long)k * D + i];
        colred_put(0, gridDim.x, blockIdx.x, D, i, sw);
      }
    }
  }
}

// ------------------------------------------------------------------ bulk-copy (TMA) row pipeline
// Every warp owns a ring of NBUF row slots in shared memory that lane 0 keeps full with cp.async.bulk (1-D bulk copies
// completing on per-slot mbarriers); the arithmetic reads the row from shared memory (conflict-free 16-byte lanes), so
// four input rows per token cost no registers.  It is used where it removes a whole kernel: the backward fused with the
// LayerScale backward.

// RMSNorm backward on the fp32 stream, optionally FUSED with the LayerScale backward that follows it in the block
// (Block.backward: dx = rmsnorm_bwd(dy, x) + dx_in is the gradient of the residual stream, which the preceding branch's
// LayerScale consumes at once: dyb = rs * gamma * dx, dgamma += sum rs*dx*ybr, dcolsum += gamma * sum rs*dx):
//   inputs per row: dy bf16 [D], x fp32 [D], dx_in fp32 [D] (optional), ybr bf16 [D] (LS only)
//   outputs: dx fp32 [D]; LS: dyb bf16 [D]
// The separate layerscale_bwd kernel re-read dx (4 D bytes/row) and ran at 0.62 of the HBM rate; fused, the
// gradient of the stream never makes that extra round trip.  smem: [warp][NBUF][slot] + [warp][nacc][D] fp32.
template <int NBUF, bool LS>
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
  constexpr int NW = 4;
  extern __shared__ __align__(128) uint8_t rt_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool has_in = dx_in != nullptr;
  const uint32_t by_dy = static_cast<uint32_t>(D) * 2u, by_x = static_cast<uint32_t>(D) * 4u;
  const uint32_t slot = by_x + by_dy + (has_in ? by_x : 0u) + (LS ? by_dy : 0u);      // bytes per buffered row
  uint8_t* base = rt_smem + static_cast<long>(warp) * NBUF * slot;
  constexpr int NACC = LS ? 3 : 1;
  float* acc = reinterpret_cast<float*>(rt_smem + static_cast<long>(NW) * NBUF * slot) + static_cast<long>(warp) * NACC * D;
  uint64_t* bars = reinterpret_cast<uint64_t*>(rt_smem + static_cast<long>(NW) * NBUF * slot +
                                               static_cast<long>(NW) * NACC * D * 4) + warp * NBUF;
  const long W = static_cast<long>(gridDim.x) * NW;
  const long gw = static_cast<long>(blockIdx.x) * NW + warp;
  auto fill = [&](int b, long row) {
    uint8_t* s0 = base + static_cast<long>(b) * slot;
    mbar_expect_tx(&bars[b], slot);
    bulk_load_1d(s0, x + row * ldx, by_x, &bars[b]);
    bulk_load_1d(s0 + by_x, dy + row * lddy, by_dy, &bars[b]);
    uint32_t off = by_x + by_dy;
    if (has_in) { bulk_load_1d(s0 + off, dx_in + row * lddx_in, by_x, &bars[b]); off += by_x; }
    if (LS) bulk_load_1d(s0 + off, ybr + row * ldyb, by_dy, &bars[b]);
  };
  for (int i = lane; i < NACC * D; i += 32) acc[i] = 0.f;
  if (lane == 0) {
#pragma unroll
    for (int b = 0; b < NBUF; ++b) mbar_init(&bars[b], 1);
    fence_mbar_init();
#pragma unroll
    for (int b = 0; b < NBUF; ++b) {
      const long row = gw + b * W;
      if (row < M) fill(b, row);
    }
  }
  __syncwarp();
  const int nq = D >> 2;
  const float invD = 1.0f / static_cast<float>(D);
  long it = 0;
  for (long row = gw; row < M; row += W, ++it) {
    const int b = static_cast<int>(it % NBUF);
    mbar_wait(&bars[b], static_cast<uint32_t>((it / NBUF) & 1));
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
    const float rsc = (LS && rowscale) ? rowscale[row] : 1.f;
    float* dxr = dx_out + row * lddx;
    for (int g = lane; g < nq; g += 32) {
      const float4 a = xs[g];
      const uint2 gq = gs[g], wq = *reinterpret_cast<const uint2*>(w + g * 4);
      const float2 g0 = unpack_bf16(gq.x), g1 = unpack_bf16(gq.y), w0 = unpack_bf16(wq.x), w1 = unpack_bf16(wq.y);
      const float xh0 = a.x * rstd, xh1 = a.y * rstd, xh2 = a.z * rstd, xh3 = a.w * rstd;
      float4 o;
      o.x = rstd * (g0.x * w0.x - xh0 * s2); o.y = rstd * (g0.y * w0.y - xh1 * s2);
      o.z = rstd * (g1.x * w1.x - xh2 * s2); o.w = rstd * (g1.y * w1.y - xh3 * s2);
      if (has_in) { const float4 r = rs_in[g]; o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w; }
      *reinterpret_cast<float4*>(dxr + g * 4) = o;
      float4* aw = reinterpret_cast<float4*>(acc + g * 4);
      float4 a0 = *aw;
      a0.x += g0.x * xh0; a0.y += g0.y * xh1; a0.z += g1.x * xh2; a0.w += g1.y * xh3;
      *aw = a0;
      if (LS) {
        const uint2 yq = ys[g], gmq = *reinterpret_cast<const uint2*>(gamma + g * 4);
        const float2 y0 = unpack_bf16(yq.x), y1 = unpack_bf16(yq.y), m0 = unpack_bf16(gmq.x), m1 = unpack_bf16(gmq.y);
        const float d0 = o.x * rsc, d1 = o.y * rsc, d2 = o.z * rsc, d3 = o.w * rsc;
        uint2 ob;
        ob.x = pack_bf16(d0 * m0.x, d1 * m0.y); ob.y = pack_bf16(d2 * m1.x, d3 * m1.y);
        *reinterpret_cast<uint2*>(dyb + row * lddyb + g * 4) = ob;
        float4* ag = reinterpret_cast<float4*>(acc + D + g * 4);
        float4* as = reinterpret_cast<float4*>(acc + 2 * D + g * 4);
        float4 ga = *ag, sa = *as;
        ga.x += d0 * y0.x; ga.y += d1 * y0.y; ga.z += d2 * y1.x; ga.w += d3 * y1.y;
        sa.x += d0; sa.y += d1; sa.z += d2; sa.w += d3;
        *ag = ga; *as = sa;
      }
    }
    __syncwarp();
    const long nxt = row + static_cast<long>(NBUF) * W;
    if (lane == 0 && nxt < M) fill(b, nxt);
  }
  __syncthreads();
  const float* accs = reinterpret_cast<const float*>(rt_smem + static_cast<long>(NW) * NBUF * slot);
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float sw = 0.f, sg = 0.f, sc = 0.f;
#pragma unroll
    for (int k = 0; k < NW; ++k) {
      sw += accs[(static_cast<long>(k) * NACC) * D + i];
      if (LS) { sg += accs[(static_cast<long>(k) * NACC + 1) * D + i]; sc += accs[(static_cast<long>(k) * NACC + 2) * D + i]; }
    }
    if (dweight) colred_put(0, gridDim.x, blockIdx.x, D, i, sw);
    if (LS) {
      if (dgamma) colred_put(1, gridDim.x, blockIdx.x, D, i, sg);
      if (dcolsum) colred_put(2, gridDim.x, blockIdx.x, D, i, sc * __bfloat162float(gamma[i]));
    }
  }
}

template <bool LS>
static int launch_rms_bwd_tma(const void* dy, long lddy, const void* x, long ldx, const void* w, const float* rstd, int M,
                              int D, const float* dx_in, long lddx_in, void* dx_out, long lddx, float* dweight,
                              const void* ybr, long ldyb, const void* gamma, const float* rowscale, void* dyb, long lddyb,
                              float* dgamma, float* dcolsum, cudaStream_t stream) {
  constexpr int NBUF = LS ? 2 : 3, NW = 4;     // 8-12 rows in flight per SM
  const size_t slot = static_cast<size_t>(D) * (4 + 2 + (dx_in ? 4 : 0) + (LS ? 2 : 0));
  const size_t smem = NW * NBUF * slot + static_cast<size_t>(NW) * (LS ? 3 : 1) * D * 4 + NW * NBUF * 8;
  auto kern = rms_bwd_tma_kernel<NBUF, LS>;
  static bool set[64] = {};
  int dev = 0; cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(rms_bwd_tma)", e);
    set[dev] = true;
  }
  if (smem > 226 * 1024) return set_error("rms_bwd_tma: row too long for the shared-memory ring");
  int grid = num_sms();
  const int need = (M + NW - 1) / NW;
  if (grid > need) grid = need;
  if (colred_check(3, grid, D, "rms_bwd_tma: gradient scratch too small")) return 1;
  launch_pdl(kern, dim3(grid), dim3(NW * 32), smem, stream, reinterpret_cast<const __nv_bfloat16*>(dy), lddy, reinterpret_cast<const float*>(x), ldx,
                                        reinterpret_cast<const __nv_bfloat16*>(w), rstd, M, D, dx_in, lddx_in,
                                        reinterpret_cast<float*>(dx_out), lddx, dweight,
                                        reinterpret_cast<const __nv_bfloat16*>(ybr), ldyb,
                                        reinterpret_cast<const __nv_bfloat16*>(gamma), rowscale,
                                        reinterpret_cast<__nv_bfloat16*>(dyb), lddyb, dgamma, dcolsum);
  count_launch();
  if (int rc = check_launch("rms_bwd_tma_kernel")) return rc;
  return colred_finish(3, grid, D, dweight, LS ? dgamma : nullptr, LS ? dcolsum : nullptr, stream);
}

template <bool XF32, int NCH, bool PAIR = false>
static int launch_rms_fwd_reg(const void* x, long ldx, const void* w, float eps, int M, int D, void* y, long ldy,
                              float* rstd, cudaStream_t stream, const void* w1 = nullptr, long x_pair_off = 0,
                              long y_pair_off = 0) {
  const int wpb = 8;
  const long rows = PAIR ? 2L * M : M;
  long blocks = (rows + wpb - 1) / wpb;
  const long cap = (long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  launch_pdl(rms_fwd_reg_kernel<XF32, NCH, PAIR>, dim3((int)blocks), dim3(256), 0, stream, 
      x, ldx, reinterpret_cast<const __nv_bfloat16*>(w), eps, (int)rows, D, reinterpret_cast<__nv_bfloat16*>(y), ldy, rstd,
      reinterpret_cast<const __nv_bfloat16*>(w1), x_pair_off, y_pair_off);
  count_launch();
  return check_launch("rms_fwd_reg_kernel");
}

template <bool XF32, bool DXF32, int NCH, bool PAIR = false>
static int launch_rms_bwd_reg(const void* dy, long lddy, const void* x, long ldx, const void* w, const float* rstd,
                              int M, int D, const float* dx_in, long lddx_in, void* dx_out, long lddx,
                              float* dweight, cudaStream_t stream, const void* w1 = nullptr, float* dweight1 = nullptr,
                              long x_pair_off = 0, long dy_pair_off = 0, long dx_pair_off = 0) {
  auto kern = rms_bwd_reg_kernel<XF32, DXF32, NCH, PAIR>;
  const int wpb = 8;
  const size_t smem = dweight ? (size_t)wpb * D * sizeof(float) : 0;
  if (smem > 48 * 1024) {
    static bool set[64] = {};
    if (first_use_on_device(set)) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
      if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(rms_bwd_reg)", e);
    }
  }
  const long rows = PAIR ? 2L * M : M;
  long blocks = (rows + wpb * 2 - 1) / (wpb * 2);
  const long cap = (long)num_sms() * 2;   // 2 CTAs/SM resident (<=128 registers): one persistent wave
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (colred_check(2, blocks, D, "rms_bwd_reg: gradient scratch too small")) return 1;
  launch_pdl(kern, dim3((int)blocks), dim3(wpb * 32), smem, stream, reinterpret_cast<const __nv_bfloat16*>(dy), lddy, x, ldx,
                                                reinterpret_cast<const __nv_bfloat16*>(w), rstd, (int)rows, D, dx_in,
                                                lddx_in, dx_out, lddx, dweight,
                                                reinterpret_cast<const __nv_bfloat16*>(w1), dweight1, x_pair_off,
                                                dy_pair_off, dx_pair_off);
  count_launch();
  if (int rc = check_launch("rms_bwd_reg_kernel")) return rc;
  if (dweight == nullptr) return 0;
  return colred_finish(PAIR ? 2 : 1, (int)blocks, D, dweight, PAIR ? dweight1 : nullptr, nullptr, stream);
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_norm_fwd(const void* x, int x_is_f32, long ldx, const void* weight,
                            const void* bias, float eps, int is_layernorm, int M, int D, void* y,
                            long ldy, float* mean, float* rstd, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (ldy & 7)) return set_error("ivb_norm_fwd: D/ld must be multiples of 8");
  if (!is_layernorm && D <= 1536) {   // register-resident RMSNorm: the row is read from HBM exactly once
    const int nchunks = (D + 255) / 256;
#define IVB_RF(XF)                                                                                   \
    do {                                                                                             \
      if (nchunks <= 2) return launch_rms_fwd_reg<XF, 2>(x, ldx, weight, eps, M, D, y, ldy, rstd, stream); \
      if (nchunks <= 4) return launch_rms_fwd_reg<XF, 4>(x, ldx, weight, eps, M, D, y, ldy, rstd, stream); \
      return launch_rms_fwd_reg<XF, 6>(x, ldx, weight, eps, M, D, y, ldy, rstd, stream);             \
    } while (0)
    if (x_is_f32) IVB_RF(true); else IVB_RF(false);
#undef IVB_RF
  }
  const int wpb = 8;
  long blocks = (M + wpb - 1) / wpb;
  const long cap = (long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(weight);
  const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(bias);
  __nv_bfloat16* yo = reinterpret_cast<__nv_bfloat16*>(y);
#define IVB_LAUNCH_NF(XF, LNN) \
  launch_pdl(norm_fwd_kernel<XF, LNN>, dim3((int)blocks), dim3(256), 0, stream, x, ldx, w, b, eps, M, D, yo, ldy, mean, rstd)
  if (x_is_f32) { if (is_layernorm) IVB_LAUNCH_NF(true, true); else IVB_LAUNCH_NF(true, false); }
  else          { if (is_layernorm) IVB_LAUNCH_NF(false, true); else IVB_LAUNCH_NF(false, false); }
#undef IVB_LAUNCH_NF
  count_launch();
  return check_launch("norm_fwd_kernel");
}

template <bool XF32, bool LN, bool DXF32>
static int launch_norm_bwd(const void* dy, long lddy, const void* x, long ldx, const void* weight,
                           const float* mean, const float* rstd, int M, int D, const float* dx_in,
                           long lddx_in, void* dx_out, long lddx, float* dweight, float* dbias,
                           cudaStream_t stream) {
  auto kern = norm_bwd_kernel<XF32, LN, DXF32>;
  int wpb = 8;
  size_t smem = dweight ? (size_t)(LN ? 2 : 1) * wpb * D * sizeof(float) : 0;
  if (smem > 200 * 1024) { wpb = 4; smem /= 2; }
  if (smem > 200 * 1024) { wpb = 2; smem /= 2; }
  if (smem > 48 * 1024) {
    static size_t set_to = 0;
    if (smem > set_to) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
      if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(norm_bwd)", e);
      set_to = 220 * 1024;
    }
  }
  // >= 2 rows per warp so the smem flush amortises, but enough CTAs to keep ~32 warps/SM in flight:
  // this kernel is pure HBM streaming and latency-bound below that (measured 2.8x off the HBM time
  // with 1.4 CTAs/SM).
  long blocks = (M + wpb * 2 - 1) / (wpb * 2);
  const long cap = (long)num_sms() * (smem > 96 * 1024 ? 2 : 4);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (colred_check(2, blocks, D, "norm_bwd: gradient scratch too small")) return 1;
  launch_pdl(kern, dim3((int)blocks), dim3(wpb * 32), smem, stream, 
      reinterpret_cast<const __nv_bfloat16*>(dy), lddy, x, ldx,
      reinterpret_cast<const __nv_bfloat16*>(weight), mean, rstd, M, D, dx_in, lddx_in, dx_out,
      lddx, dweight, dbias);
  count_launch();
  if (int rc = check_launch("norm_bwd_kernel")) return rc;
  if (dweight == nullptr) return 0;
  return colred_finish(2, (int)blocks, D, dweight, LN ? dbias : nullptr, nullptr, stream);
}

extern "C" int ivb_norm_bwd(const void* dy, long lddy, const void* x, int x_is_f32, long ldx,
                            const void* weight, const float* mean, const float* rstd,
                            int is_layernorm, int M, int D, const float* dx_in, long lddx_in,
                            void* dx_out, int dx_out_is_f32, long lddx, float* dweight,
                            float* dbias, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (lddy & 7) || (lddx & 7))
    return set_error("ivb_norm_bwd: D/ld must be multiples of 8");
  if (is_layernorm && mean == nullptr) return set_error("ivb_norm_bwd: LayerNorm needs mean");
  if (!is_layernorm && D <= 1536) {
    const int nchunks = (D + 255) / 256;
#define IVB_RB(XF, DXF)                                                                                          \
    do {                                                                                                         \
      if (nchunks <= 2) return launch_rms_bwd_reg<XF, DXF, 2>(dy, lddy, x, ldx, weight, rstd, M, D, dx_in, lddx_in, dx_out, lddx, dweight, stream); \
      if (nchunks <= 4) return launch_rms_bwd_reg<XF, DXF, 4>(dy, lddy, x, ldx, weight, rstd, M, D, dx_in, lddx_in, dx_out, lddx, dweight, stream); \
      return launch_rms_bwd_reg<XF, DXF, 6>(dy, lddy, x, ldx, weight, rstd, M, D, dx_in, lddx_in, dx_out, lddx, dweight, stream);                   \
    } while (0)
    if (x_is_f32) { if (dx_out_is_f32) IVB_RB(true, true); else IVB_RB(true, false); }
    else          { if (dx_out_is_f32) IVB_RB(false, true); else IVB_RB(false, false); }
#undef IVB_RB
  }
#define IVB_NB(XF, LNN, DXF)                                                                     \
  return launch_norm_bwd<XF, LNN, DXF>(dy, lddy, x, ldx, weight, mean, rstd, M, D, dx_in, lddx_in, \
                                       dx_out, lddx, dweight, dbias, stream)
  if (x_is_f32) {
    if (is_layernorm) { if (dx_out_is_f32) IVB_NB(true, true, true); else IVB_NB(true, true, false); }
    else              { if (dx_out_is_f32) IVB_NB(true, false, true); else IVB_NB(true, false, false); }
  } else {
    if (is_layernorm) { if (dx_out_is_f32) IVB_NB(false, true, true); else IVB_NB(false, true, false); }
    else              { if (dx_out_is_f32) IVB_NB(false, false, true); else IVB_NB(false, false, false); }
  }
#undef IVB_NB
}

extern "C" int ivb_layerscale_bwd(const float* dx, long lddx, const void* y, long ldy,
                                  const void* gamma, int M, int D, void* dy, long lddy,
                                  float* dgamma, float* dcolsum, const float* rowscale,
                                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (lddx & 7) || (lddy & 7)) return set_error("ivb_layerscale_bwd: D/ld must be multiples of 8");
  const int nstrips = (D + 255) / 256;
  const int rbs = (M + 63) / 64;
  const __nv_bfloat16* yy = reinterpret_cast<const __nv_bfloat16*>(y);
  const __nv_bfloat16* gg = reinterpret_cast<const __nv_bfloat16*>(gamma);
  __nv_bfloat16* dyo = reinterpret_cast<__nv_bfloat16*>(dy);
  if (colred_check(2, rbs, D, "ivb_layerscale_bwd: gradient scratch too small")) return 1;
  if (y != nullptr)
    launch_pdl(layerscale_bwd_kernel<true>, dim3(nstrips * rbs), dim3(256), 0, stream, dx, lddx, yy, ldy, gg, M, D, dyo, lddy, dgamma, dcolsum, nstrips, rowscale);
  else
    launch_pdl(layerscale_bwd_kernel<false>, dim3(nstrips * rbs), dim3(256), 0, stream, dx, lddx, yy, ldy, gg, M, D, dyo, lddy, dgamma, dcolsum, nstrips, rowscale);
  count_launch();
  if (int rc = check_launch("layerscale_bwd_kernel")) return rc;
  return colred_finish(2, rbs, D, y != nullptr ? dgamma : nullptr, dcolsum, nullptr, stream);
}

extern "C" int ivb_colsum_bf16(const void* x, long ldx, int M, int N, float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((N & 7) || (ldx & 7)) return set_error("ivb_colsum_bf16: N/ld must be multiples of 8");
  const int nstrips = (N + 255) / 256;
  const int rows_per_cta = 128;
  const int rbs = (M + rows_per_cta - 1) / rows_per_cta;
  if (colred_check(1, rbs, N, "ivb_colsum_bf16: gradient scratch too small")) return 1;
  launch_pdl(colsum_bf16_kernel, dim3(nstrips * rbs), dim3(256), 0, stream, reinterpret_cast<const __nv_bfloat16*>(x),
                                                        ldx, M, N, out, nstrips, rows_per_cta);
  count_launch();
  if (int rc = check_launch("colsum_bf16_kernel")) return rc;
  return colred_finish(1, rbs, N, out, nullptr, nullptr, stream);
}

// q-norm and k-norm of one block in a single launch: the two [M, D] column slices x and x + pair_off of a
// [M, ldx] bf16 buffer, weights w0 / w1, outputs at y and y + y_pair_off; rstd [M][2] (token-major).
extern "C" int ivb_rmsnorm_pair_fwd(const void* x, long ldx, long x_pair_off, const void* w0, const void* w1,
                                    float eps, int M, int D, void* y, long ldy, long y_pair_off, float* rstd,
                                    void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((D & 7) || (ldx & 7) || (ldy & 7) || (x_pair_off & 7) || (y_pair_off & 7))
    return set_error("ivb_rmsnorm_pair_fwd: D/ld/offsets must be multiples of 8");
  if (D > 1536) return set_error("ivb_rmsnorm_pair_fwd: D > 1536 (use two ivb_norm_fwd calls)");
  const int nchunks = (D + 255) / 256;
  if (nchunks <= 2) return launch_rms_fwd_reg<false, 2, true>(x, ldx, w0, eps, M, D, y, ldy, rstd, stream, w1, x_pair_off, y_pair_off);
  if (nchunks <= 4) return launch_rms_fwd_reg<false, 4, true>(x, ldx, w0, eps, M, D, y, ldy, rstd, stream, w1, x_pair_off, y_pair_off);
  return launch_rms_fwd_reg<false, 6, true>(x, ldx, w0, eps, M, D, y, ldy, rstd, stream, w1, x_pair_off, y_pair_off);
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
  const int nchunks = (D + 255) / 256;
#define IVB_PB(N_) return launch_rms_bwd_reg<false, false, N_, true>(dy, lddy, x, ldx, w0, rstd, M, D, nullptr, 0, dx_out, lddx, \
                                                                      dweight0, stream, w1, dweight1, x_pair_off, dy_pair_off, dx_pair_off)
  if (nchunks <= 2) IVB_PB(2);
  if (nchunks <= 4) IVB_PB(4);
  IVB_PB(6);
#undef IVB_PB
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
  if (static_cast<size_t>(D) * (4 + 2 + (dx_in ? 4 : 0) + 2) * 8 + static_cast<size_t>(D) * 48 + 64 > 226 * 1024)
    return set_error("ivb_rmsnorm_bwd_layerscale: D too large for the shared-memory row ring (use the separate kernels)");
  return launch_rms_bwd_tma<true>(dy, lddy, x, ldx, weight, rstd, M, D, dx_in, lddx_in, dx_out, lddx, dweight, ybr, ldyb, gamma,
                                  rowscale, dyb, lddyb, dgamma, dcolsum, stream);
}
