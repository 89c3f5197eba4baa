// ivb_dpe.cu — the global extractor's position conv and key LayerNorm of InternVideo-MM (InternVideo1's multimodal
// model; the UniFormerV2-style extractor of clip_utils/utils/clip_vit_only_global.py:203-231): at one extractor tap,
//   patch row (t, h, w):  y = LN3(x + bias + sum_{dt,dh,dw in {-1,0,1}} wt[c, dt, dh, dw] x[t+dt, h+dh, w+dw])
//   cls row:              y = LN3(x)
// with zero padding at the edges of the T x H x W grid.  The reference computes the depthwise Conv3d `dpe` on a copy of
// the stream and feeds the sum only to `ln_3` (Extractor.forward :147), so the two fuse without writing the conv.
//
// One CTA walks the W rows of one (clip, frame, grid row) line, one thread per 8 channels, so the LayerNorm of a row is
// a CTA reduction over C.  The 3x3x3 stencil is split by its w tap: column w' of the nine (t+dt, h+dh) neighbour lines
// is read once and gives three partial sums P_dw, added to output rows w'+1, w' and w'-1.  Each input row is therefore
// read by the nine lines around it, once each (L2 serves the repeats), and each output row is complete one column after
// its own.  The weights are staged once per CTA in shared memory, transposed to [27][C] so a thread reads its 8
// channels of a tap as one 16-byte vector.  Every sum runs in fp32 in a fixed order (no atomics); the output is rounded
// to bf16 once.
#include <cstdio>

#include "ivb_internal.h"
#include "ivb_rows.cuh"

namespace ivb {

constexpr int DPE_MAX_C = 4096;
constexpr int DPE_TAPS = 27;
constexpr int DPE_SMEM_MAX = DPE_TAPS * DPE_MAX_C * 2;

// Sum of v over the CTA, the same bits in every thread: warp shuffles, then every thread adds the warp partials in
// warp order.  red: 32 floats of shared memory, free again when the call returns.
__device__ __forceinline__ float dpe_block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) s += red[i];
  __syncthreads();
  return s;
}

// LayerNorm of the row whose 8 channels c0 .. c0+7 this thread holds in v (two-pass variance), written as bf16.
__device__ __forceinline__ void dpe_ln_store(const float v[8], bool active, int C, int c0, const __nv_bfloat16* ln_w,
                                             const __nv_bfloat16* ln_b, float eps, __nv_bfloat16* y, long yoff,
                                             float* red) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += v[i];
  const float mean = dpe_block_sum(active ? s : 0.f, red) / static_cast<float>(C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) q = fmaf(v[i] - mean, v[i] - mean, q);
  const float var = dpe_block_sum(active ? q : 0.f, red) / static_cast<float>(C);
  if (!active) return;
  const float rstd = rsqrtf(var + eps);
  float g[8], b[8], o[8];
  load8<false>(ln_w, c0, g);
  load8<false>(ln_b, c0, b);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = fmaf((v[i] - mean) * rstd, g[i], b[i]);
  store8<false>(y, yoff + c0, o);
}

template <bool F32>
__global__ void __launch_bounds__(512) dpe_ln_fwd_kernel(const void* __restrict__ x, long ldx,
                                                         const __nv_bfloat16* __restrict__ conv_w,
                                                         const __nv_bfloat16* __restrict__ conv_b,
                                                         const __nv_bfloat16* __restrict__ ln_w,
                                                         const __nv_bfloat16* __restrict__ ln_b, float eps, int N,
                                                         int T, int H, int W, int C, __nv_bfloat16* __restrict__ y,
                                                         long ldy) {
  extern __shared__ __align__(16) __nv_bfloat16 wsm[];     // [27][C]: tap k = ((dt+1)*3 + dh+1)*3 + dw+1
  __shared__ float red[32];
  for (int i = threadIdx.x; i < DPE_TAPS * C; i += blockDim.x) {
    const int c = i / DPE_TAPS, k = i - c * DPE_TAPS;
    wsm[k * C + c] = conv_w[i];
  }
  __syncthreads();

  const int c0 = threadIdx.x * 8;
  const bool active = c0 < C;
  const int cc = active ? c0 : 0;           // idle threads read channel 0 and drop it
  float bias[8];
  load8<false>(conv_b, cc, bias);
  const long L = 1 + static_cast<long>(H) * W;
  const long items = static_cast<long>(N) * T * (H + 1);
  for (long it = blockIdx.x; it < items; it += gridDim.x) {
    const int h = static_cast<int>(it % (H + 1));
    const long nt = it / (H + 1);
    const int t = static_cast<int>(nt % T);
    const long frame = nt - t;              // (n*T + 0): the clip's first frame
    if (h == H) {                           // the frame's cls row: no conv
      float v[8];
      load8<F32>(x, nt * L * ldx + cc, v);
      dpe_ln_store(v, active, C, c0, ln_w, ln_b, eps, y, nt * L * ldy, red);
      continue;
    }
    float prev[8], cur[8], next[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) prev[i] = cur[i] = next[i] = 0.f;
    for (int w = 0; w < W; ++w) {
      float p[3][8];
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) p[j][i] = 0.f;
#pragma unroll
      for (int dt = -1; dt <= 1; ++dt) {
        const int tt = t + dt;
        if (tt < 0 || tt >= T) continue;
#pragma unroll
        for (int dh = -1; dh <= 1; ++dh) {
          const int hh = h + dh;
          if (hh < 0 || hh >= H) continue;
          float xv[8];
          load8<F32>(x, ((frame + tt) * L + 1 + static_cast<long>(hh) * W + w) * ldx + cc, xv);
          if (dt == 0 && dh == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) cur[i] += xv[i];
          }
#pragma unroll
          for (int dw = 0; dw < 3; ++dw) {
            float wv[8];
            unpack8(*reinterpret_cast<const uint4*>(wsm + (((dt + 1) * 3 + dh + 1) * 3 + dw) * C + cc), wv);
#pragma unroll
            for (int i = 0; i < 8; ++i) p[dw][i] = fmaf(wv[i], xv[i], p[dw][i]);
          }
        }
      }
      // column w is tap dw = +1 of row w-1, the centre of row w and tap dw = -1 of row w+1
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        prev[i] += p[2][i];
        cur[i] += p[1][i];
        next[i] += p[0][i];
      }
      const long row = (nt * L + 1 + static_cast<long>(h) * W + w - 1);
      if (w > 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) prev[i] += bias[i];
        dpe_ln_store(prev, active, C, c0, ln_w, ln_b, eps, y, row * ldy, red);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        prev[i] = cur[i];
        cur[i] = next[i];
        next[i] = 0.f;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) prev[i] += bias[i];
    dpe_ln_store(prev, active, C, c0, ln_w, ln_b, eps, y, (nt * L + static_cast<long>(h) * W + W) * ldy, red);
  }
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_dpe_ln_fwd(const void* x, int x_is_f32, long ldx, const void* conv_w, const void* conv_b,
                              const void* ln_w, const void* ln_b, float eps, int N, int T, int H, int W, int C, void* y,
                              long ldy, void* stream) {
  if (N == 0) return 0;
  if (x == nullptr || conv_w == nullptr || conv_b == nullptr || ln_w == nullptr || ln_b == nullptr || y == nullptr)
    return set_error("ivb_dpe_ln_fwd: x, conv_w, conv_b, ln_w, ln_b and y are required");
  if (N < 0 || T < 1 || H < 1 || W < 1) return set_error("ivb_dpe_ln_fwd: N >= 0 and T, H, W >= 1");
  if (C < 8 || C > DPE_MAX_C || (C & 7)) return set_error("ivb_dpe_ln_fwd: C must be a multiple of 8 in [8, 4096]");
  if ((ldx & 7) || (ldy & 7) || ldx < C || ldy < C)
    return set_error("ivb_dpe_ln_fwd: ldx and ldy must be multiples of 8 elements and >= C");
  if (misaligned(16, x, conv_b, ln_w, ln_b, y))
    return set_error("ivb_dpe_ln_fwd: x, conv_b, ln_w, ln_b and y must be 16-byte aligned");
  if (misaligned(2, conv_w)) return set_error("ivb_dpe_ln_fwd: conv_w must be 2-byte aligned");
  const int threads = (C / 8 + 31) / 32 * 32;
  const int smem = DPE_TAPS * C * 2;
  const long items = static_cast<long>(N) * T * (H + 1);
  const int grid = persistent_grid(items, 1, 8);
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const auto* cw = reinterpret_cast<const __nv_bfloat16*>(conv_w);
  const auto* cb = reinterpret_cast<const __nv_bfloat16*>(conv_b);
  const auto* lw = reinterpret_cast<const __nv_bfloat16*>(ln_w);
  const auto* lb = reinterpret_cast<const __nv_bfloat16*>(ln_b);
  auto* yy = reinterpret_cast<__nv_bfloat16*>(y);
  if (x_is_f32) {
    if (int rc = raise_smem_limit<dpe_ln_fwd_kernel<true>>(DPE_SMEM_MAX, "dpe_ln_fwd_kernel")) return rc;
    return launch("dpe_ln_fwd_kernel", dpe_ln_fwd_kernel<true>, grid, threads, smem, s, NO_PDL, x, ldx, cw, cb, lw, lb,
                  eps, N, T, H, W, C, yy, ldy);
  }
  if (int rc = raise_smem_limit<dpe_ln_fwd_kernel<false>>(DPE_SMEM_MAX, "dpe_ln_fwd_kernel")) return rc;
  return launch("dpe_ln_fwd_kernel", dpe_ln_fwd_kernel<false>, grid, threads, smem, s, NO_PDL, x, ldx, cw, cb, lw, lb,
                eps, N, T, H, W, C, yy, ldy);
}
