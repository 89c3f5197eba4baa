// ivb_colred.cuh — deterministic cross-CTA column sums for parameter gradients.
//
// A row-parallel backward kernel reduces its rows into one per-column partial per CTA.  Adding those partials into the
// fp32 gradient with atomics makes the result depend on the order in which CTAs finish; AdamW then turns last-bit
// differences of a near-zero gradient (LayerScale gamma starts at 1e-5) into visible parameter differences, so two
// runs of the same training step would disagree.  Instead every CTA stores its partial in a scratch slot
//   g_colred[(out * nslots + slot) * D + col]
// and colred_finish() adds the partials into the gradient in slot order: same inputs, same bits.
// The same scratch, with D = 1, sums the loss kernels' scalars (the losses and dtemp) in CTA order.
// The scratch is static device memory of the one translation unit that includes this header (24 MB in ivb_norm.cu);
// kernels of other translation units reach it through scalar_slots / scalar_finish (ivb_internal.h).
// It holds ONE reduction at a time per device: the entry points that use it must not run concurrently on two streams of
// the same device (include/ivb200.h, Conventions).  A call whose partials would not fit returns an error.
#pragma once
#include "ivb_internal.h"

namespace ivb {

#define IVB_COLRED_FLOATS (6L << 20)   // 24 MB: the largest bench user is the cfg-3 LayerScale / bias backward, ~4.2 M

static __device__ float g_colred[IVB_COLRED_FLOATS];

__device__ __forceinline__ void colred_put(int out, int nslots, int slot, int D, int col, float v) {
  g_colred[(static_cast<long>(out) * nslots + slot) * D + col] = v;
}

// Inside a CTA, every warp adds the rows it visits, in visiting order, into its own `nacc` accumulator rows of D fp32
// in shared memory, laid out [warp][nacc][D].  colred_zero returns the calling warp's rows, zeroed.
__device__ __forceinline__ float* colred_zero(float* smem, int nacc, int D) {
  float* acc = smem + static_cast<long>(threadIdx.x >> 5) * nacc * D;
  for (int i = threadIdx.x & 31; i < nacc * D; i += 32) acc[i] = 0.f;
  __syncwarp();
  return acc;
}

// acc[0, N) += a * b (or += a) for N = 4 or 8 columns, as 16-byte read-modify-writes.
template <int N>
__device__ __forceinline__ void colred_add(float* acc, const float* a, const float* b) {
#pragma unroll
  for (int q = 0; q < N / 4; ++q) {
    float4* p = reinterpret_cast<float4*>(acc) + q;
    float4 s = *p;
    s.x += a[4 * q] * b[4 * q]; s.y += a[4 * q + 1] * b[4 * q + 1];
    s.z += a[4 * q + 2] * b[4 * q + 2]; s.w += a[4 * q + 3] * b[4 * q + 3];
    *p = s;
  }
}
template <int N>
__device__ __forceinline__ void colred_add(float* acc, const float* a) {
#pragma unroll
  for (int q = 0; q < N / 4; ++q) {
    float4* p = reinterpret_cast<float4*>(acc) + q;
    float4 s = *p;
    s.x += a[4 * q]; s.y += a[4 * q + 1]; s.z += a[4 * q + 2]; s.w += a[4 * q + 3];
    *p = s;
  }
}

// End of the CTA's rows (after __syncthreads): for every column, slot blockIdx.x of output o < NACC * STEP (when bit o
// of `want` is set) receives accumulator o / STEP summed over warps o % STEP, o % STEP + STEP, ... < nwarps in
// increasing order, times scale[col] for the last output when scale is given.  STEP = 2 serves two gradients, one from
// the even and one from the odd warps.
template <int NACC, int STEP = 1>
__device__ __forceinline__ void colred_flush(const float* smem, int nwarps, int D, unsigned want,
                                             const __nv_bfloat16* scale = nullptr) {
  constexpr int NOUT = NACC * STEP;
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float s[NOUT] = {};
    for (int k = 0; k < nwarps; k += STEP) {
#pragma unroll
      for (int o = 0; o < NOUT; ++o) s[o] += smem[(static_cast<long>(k + o % STEP) * NACC + o / STEP) * D + i];
    }
#pragma unroll
    for (int o = 0; o < NOUT; ++o)
      if (want & (1u << o))
        colred_put(o, gridDim.x, blockIdx.x, D, i,
                   scale != nullptr && o == NOUT - 1 ? s[o] * __bfloat162float(scale[i]) : s[o]);
  }
}

static __global__ void __launch_bounds__(256) colred_finish_kernel(int nslots, int D, float* o0, float* o1, float* o2) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int out = blockIdx.y;
  float* dst = out == 0 ? o0 : (out == 1 ? o1 : o2);
  if (col >= D || dst == nullptr) return;
  const float* part = g_colred + static_cast<long>(out) * nslots * D + col;
  float s = 0.f;
  for (int k = 0; k < nslots; ++k) s += part[static_cast<long>(k) * D];
  dst[col] += s;
}

// Is there room for `nout` outputs of `nslots` partials of D columns?
static inline int colred_check(int nout, long nslots, int D, const char* who) {
  if (static_cast<long>(nout) * nslots * D > IVB_COLRED_FLOATS) return set_error(who);
  return 0;
}

// dst_o[col] += sum over slots (in slot order) of the partials of output o, for the non-null outputs among o0..o2.
static inline int colred_finish(int nout, int nslots, int D, float* o0, float* o1, float* o2, cudaStream_t stream) {
  if (o0 == nullptr && o1 == nullptr && o2 == nullptr) return 0;
  return launch("colred_finish_kernel", colred_finish_kernel, dim3((D + 255) / 256, nout), 256, 0, stream, NO_PDL, nslots,
                D, o0, o1, o2);
}

}  // namespace ivb
