// ivb_colred.cuh — deterministic cross-CTA column sums for parameter gradients.
//
// A row-parallel backward kernel reduces its rows into one per-column partial per CTA.  Adding those partials into the
// fp32 gradient with atomics makes the result depend on the order in which CTAs finish; AdamW then turns last-bit
// differences of a near-zero gradient (LayerScale gamma starts at 1e-5) into visible parameter differences, so two
// runs of the same training step would disagree.  Instead every CTA stores its partial in a scratch slot
//   g_colred[(out * nslots + slot) * D + col]
// and colred_finish() adds the partials into the gradient in slot order: same inputs, same bits.
// The scratch is static device memory of the including translation unit (24 MB in ivb_norm.cu, 16 MB in ivb_loss.cu).
// It holds ONE reduction at a time per device: the entry points that use it must not run concurrently on two streams of
// the same device (include/ivb200.h, Conventions).  A call whose partials would not fit returns an error.
#pragma once
#include "ivb_internal.h"

namespace ivb {

#ifndef IVB_COLRED_FLOATS
#define IVB_COLRED_FLOATS (6L << 20)   // 24 MB: the largest bench user is the cfg-3 LayerScale / bias backward, ~4.2 M
#endif

static __device__ float g_colred[IVB_COLRED_FLOATS];

__device__ __forceinline__ void colred_put(int out, int nslots, int slot, int D, int col, float v) {
  g_colred[(static_cast<long>(out) * nslots + slot) * D + col] = v;
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
  colred_finish_kernel<<<dim3((D + 255) / 256, nout), 256, 0, stream>>>(nslots, D, o0, o1, o2);
  count_launch();
  return check_launch("colred_finish_kernel");
}

}  // namespace ivb
