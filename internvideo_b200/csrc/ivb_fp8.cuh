// ivb_fp8.cuh — the power-of-two FP8 scale and the E4M3 / E5M2 conversion, shared by the per-tensor casts
// (ivb_fp8.cu), the per-row casts (ivb_fp8.cu) and the norm kernels that write FP8 rows (ivb_norm.cu).
#pragma once
#include "ivb_ptx.cuh"

namespace ivb {

// scale = 2^e with e the largest integer such that amax * 2^e <= fmax = 1.75 * 2^F, from the bits of amax (exact, no
// rounding of fmax / amax); e is clamped to [-126, 126] so that scale and 1 / scale are normal floats.
__device__ __forceinline__ void fp8_scale(unsigned amax_bits, int F, float& scale, float& scale_inv) {
  if ((amax_bits & 0x7f800000u) == 0x7f800000u) {   // Inf or NaN
    scale = 1.0f;
    scale_inv = __int_as_float(0x7fc00000);
    return;
  }
  if (amax_bits == 0) {
    scale = scale_inv = 1.0f;
    return;
  }
  const int E = static_cast<int>((amax_bits >> 23) & 0xff) - 127;
  int e = F - E - ((amax_bits & 0x7fffffu) > 0x600000u ? 1 : 0);
  e = min(126, max(-126, e));
  scale = __int_as_float((e + 127) << 23);
  scale_inv = __int_as_float((127 - e) << 23);
}

template <bool E5M2>
__device__ __forceinline__ uint32_t cvt_fp8x2(float lo, float hi) {
  uint16_t r;
  if constexpr (E5M2)
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// 8 values times `scale`, rounded to E4M3, as one 8-byte word (element 0 in the lowest byte).
__device__ __forceinline__ uint2 cvt_e4m3x8(const float v[8], float scale) {
  uint32_t q[2];
#pragma unroll
  for (int k = 0; k < 2; ++k)
    q[k] = cvt_fp8x2<false>(v[4 * k] * scale, v[4 * k + 1] * scale) |
           (cvt_fp8x2<false>(v[4 * k + 2] * scale, v[4 * k + 3] * scale) << 16);
  return make_uint2(q[0], q[1]);
}

}  // namespace ivb
