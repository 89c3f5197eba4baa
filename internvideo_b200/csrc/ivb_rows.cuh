// ivb_rows.cuh — 8-element row accesses of the HBM-bound kernels: one 16-byte bf16 vector or two 16-byte fp32
// vectors, converted to / from 8 floats.  Element offsets are multiples of 8 and base pointers 16-byte aligned.
#pragma once
#include "ivb_ptx.cuh"

namespace ivb {

__device__ __forceinline__ void unpack8(const uint4& u, float v[8]) {
  float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
  v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y; v[4] = f2.x; v[5] = f2.y; v[6] = f3.x; v[7] = f3.y;
}

template <bool F32>
__device__ __forceinline__ void load8(const void* base, long elem_off, float v[8]) {
  if (F32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem_off);
    float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(base) + elem_off);
    unpack8(u, v);
  }
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

}  // namespace ivb
