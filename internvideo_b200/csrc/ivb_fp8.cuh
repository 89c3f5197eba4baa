// ivb_fp8.cuh — the power-of-two FP8 scale, the E4M3 / E5M2 conversion, and the pieces every FP8 cast is built from:
// the bf16 amax of a 16-byte chunk, a bounded chunk read, the column amax of a CTA, a transposing byte tile and a
// tail-safe row store.  Used by the casts of ivb_fp8.cu, the attention pack of ivb_attn_fp8.cu and the norm kernels
// that write FP8 rows (ivb_norm.cu).
//
// An amax is taken over bf16 magnitude bits (the sign cleared): as integers NaN > Inf > every finite value, so an
// integer max is the amax, the same bits in any order, and a non-finite group reaches fp8_scale as non-finite.
#pragma once
#include "ivb_ptx.cuh"
#include "ivb_rows.cuh"

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

// The largest magnitude bits of the 8 bf16 values of a chunk.
__device__ __forceinline__ unsigned bf16_mag_max(uint4 v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  unsigned m = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) m = max(m, max(w[k] & 0x7fffu, (w[k] >> 16) & 0x7fffu));
  return m;
}

// m[k] = max(m[k], magnitude bits of element k of the chunk): the running amax of a chunk's 8 columns.
__device__ __forceinline__ void bf16_mag_cols(uint4 v, unsigned (&m)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    m[2 * k] = max(m[2 * k], w[k] & 0x7fffu);
    m[2 * k + 1] = max(m[2 * k + 1], (w[k] >> 16) & 0x7fffu);
  }
}

// Elements c .. c + 7 of a bf16 row of n elements as one chunk, zeros past element n - 1, which is never read: one
// 16-byte load when the chunk lies inside the row (row + c 16-byte aligned), else 2-byte loads.
__device__ __forceinline__ uint4 load_chunk(const __nv_bfloat16* row, int c, int n) {
  if (c + 8 <= n) return *reinterpret_cast<const uint4*>(row + c);
  uint32_t w[4] = {0u, 0u, 0u, 0u};
  if (c < n) {
    const uint16_t* s16 = reinterpret_cast<const uint16_t*>(row + c);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (c + k < n) w[k >> 1] |= static_cast<uint32_t>(s16[k]) << (16 * (k & 1));
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// The column amax of a CTA of NT threads whose lane l holds in m the running amax of the 8 columns of chunk
// l % CHUNKS of its rows (CHUNKS chunks per row: lanes l, l ^ CHUNKS, ... hold the same chunk).  Shuffles, then one
// word per (warp, column) in red, then a max over the warps: no atomics, the same bits on every run.  Leaves column
// c's magnitude word in red[0][c] and returns it to thread c (c < 8 CHUNKS).
template <int CHUNKS, int NT>
__device__ __forceinline__ unsigned col_amax(unsigned (&m)[8], unsigned (&red)[NT / 32][8 * CHUNKS]) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int o = CHUNKS; o < 32; o <<= 1) m[k] = max(m[k], __shfl_xor_sync(0xffffffffu, m[k], o));
  const int lane = threadIdx.x & 31;
  if (lane < CHUNKS) {
#pragma unroll
    for (int k = 0; k < 8; ++k) red[threadIdx.x >> 5][lane * 8 + k] = m[k];
  }
  __syncthreads();
  unsigned mx = 0;
  if (threadIdx.x < 8 * CHUNKS) {   // thread c alone reads and writes column c
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) mx = max(mx, red[w][threadIdx.x]);
    red[0][threadIdx.x] = mx;
  }
  __syncthreads();
  return mx;
}

// The first n bytes of q (element 0 in the lowest byte) to a row at dst: one store of all of q when n >= sizeof(q)
// (dst aligned to it), else byte stores, none past dst[n - 1].  V: uint2 or uint4.
template <typename V>
__device__ __forceinline__ void store_fp8(uint8_t* dst, V q, int n) {
  constexpr int W = sizeof(V);
  if (n >= W) {
    *reinterpret_cast<V*>(dst) = q;
  } else {
    uint32_t w[4] = {q.x, q.y, 0u, 0u};
    if constexpr (W == 16) w[2] = q.z, w[3] = q.w;
#pragma unroll
    for (int k = 0; k < W; ++k)
      if (k < n) dst[k] = static_cast<uint8_t>(w[k >> 2] >> (8 * (k & 3)));
  }
}

// A transposing byte tile in shared memory: R rows of C bytes at a 16-byte aligned pitch of C + 16.  Tile row c holds
// input column c; tile column r holds input row r.
template <int R, int C>
struct Fp8TileT {
  static constexpr int PITCH = C + 16;
  __align__(16) uint8_t b[R * PITCH];

  // The 8 bytes of q (element 0 in the lowest byte): input row r, input columns c .. c + 7.
  __device__ __forceinline__ void put8(int c, int r, uint2 q) {
#pragma unroll
    for (int k = 0; k < 8; ++k) b[(c + k) * PITCH + r] = static_cast<uint8_t>((k < 4 ? q.x : q.y) >> (8 * (k & 3)));
  }
  // A chunk of input row r, input columns c .. c + 7, each times its column's scale and cast to E4M3.
  __device__ __forceinline__ void put(int c, int r, uint4 v, const float* scale) {
    float f[8];
    unpack8(v, f);
    uint32_t q[2];
#pragma unroll
    for (int k = 0; k < 2; ++k)
      q[k] = cvt_fp8x2<false>(f[4 * k] * scale[4 * k], f[4 * k + 1] * scale[4 * k + 1]) |
             (cvt_fp8x2<false>(f[4 * k + 2] * scale[4 * k + 2], f[4 * k + 3] * scale[4 * k + 3]) << 16);
    put8(c, r, make_uint2(q[0], q[1]));
  }
  // Bytes j .. j + W - 1 of tile row i, the first n of them, to dst as 16-byte pieces and a byte tail (W: a multiple
  // of 16; dst 16-byte aligned).
  template <int W>
  __device__ __forceinline__ void store(int i, int j, uint8_t* dst, int n) const {
#pragma unroll
    for (int h = 0; h < W; h += 16)
      store_fp8(dst + h, *reinterpret_cast<const uint4*>(b + i * PITCH + j + h), n - h);
  }
};

}  // namespace ivb
