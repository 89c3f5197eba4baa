// ivb_rope.cu — rotary position embedding of the q and k heads, in place (LLaMA's attention,
// transformers' modeling_llama.apply_rotary_pos_emb with rotate_half; the InternVideo2-CLIP text tower,
// backbones/internvideo2/internvideo2_clip_text.py).
//
// Head h of row r = b*L + l holds d columns x_0 .. x_{d-1}; with half = d/2 and (c, s) = (cos, sin)[l, j]:
//   x_j' = x_j c - x_{j+half} s,   x_{j+half}' = x_{j+half} c + x_j s,   j < half,
// in fp32 (two products and one add each, fused), rounded to bf16 once.  One thread owns 8 pairs: a 16-byte piece of the
// first half and the matching piece of the second, so every access is a 16-byte vector.
#include <cstdio>

#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

constexpr int ROPE_THREADS = 256;

__device__ __forceinline__ void rope_piece(__nv_bfloat16* x, int half, const float* c, const float* s) {
  uint4 lo = *reinterpret_cast<const uint4*>(x);
  uint4 hi = *reinterpret_cast<const uint4*>(x + half);
  const float4 c0 = reinterpret_cast<const float4*>(c)[0], c1 = reinterpret_cast<const float4*>(c)[1];
  const float4 s0 = reinterpret_cast<const float4*>(s)[0], s1 = reinterpret_cast<const float4*>(s)[1];
  const float cv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
  const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  uint32_t* lw = reinterpret_cast<uint32_t*>(&lo);
  uint32_t* hw = reinterpret_cast<uint32_t*>(&hi);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 a = unpack_bf16(lw[k]), b = unpack_bf16(hw[k]);
    const int j = 2 * k;
    lw[k] = pack_bf16(fmaf(a.x, cv[j], -b.x * sv[j]), fmaf(a.y, cv[j + 1], -b.y * sv[j + 1]));
    hw[k] = pack_bf16(fmaf(b.x, cv[j], a.x * sv[j]), fmaf(b.y, cv[j + 1], a.y * sv[j + 1]));
  }
  *reinterpret_cast<uint4*>(x) = lo;
  *reinterpret_cast<uint4*>(x + half) = hi;
}

// Work item i: piece p = i % pieces of head h of tensor t (0: q, 1: k) of row r, i = ((r * 2 + t) * H + h) * pieces + p.
__global__ void __launch_bounds__(ROPE_THREADS) rope_qk_kernel(__nv_bfloat16* __restrict__ q, long ldq,
                                                              __nv_bfloat16* __restrict__ k, long ldk, long rows, int L,
                                                              int H, int d, const float* __restrict__ cos_t,
                                                              const float* __restrict__ sin_t) {
  const int half = d / 2, pieces = half / 8;
  const long items = rows * 2 * H * pieces;
  for (long i = static_cast<long>(blockIdx.x) * ROPE_THREADS + threadIdx.x; i < items;
       i += static_cast<long>(gridDim.x) * ROPE_THREADS) {
    const int p = static_cast<int>(i % pieces);
    const long rest = i / pieces;
    const int h = static_cast<int>(rest % H);
    const long rt = rest / H;
    const int t = static_cast<int>(rt & 1);
    const long r = rt >> 1;
    const long l = r % L;
    __nv_bfloat16* x = (t == 0 ? q + r * ldq : k + r * ldk) + h * d + p * 8;
    rope_piece(x, half, cos_t + l * half + p * 8, sin_t + l * half + p * 8);
  }
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_rope_qk(void* q, long ldq, void* k, long ldk, int B, int L, int H, int d, const float* cos_t,
                           const float* sin_t, void* stream) {
  if (B <= 0 || L <= 0) return 0;
  if (q == nullptr || k == nullptr || cos_t == nullptr || sin_t == nullptr)
    return set_error("ivb_rope_qk: q, k, cos and sin are required");
  if (H <= 0 || d < 16 || d > 128 || (d & 15)) return set_error("ivb_rope_qk: H > 0 and d a multiple of 16 in [16, 128]");
  if ((ldq & 7) || (ldk & 7) || ldq < static_cast<long>(H) * d || ldk < static_cast<long>(H) * d)
    return set_error("ivb_rope_qk: ldq and ldk must be multiples of 8 elements and >= H*d");
  if (misaligned(16, q, k, cos_t, sin_t)) return set_error("ivb_rope_qk: q, k, cos and sin must be 16-byte aligned");
  const long rows = static_cast<long>(B) * L;
  const long items = rows * 2 * H * (d / 16);
  const int grid = persistent_grid(items, ROPE_THREADS, 8);
  return launch("rope_qk_kernel", rope_qk_kernel, grid, ROPE_THREADS, 0, reinterpret_cast<cudaStream_t>(stream), NO_PDL,
                reinterpret_cast<__nv_bfloat16*>(q), ldq, reinterpret_cast<__nv_bfloat16*>(k), ldk, rows, L, H, d,
                cos_t, sin_t);
}
