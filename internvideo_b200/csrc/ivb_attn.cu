// ivb_attn.cu — multi-head attention forward, non-causal or causal, on Hopper wgmma (flash-style, online softmax).
//
// Stands in for FA2 flash_attn_varlen_qkvpacked_func as called by the reference's
// FlashAttention.forward (InternVideo2/single_modality/models/flash_attention_class.py:47-50) and for
// Attention._naive_attn's softmax((q*scale) k^T) v (internvideo2_pretrain.py:183-188).  The kernel body is
// ivb_attn_fwd.cuh's attn_fwd; this file instantiates its plain, DropPath-plan and causal forms.
#include <math.h>
#include <stdlib.h>

#include "ivb_attn_fwd.cuh"

namespace ivb {

template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
  attn_fwd<AttnElt::BF16, KA, NO, KS>(tmQ, tmK, tmV, p, nullptr);
}

// rowscale: the attention branch's DropPath factors [B*n]
template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_plan_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p, const float* rowscale) {
  attn_fwd<AttnElt::BF16, KA, NO, KS, true>(tmQ, tmK, tmV, p, rowscale);
}

template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_causal_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
  attn_fwd<AttnElt::BF16, KA, NO, KS, false, true>(tmQ, tmK, tmV, p, nullptr);
}

}  // namespace ivb

using namespace ivb;

// ivb_attn_fwd, ivb_attn_fwd_plan (rowscale not null) and ivb_attn_fwd_causal (causal, no rowscale); `fn` names the
// entry point in messages.
static int attn_fwd(const char* fn, const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, void* out,
                    long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale, const float* rowscale,
                    cudaStream_t stream, bool causal = false) {
  return attn_fwd_setup(fn, q, ldq, k, ldk, v, ldv, out, ldo, lse2, B, n, H, d, softmax_scale,
                        [&](auto hd, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                            const AttnFwdParams& p) {
    if (causal)
      return launch_attn<attn_fwd_causal_kernel<hd.KA, hd.NO, hd.KS>, NO_PDL>(
          "cudaFuncSetAttribute(attn_fwd_causal)", "attn_fwd_causal_kernel", FwdSmem<hd.KA>::BYTES, B, n, H, stream, tq,
          tk, tv, p);
    if (rowscale != nullptr)
      return launch_attn<attn_fwd_plan_kernel<hd.KA, hd.NO, hd.KS>, NO_PDL>(
          "cudaFuncSetAttribute(attn_fwd_plan)", "attn_fwd_plan_kernel", FwdSmem<hd.KA>::BYTES, B, n, H, stream, tq, tk,
          tv, p, rowscale);
    return launch_attn<attn_fwd_kernel<hd.KA, hd.NO, hd.KS>, NO_PDL>(
        "cudaFuncSetAttribute(attn_fwd)", "attn_fwd_kernel", FwdSmem<hd.KA>::BYTES, B, n, H, stream, tq, tk, tv, p);
  });
}

extern "C" int ivb_attn_fwd(const void* q, long ldq, const void* k, long ldk, const void* v,
                            long ldv, void* out, long ldo, float* lse2, int B, int n, int H, int d,
                            float softmax_scale, void* stream) {
  return attn_fwd("ivb_attn_fwd", q, ldq, k, ldk, v, ldv, out, ldo, lse2, B, n, H, d, softmax_scale, nullptr,
                  reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_attn_fwd_plan(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, void* out,
                                 long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                                 const float* rowscale, void* stream) {
  if (rowscale == nullptr) return set_error("ivb_attn_fwd_plan: rowscale is null");
  return attn_fwd("ivb_attn_fwd_plan", q, ldq, k, ldk, v, ldv, out, ldo, lse2, B, n, H, d, softmax_scale, rowscale,
                  reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_attn_fwd_causal(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                                   void* out, long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                                   void* stream) {
  return attn_fwd("ivb_attn_fwd_causal", q, ldq, k, ldk, v, ldv, out, ldo, lse2, B, n, H, d, softmax_scale, nullptr,
                  reinterpret_cast<cudaStream_t>(stream), true);
}

// ---------------------------------------------------------------------------------------------------------------
// Head-axis attention of the VideoMAEv2 teacher AS THE REFERENCE COMPUTES IT: videomae.py:94-97 hands
// flash_attn_func q/k/v of shape [B, H, N, d] (after permute(2,0,3,1,4)), whereas FA2's convention is
// [B, seqlen, nheads, d] — so the softmax runs over the H (= 16) heads of EACH TOKEN, not over the tokens, and the
// [B, H, N, d] result is then reinterpreted by `.reshape(B, N, -1)`.  Reproduced here for drop-in parity (the
// standard token-axis attention is the wgmma kernel above).  Tiny and HBM-bound: one warp per token stages the
// token's q/k/v ([H, d] each) in shared memory, lane (i, half) owns score row i / key half.
namespace ivb {

template <int HMAX>
__global__ void __launch_bounds__(128)
headaxis_attn_kernel(const __nv_bfloat16* __restrict__ qkv, long ld, int B, int N, int H, int d, float scale,
                     __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t hsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long tok = static_cast<long>(blockIdx.x) * 4 + warp;
  if (tok >= static_cast<long>(B) * N) return;
  const int D = H * d;
  __nv_bfloat16* sq = reinterpret_cast<__nv_bfloat16*>(hsm) + static_cast<long>(warp) * 3 * D;
  __nv_bfloat16* sk = sq + D;
  __nv_bfloat16* sv = sk + D;
  const __nv_bfloat16* row = qkv + tok * ld;
  for (int c = lane * 8; c < 3 * D; c += 256)
    *reinterpret_cast<uint4*>(sq + c) = *reinterpret_cast<const uint4*>(row + c);
  __syncwarp();
  const int b = static_cast<int>(tok / N), t = static_cast<int>(tok % N);
  // lane -> (i = lane % H ... ) : each lane owns one query head i = lane (lanes >= H idle); H <= 32
  const int i = lane;
  if (i < H) {
    float s[HMAX];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < HMAX; ++j) {
      if (j < H) {
        float acc = 0.f;
        for (int c = 0; c < d; c += 2) {
          const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sq + i * d + c));
          const float2 k2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sk + j * d + c));
          acc += a.x * k2.x + a.y * k2.y;
        }
        s[j] = acc * scale;
        mx = fmaxf(mx, s[j]);
      }
    }
    float l = 0.f;
#pragma unroll
    for (int j = 0; j < HMAX; ++j)
      if (j < H) { s[j] = __expf(s[j] - mx); l += s[j]; }
    const float inv = 1.f / l;
    __nv_bfloat16* o = out + ((static_cast<long>(b) * H + i) * N + t) * d;     // [B, H, N, d] contiguous
    for (int c = 0; c < d; c += 2) {
      float ox = 0.f, oy = 0.f;
#pragma unroll
      for (int j = 0; j < HMAX; ++j) {
        if (j < H) {
          const float2 v2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sv + j * d + c));
          ox += s[j] * v2.x; oy += s[j] * v2.y;
        }
      }
      *reinterpret_cast<__nv_bfloat162*>(o + c) = __floats2bfloat162_rn(ox * inv, oy * inv);
    }
  }
}

}  // namespace ivb

extern "C" int ivb_headaxis_attn_fwd(const void* qkv, long ld, int B, int N, int H, int d, float softmax_scale,
                                     void* out, void* stream_) {
  using namespace ivb;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || N <= 0) return 0;
  if (H > 32 || H < 1) return set_error("ivb_headaxis_attn_fwd: 1 <= heads <= 32");
  if ((d & 7) || (ld & 7)) return set_error("ivb_headaxis_attn_fwd: head_dim / pitch must be multiples of 8");
  const long toks = static_cast<long>(B) * N;
  const size_t smem = static_cast<size_t>(4) * 3 * H * d * sizeof(__nv_bfloat16);
  auto kern = H <= 16 ? headaxis_attn_kernel<16> : headaxis_attn_kernel<32>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(headaxis_attn)", e);
  }
  return launch("headaxis_attn_kernel", kern, (unsigned)((toks + 3) / 4), 128, smem, stream, NO_PDL,
                reinterpret_cast<const __nv_bfloat16*>(qkv), ld, B, N, H, d, softmax_scale,
                reinterpret_cast<__nv_bfloat16*>(out));
}
