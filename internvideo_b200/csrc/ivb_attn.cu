// ivb_attn.cu — non-causal multi-head attention forward on Hopper wgmma (flash-style, online softmax).
//
// Stands in for FA2 flash_attn_varlen_qkvpacked_func as called by the reference's
// FlashAttention.forward (InternVideo2/single_modality/models/flash_attention_class.py:47-50) and for
// Attention._naive_attn's softmax((q*scale) k^T) v (internvideo2_pretrain.py:183-188).
//
// One CTA per (128-query block, head, clip), 384 threads: warpgroup 0 is the TMA producer (one elected thread),
// warpgroups 1 and 2 own 64 query rows each.  Per 64-key tile a warpgroup computes S = Q K_j^T with wgmma from
// shared memory, runs the online softmax on the accumulator fragments (a row lives in the four threads of a quad),
// and issues O += P V_j with P taken straight from registers (the fp32 accumulator layout of S is the bf16
// register-A layout of the next wgmma).  K/V tiles are double-buffered with TMA; q/k/v are read straight out of
// the [tokens, (3|2)*H*d] projection buffers through 4-D tensor maps (d, head, token, clip), so head_dim 88 is
// zero-padded by TMA's OOB fill and the sequence tail (n = 417, 833, 1025, 2049...) needs no host-side padding.
#include <math.h>
#include <stdlib.h>

#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

constexpr int ATT_BQ = 128;   // queries per CTA (two warpgroups of 64)
constexpr int ATT_BKV = 64;   // keys per step
constexpr int ATT_NS = 2;     // K/V stages

struct AttnFwdParams {
  int B, n, H, d;
  float sc_log2;     // softmax_scale * log2(e)
  __nv_bfloat16* out;
  long ldo;
  float* lse2;       // [B, H, n]  log2-domain logsumexp of the scaled scores
};

// Quad reductions: the four threads (lane & 3) of a quad share an accumulator row.
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// KA: number of 64-wide atoms covering head_dim (1: d<=64, 2: d<=128).  NO: wgmma N of P·V (d rounded up).
template <int KA, int NO>
__global__ void __launch_bounds__(384, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
  constexpr int Q_BYTES = KA * ATT_BQ * 128;        // KA atoms of [128 rows x 128 B]
  constexpr int KV_BYTES = KA * ATT_BKV * 128;      // KA atoms of [64 rows x 128 B]
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;                  // ATT_NS stages
  uint8_t* sV = sK + ATT_NS * KV_BYTES;        // ATT_NS stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ATT_NS * KV_BYTES);
  uint64_t* bar_q = bars;                       // 1
  uint64_t* full_k = bars + 1;                  // ATT_NS
  uint64_t* full_v = full_k + ATT_NS;           // ATT_NS
  uint64_t* empty_k = full_v + ATT_NS;          // ATT_NS (one arrival per MMA warpgroup)
  uint64_t* empty_v = empty_k + ATT_NS;         // ATT_NS

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = tid >> 7;
  const int q0 = blockIdx.x * ATT_BQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int nblk = (p.n + ATT_BKV - 1) / ATT_BKV;
  const int ksteps = (p.d + 15) / 16;

  if (tid == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();
    mbar_init(bar_q, 1);
    for (int i = 0; i < ATT_NS; ++i) {
      mbar_init(&full_k[i], 1); mbar_init(&full_v[i], 1);
      mbar_init(&empty_k[i], 2); mbar_init(&empty_v[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<24>();
    // ===================== TMA producer =====================
    if (warp == 0 && elect_one()) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
      mbar_expect_tx(bar_q, Q_BYTES);
#pragma unroll
      for (int a = 0; a < KA; ++a)
        tma_load_4d(sQ + a * (ATT_BQ * 128), &tmQ, a * 64, h, q0, b, bar_q);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % ATT_NS;
        const uint32_t ph = ((j / ATT_NS) & 1) ^ 1;
        mbar_wait(&empty_k[st], ph);
        mbar_expect_tx(&full_k[st], KV_BYTES);
#pragma unroll
        for (int a = 0; a < KA; ++a)
          tma_load_4d(sK + st * KV_BYTES + a * (ATT_BKV * 128), &tmK, a * 64, h, j * ATT_BKV, b, &full_k[st]);
        mbar_wait(&empty_v[st], ph);
        mbar_expect_tx(&full_v[st], KV_BYTES);
#pragma unroll
        for (int a = 0; a < KA; ++a)
          tma_load_4d(sV + st * KV_BYTES + a * (ATT_BKV * 128), &tmV, a * 64, h, j * ATT_BKV, b, &full_v[st]);
      }
    }
  } else {
    setmaxnreg_inc<240>();
    // ===================== MMA + softmax warpgroups =====================
    const int cw = wg - 1;                                  // query rows [64*cw, 64*cw + 64) of the block
    const bool signal = (tid & 127) == 0;
    const int rloc = cw * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows: rloc, rloc + 8
    const uint32_t qa = smem_u32(sQ) + cw * 8192;
    float o[NO / 2];
#pragma unroll
    for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};

    mbar_wait(bar_q, 0);
    for (int j = 0; j < nblk; ++j) {
      const int st = j % ATT_NS;
      const uint32_t ph = (j / ATT_NS) & 1;
      mbar_wait(&full_k[st], ph);
      const uint32_t ka = smem_u32(sK + st * KV_BYTES);
      float s[ATT_BKV / 2];
      wgmma_fence();
      for (int kk = 0; kk < ksteps; ++kk) {
        const uint32_t off = (kk & 3) * 32;
        Wgmma<ATT_BKV>::ss<0, 0>(s, gmma_desc(qa + (kk >> 2) * (ATT_BQ * 128) + off, 16, 1024),
                                 gmma_desc(ka + (kk >> 2) * (ATT_BKV * 128) + off, 16, 1024), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(s, ATT_BKV / 2);
      if (signal) mbar_arrive(&empty_k[st]);

      const int valid = p.n - j * ATT_BKV;  // columns >= valid are beyond the sequence
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < ATT_BKV / 2; ++i) {
        const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        float v = s[i] * p.sc_log2;
        if (col >= valid) v = -INFINITY;
        s[i] = v;
        mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
      }
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float m_new = fmaxf(m_run[r], quad_max(mx[r]));
        alpha[r] = exp2f(m_run[r] - m_new);
        m_run[r] = m_new;
      }
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < ATT_BKV / 2; ++i) {
        const int r = (i >> 1) & 1;
        s[i] = exp2f(s[i] - m_run[r]);
        rs[r] += s[i];
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + rs[r];
#pragma unroll
      for (int i = 0; i < NO / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      uint32_t pa[ATT_BKV / 16][4];
#pragma unroll
      for (int kk = 0; kk < ATT_BKV / 16; ++kk) acc_to_a_frag(s, kk, pa[kk]);

      mbar_wait(&full_v[st], ph);
      const uint32_t va = smem_u32(sV + st * KV_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < ATT_BKV / 16; ++kk)
        Wgmma<NO>::rs<1>(o, pa[kk], gmma_desc(va + kk * 2048, ATT_BKV * 128, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(o, NO / 2);
      if (signal) mbar_arrive(&empty_v[st]);
    }

#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] = quad_sum(l_run[r]);
      const int q = q0 + rloc + 8 * r;
      if (q < p.n) {
        const float inv_l = 1.0f / l_run[r];
        __nv_bfloat16* orow = p.out + (static_cast<long>(b) * p.n + q) * p.ldo + h * p.d;
#pragma unroll
        for (int jn = 0; jn < NO / 8; ++jn) {
          const int c = 8 * jn + 2 * (lane & 3);
          if (c < p.d)
            *reinterpret_cast<uint32_t*>(orow + c) = pack_bf16(o[4 * jn + 2 * r] * inv_l, o[4 * jn + 2 * r + 1] * inv_l);
        }
        if (p.lse2 != nullptr && (lane & 3) == 0)
          p.lse2[(static_cast<long>(b) * p.H + h) * p.n + q] = m_run[r] + log2f(l_run[r]);
      }
    }
  }
}

// 4-D view (d, head, token, clip) of a [B*n, ld] projection buffer starting at `base`.
int make_head_tmap(CUtensorMap* tm, const void* base, long ld, int B, int n, int H, int d,
                   int box_tokens) {
  const uint64_t dims[4] = {(uint64_t)d, (uint64_t)H, (uint64_t)n, (uint64_t)B};
  const long strides[3] = {(long)d, ld, (long)n * ld};
  const uint32_t box[4] = {64, 1, (uint32_t)box_tokens, 1};
  return make_tmap_4d(tm, base, dims, strides, box);
}

template <int KA, int NO>
static int launch_attn_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                           const AttnFwdParams& p, cudaStream_t stream) {
  constexpr int SMEM = KA * ATT_BQ * 128 + 2 * ATT_NS * KA * ATT_BKV * 128 + 128;  // tiles + barriers
  auto kern = attn_fwd_kernel<KA, NO>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(attn_fwd)", e);
  }
  dim3 grid((p.n + ATT_BQ - 1) / ATT_BQ, p.H, p.B);
  kern<<<grid, 384, SMEM, stream>>>(tq, tk, tv, p);
  count_launch();
  return check_launch("attn_fwd_kernel");
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_attn_fwd(const void* q, long ldq, const void* k, long ldk, const void* v,
                            long ldv, void* out, long ldo, float* lse2, int B, int n, int H, int d,
                            float softmax_scale, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || n <= 0) return 0;
  if (d % 8 != 0 || d > 128 || d < 16) return set_error("ivb_attn_fwd: head_dim must be a multiple of 8 in [16,128]");
  if ((ldq & 7) || (ldk & 7) || (ldv & 7) || (ldo & 7)) return set_error("ivb_attn_fwd: pitches must be multiples of 8");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_head_tmap(&tq, q, ldq, B, n, H, d, ATT_BQ))) return rc;
  if ((rc = make_head_tmap(&tk, k, ldk, B, n, H, d, ATT_BKV))) return rc;
  if ((rc = make_head_tmap(&tv, v, ldv, B, n, H, d, ATT_BKV))) return rc;
  AttnFwdParams p;
  p.B = B; p.n = n; p.H = H; p.d = d;
  p.sc_log2 = softmax_scale * 1.4426950408889634f;
  p.out = reinterpret_cast<__nv_bfloat16*>(out); p.ldo = ldo; p.lse2 = lse2;
  const int no = (d + 31) / 32 * 32;
  if (d <= 64) {
    if (no <= 32) return launch_attn_fwd<1, 32>(tq, tk, tv, p, stream);
    return launch_attn_fwd<1, 64>(tq, tk, tv, p, stream);
  }
  if (no <= 96) return launch_attn_fwd<2, 96>(tq, tk, tv, p, stream);
  return launch_attn_fwd<2, 128>(tq, tk, tv, p, stream);
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
  kern<<<(unsigned)((toks + 3) / 4), 128, smem, stream>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), ld, B, N, H, d,
                                                          softmax_scale, reinterpret_cast<__nv_bfloat16*>(out));
  count_launch();
  return check_launch("headaxis_attn_kernel");
}
