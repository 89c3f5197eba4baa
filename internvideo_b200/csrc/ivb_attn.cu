// ivb_attn.cu — multi-head attention forward, non-causal or causal, on Hopper wgmma (flash-style, online softmax).
//
// Stands in for FA2 flash_attn_varlen_qkvpacked_func as called by the reference's
// FlashAttention.forward (InternVideo2/single_modality/models/flash_attention_class.py:47-50) and for
// Attention._naive_attn's softmax((q*scale) k^T) v (internvideo2_pretrain.py:183-188).
//
// One CTA per (128-query block, head, clip) (ivb_attn.cuh): Q is loaded once, 64-key K/V tiles stream through a
// two-stage ring.  Per key tile an MMA warpgroup computes S = Q K_j^T with wgmma, runs the online softmax on the
// accumulator fragments (a row lives in the four threads of a quad) and issues O += P V_j with P straight from registers
// (the fp32 accumulator layout of S is the bf16 register-A layout of the next wgmma).  TMA zero-fills head_dim 88 and
// the sequence tail (n = 417, 833, ...).
#include <math.h>
#include <stdlib.h>

#include "ivb_attn.cuh"

namespace ivb {

constexpr int ATT_NS = 2;  // K/V stages

// Q; the K ring and the V ring, each with its own full/empty barriers.
template <int KA>
using FwdSmem = AttnSmem<KA, 1, ATT_NS, 0, 2>;

struct AttnFwdParams {
  int B, n, H, d;
  float sc_log2;     // softmax_scale * log2(e)
  __nv_bfloat16* out;
  long ldo;
  float* lse2;       // [B, H, n]  log2-domain logsumexp of the scaled scores
};

// KA: number of 64-wide atoms covering head_dim (1: d<=64, 2: d<=128).  NO: wgmma N of P·V (d rounded up).
// KS: k16 steps of S = Q K^T, ceil(d / 16).
// PLAN: the CTA of a dropped clip (attn_prologue) writes zeros to its out rows and lse2 0, a finite value, to its rows.
// CAUSAL: key tiles stream up to causal_tile_end, and a warpgroup masks the tiles that cross its diagonal.
template <int KA, int NO, int KS, bool PLAN, bool CAUSAL = false>
__device__ __forceinline__ void attn_fwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                         const AttnFwdParams& p, const float* rowscale) {
  using Smem = FwdSmem<KA>;
  const AttnCta c = attn_prologue<Smem, PLAN>(p.n, rowscale);
  if (PLAN && c.dead) {
    zero_rows(p.out, p.ldo, c, p.n, p.d);
    if (p.lse2 != nullptr)
      for (int r = threadIdx.x; r < min(ATT_ROWS, p.n - c.row0); r += ATT_THREADS)
        p.lse2[(static_cast<long>(c.b) * p.H + c.h) * p.n + c.row0 + r] = 0.0f;
    return;
  }
  const int nblk = CAUSAL ? causal_tile_end(c, p.n) : c.nblk;
  attn_roles(c, [&] {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_expect_tx(Smem::bar_row(), Smem::ROW_BYTES);
    load_head_rows<KA, ATT_ROWS>(Smem::rows(0), &tmQ, c.h, c.row0, c.b, Smem::bar_row());
    for (int j = 0; j < nblk; ++j) {
      const RingSlot<ATT_NS> s(j);
      mbar_wait(Smem::empty(0, s.st), s.ph ^ 1);
      mbar_expect_tx(Smem::full(0, s.st), Smem::TILE_BYTES);
      load_head_rows<KA, ATT_COLS>(Smem::tile(0, s.st), &tmK, c.h, j * ATT_COLS, c.b, Smem::full(0, s.st));
      mbar_wait(Smem::empty(1, s.st), s.ph ^ 1);
      mbar_expect_tx(Smem::full(1, s.st), Smem::TILE_BYTES);
      load_head_rows<KA, ATT_COLS>(Smem::tile(1, s.st), &tmV, c.h, j * ATT_COLS, c.b, Smem::full(1, s.st));
    }
  }, [&](int cw) {
    // ===================== MMA + softmax warpgroups =====================
    // Pipelined within the warpgroup: S_{j+1} = Q K_{j+1}^T is issued before O += P_j V_j, so the tensor core runs
    // both while the softmax of tile j+1 waits only for S_{j+1}; O is rescaled once P_j V_j has retired.
    const uint32_t qa = smem_u32(Smem::rows(0)) + cw * 8192;   // query rows [64*cw, 64*cw + 64) of the block
    float o[NO / 2];
#pragma unroll
    for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};
    float s[ATT_COLS / 2];
    float alpha[2];
    uint32_t pa[ATT_COLS / 16][4];
    const int q0 = c.row0 + c.rloc;       // this thread's first query row
    auto mask = [&](int j) {              // CAUSAL: tile j holds a key after one of the warpgroup's queries
      if (CAUSAL && (j + 1) * ATT_COLS > c.row0 + cw * 64) causal_mask_tile<false>(s, q0, j * ATT_COLS, c.lane);
    };

    auto issue_s = [&](int j) {
      const uint32_t ka = smem_u32(Smem::tile(0, RingSlot<ATT_NS>(j).st));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        const uint32_t off = (kk & 3) * 32;
        Wgmma<ATT_COLS>::ss<0, 0>(s, gmma_desc(qa + (kk >> 2) * (ATT_ROWS * 128) + off, 16, 1024),
                                  gmma_desc(ka + (kk >> 2) * (ATT_COLS * 128) + off, 16, 1024), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
    };

    mbar_wait(Smem::bar_row(), 0);
    mbar_wait(Smem::full(0, 0), 0);
    issue_s(0);
    wgmma_wait<0>();
    wgmma_reg_fence(s, ATT_COLS / 2);
    if (c.signal) mbar_arrive(Smem::empty(0, 0));
    mask(0);
    softmax_tile(s, p.n, c.lane, p.sc_log2, m_run, l_run, alpha);
#pragma unroll
    for (int kk = 0; kk < ATT_COLS / 16; ++kk) acc_to_a_frag(s, kk, pa[kk]);

    auto issue_pv = [&](int j) {
      const RingSlot<ATT_NS> v(j);
      mbar_wait(Smem::full(1, v.st), v.ph);
      const uint32_t va = smem_u32(Smem::tile(1, v.st));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < ATT_COLS / 16; ++kk)
        Wgmma<NO>::rs<1>(o, pa[kk], gmma_desc(va + kk * 2048, ATT_COLS * 128, 1024), 1u);
      wgmma_commit();
    };
    for (int j = 0; j + 1 < nblk; ++j) {
      const RingSlot<ATT_NS> k(j + 1);
      mbar_wait(Smem::full(0, k.st), k.ph);
      issue_s(j + 1);
      issue_pv(j);
      wgmma_wait<1>();
      wgmma_reg_fence(s, ATT_COLS / 2);
      if (c.signal) mbar_arrive(Smem::empty(0, k.st));
      mask(j + 1);
      softmax_tile(s, p.n - (j + 1) * ATT_COLS, c.lane, p.sc_log2, m_run, l_run, alpha);
      wgmma_wait<0>();
      wgmma_reg_fence(o, NO / 2);
      if (c.signal) mbar_arrive(Smem::empty(1, RingSlot<ATT_NS>(j).st));
#pragma unroll
      for (int i = 0; i < NO / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
#pragma unroll
      for (int kk = 0; kk < ATT_COLS / 16; ++kk) acc_to_a_frag(s, kk, pa[kk]);
    }
    issue_pv(nblk - 1);
    wgmma_wait<0>();
    wgmma_reg_fence(o, NO / 2);

    float inv_l[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] = quad_sum(l_run[r]);
      inv_l[r] = 1.0f / l_run[r];
    }
    store_rows<NO>(o, p.out, p.ldo, c, p.n, p.d, inv_l);
    if (p.lse2 != nullptr && (c.lane & 3) == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int q = c.row0 + c.rloc + 8 * r;
        if (q < p.n) p.lse2[(static_cast<long>(c.b) * p.H + c.h) * p.n + q] = m_run[r] + log2f(l_run[r]);
      }
    }
  });
}

template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
  attn_fwd<KA, NO, KS, false>(tmQ, tmK, tmV, p, nullptr);
}

// rowscale: the attention branch's DropPath factors [B*n]
template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_plan_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p, const float* rowscale) {
  attn_fwd<KA, NO, KS, true>(tmQ, tmK, tmV, p, rowscale);
}

template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_causal_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
  attn_fwd<KA, NO, KS, false, true>(tmQ, tmK, tmV, p, nullptr);
}

}  // namespace ivb

using namespace ivb;

// ivb_attn_fwd, ivb_attn_fwd_plan (rowscale not null) and ivb_attn_fwd_causal (causal, no rowscale); `fn` names the
// entry point in messages.
static int attn_fwd(const char* fn, const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, void* out,
                    long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale, const float* rowscale,
                    cudaStream_t stream, bool causal = false) {
  if (B <= 0 || n <= 0) return 0;
  int rc;
  if ((rc = check_head_args(fn, d, {ldq, ldk, ldv, ldo}))) return rc;
  CUtensorMap tq, tk, tv;
  if ((rc = make_head_tmap(&tq, q, ldq, B, n, H, d, ATT_ROWS))) return rc;
  if ((rc = make_head_tmap(&tk, k, ldk, B, n, H, d, ATT_COLS))) return rc;
  if ((rc = make_head_tmap(&tv, v, ldv, B, n, H, d, ATT_COLS))) return rc;
  const AttnFwdParams p{B, n, H, d, softmax_scale * 1.4426950408889634f, reinterpret_cast<__nv_bfloat16*>(out), ldo, lse2};
  return dispatch_head_dim(d, [&](auto hd) {
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
