// ivb_attn_bwd.cu — attention backward, non-causal or causal, on Hopper wgmma (two passes, no atomics, recompute of P from lse).
//
// Stands in for FA2's backward of flash_attn_varlen_qkvpacked_func (the autograd of
// FlashAttention.forward, flash_attention_class.py:47-50) / autograd of _naive_attn
// (internvideo2_pretrain.py:183-188).
//
//   delta[q]   = sum_d dO[q,d] * O[q,d]                                  (attn_bwd_prep_kernel)
//   MODE 1 (dK,dV): CTA owns 128 keys; streams 64-query tiles:
//        S^T = K Q_i^T, dP^T = V dO_i^T      (register accumulators, row = key)
//        P^T = exp2(S^T*sc - lse2[q]),  dS^T = P^T * (dP^T - delta[q]) * scale
//        dV += P^T dO_i,  dK += dS^T Q_i     (P^T / dS^T from registers, Q_i / dO_i tiles as MN-major B operands)
//   MODE 0 (dQ):    CTA owns 128 queries; streams 64-key tiles:
//        S = Q K_j^T, dP = dO V_j^T;  dS = P * (dP - delta[q]) * scale;  dQ += dS K_j
// Transposed operands are never materialised: the same 128B-swizzled TMA tile [rows x 64 cols] is a
// K-major operand (rows = M/N index) for one MMA and an MN-major operand (rows = K index) for the
// other, only the wgmma descriptor differs.
//
// CTA roles and barriers as in ivb_attn.cuh: `row` covers X and Y (the 128 owned rows), full[s] the streamed tiles
// U_j, W_j and, in MODE 1, the tile's 64 lse2/delta values.  When both warpgroups are live they take turns issuing S/dP (named barriers 1 and 2): one warpgroup's MMAs run on
// the tensor core while the other computes P / dS.  Software pipelining inside a warpgroup (S/dP of tile j+1 in
// flight during the math of tile j) does not fit the register file at d > 64 in MODE 1: dK + dV take NO registers,
// two S/dP tiles 128 and the A fragments 32.
#include <math.h>
#include <stdlib.h>

#include "ivb_attn.cuh"

namespace ivb {

struct AttnBwdParams {
  int B, n, H, d;
  int n_pad;           // row pitch of the padded lse2/delta workspaces (multiple of 64)
  float sc_log2;       // scale * log2(e)
  float scale;
  const float* lse2p;  // [B,H,n_pad]
  const float* deltap; // [B,H,n_pad]
  __nv_bfloat16* out1; long ld1;  // MODE0: dQ      MODE1: dV
  __nv_bfloat16* out2; long ld2;  //                MODE1: dK
};

// delta = rowsum(dO * O) per (token, head); also copies lse2 into the padded layout the main kernels read.
__global__ void attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ o, long ldo,
                                     const __nv_bfloat16* __restrict__ dout, long lddo,
                                     const float* __restrict__ lse2, float* __restrict__ lse2p,
                                     float* __restrict__ deltap, int B, int n, int n_pad, int H, int d) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;  // (b*n+q)*H + h
  const long total = static_cast<long>(B) * n * H;
  if (i >= total) return;
  const int h = static_cast<int>(i % H);
  const long tok = i / H;
  const __nv_bfloat16* po = o + tok * ldo + h * d;
  const __nv_bfloat16* pd = dout + tok * lddo + h * d;
  float s = 0.f;
  for (int c = 0; c < d; c += 8) {
    uint4 a = *reinterpret_cast<const uint4*>(po + c);
    uint4 g = *reinterpret_cast<const uint4*>(pd + c);
    float2 a0 = unpack_bf16(a.x), a1 = unpack_bf16(a.y), a2 = unpack_bf16(a.z), a3 = unpack_bf16(a.w);
    float2 g0 = unpack_bf16(g.x), g1 = unpack_bf16(g.y), g2 = unpack_bf16(g.z), g3 = unpack_bf16(g.w);
    s += a0.x * g0.x + a0.y * g0.y + a1.x * g1.x + a1.y * g1.y + a2.x * g2.x + a2.y * g2.y +
         a3.x * g3.x + a3.y * g3.y;
  }
  const long b = tok / n, q = tok % n;
  deltap[(b * H + h) * n_pad + q] = s;
  lse2p[(b * H + h) * n_pad + q] = lse2[(b * H + h) * n + q];
}

constexpr int BWD_NST = 3;  // streamed-tile stages

// X and Y; the U and W rings under one full/empty pair per stage; lse2 and delta of each streamed tile (MODE 1).
template <int KA>
using BwdSmem = AttnSmem<KA, 2, BWD_NST, 2, 1>;

// KA: 64-wide atoms covering head_dim (1: d <= 64, 2: d <= 128); NO: wgmma N of the accumulate MMAs;
// KS: k16 steps of the S/dP MMAs, ceil(d / 16).
// PLAN: the CTA of a dropped clip (attn_prologue) writes zeros to its output rows (dQ, or dV and dK).
// CAUSAL: MODE 1 streams the query tiles from causal_tile_begin, MODE 0 the key tiles up to causal_tile_end, and a
// warpgroup masks the tiles that cross its diagonal (P = 0 where key > query).
template <int MODE, int KA, int NO, int KS, bool PLAN, bool CAUSAL = false>
__device__ __forceinline__ void attn_bwd(const CUtensorMap& tmX, const CUtensorMap& tmY, const CUtensorMap& tmU,
                                         const CUtensorMap& tmW, const AttnBwdParams& p, const float* rowscale) {
  using Smem = BwdSmem<KA>;
  const AttnCta c = attn_prologue<Smem, PLAN>(p.n, rowscale);
  if (PLAN && c.dead) {
    zero_rows(p.out1, p.ld1, c, p.n, p.d);
    if (MODE == 1) zero_rows(p.out2, p.ld2, c, p.n, p.d);
    return;
  }
  const long hb = (static_cast<long>(c.b) * p.H + c.h) * p.n_pad;
  const int jb = CAUSAL && MODE == 1 ? causal_tile_begin(c) : 0;         // streamed tiles [jb, je)
  const int je = CAUSAL && MODE == 0 ? causal_tile_end(c, p.n) : c.nblk;
  pdl_wait();
  pdl_launch_dependents();

  attn_roles(c, [&] {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmX); tma_prefetch_desc(&tmY); tma_prefetch_desc(&tmU); tma_prefetch_desc(&tmW);
    mbar_expect_tx(Smem::bar_row(), 2 * Smem::ROW_BYTES);
    load_head_rows<KA, ATT_ROWS>(Smem::rows(0), &tmX, c.h, c.row0, c.b, Smem::bar_row());
    load_head_rows<KA, ATT_ROWS>(Smem::rows(1), &tmY, c.h, c.row0, c.b, Smem::bar_row());
    for (int j = jb; j < je; ++j) {
      const RingSlot<BWD_NST> s(j - jb);
      uint64_t* full = Smem::full(0, s.st);
      mbar_wait(Smem::empty(0, s.st), s.ph ^ 1);
      mbar_expect_tx(full, 2 * Smem::TILE_BYTES + (MODE == 1 ? 2 * Smem::VEC_BYTES : 0));
      load_head_rows<KA, ATT_COLS>(Smem::tile(0, s.st), &tmU, c.h, j * ATT_COLS, c.b, full);
      load_head_rows<KA, ATT_COLS>(Smem::tile(1, s.st), &tmW, c.h, j * ATT_COLS, c.b, full);
      if (MODE == 1) {   // the padded workspaces hold whole 64-query tiles, 256-byte aligned
        bulk_load_1d(Smem::vec(0, s.st), p.lse2p + hb + j * ATT_COLS, Smem::VEC_BYTES, full);
        bulk_load_1d(Smem::vec(1, s.st), p.deltap + hb + j * ATT_COLS, Smem::VEC_BYTES, full);
      }
    }
  }, [&](int cw) {
    // ===================== MMA + math warpgroups =====================
    const bool pingpong = c.live == 2;
    const uint32_t xa = smem_u32(Smem::rows(0)) + cw * 8192, ya = smem_u32(Smem::rows(1)) + cw * 8192;
    float acc1[NO / 2];                     // MODE 1: dV   MODE 0: dQ
    float acc2[MODE == 1 ? NO / 2 : 1];     // MODE 1: dK
#pragma unroll
    for (int i = 0; i < NO / 2; ++i) acc1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (MODE == 1 ? NO / 2 : 1); ++i) acc2[i] = 0.f;
    float row_lse[2] = {0.f, 0.f}, row_delta[2] = {0.f, 0.f};
    if (MODE == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int q = c.row0 + c.rloc + 8 * r;
        if (q < p.n_pad) { row_lse[r] = p.lse2p[hb + q]; row_delta[r] = p.deltap[hb + q]; }
      }
    }

    // Named barrier 1 + cw: "warpgroup cw may issue S/dP".  Warpgroup 0 goes first.
    if (pingpong && cw == 1) named_bar_arrive(1, 256);
    mbar_wait(Smem::bar_row(), 0);
    for (int j = jb; j < je; ++j) {
      const RingSlot<BWD_NST> s(j - jb);
      mbar_wait(Smem::full(0, s.st), s.ph);
      const uint32_t ua = smem_u32(Smem::tile(0, s.st)), wa = smem_u32(Smem::tile(1, s.st));
      const float* lse_tile = Smem::vec(0, s.st);
      const float* delta_tile = Smem::vec(1, s.st);
      float sc[ATT_COLS / 2], dp[ATT_COLS / 2];
      if (pingpong) named_bar_sync(1 + cw, 256);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        const uint32_t off = (kk & 3) * 32;
        const uint32_t ro = (kk >> 2) * (ATT_ROWS * 128) + off, co = (kk >> 2) * (ATT_COLS * 128) + off;
        Wgmma<ATT_COLS>::ss<0, 0>(sc, gmma_desc(xa + ro, 16, 1024), gmma_desc(ua + co, 16, 1024), kk > 0 ? 1u : 0u);
        Wgmma<ATT_COLS>::ss<0, 0>(dp, gmma_desc(ya + ro, 16, 1024), gmma_desc(wa + co, 16, 1024), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      // Hand the turn over; warpgroup 1 skips its last hand-over, which no one would wait for.
      if (pingpong && !(cw == 1 && j == je - 1)) named_bar_arrive(2 - cw, 256);
      wgmma_wait<0>();
      wgmma_reg_fence(sc, ATT_COLS / 2);
      wgmma_reg_fence(dp, ATT_COLS / 2);
      if constexpr (CAUSAL) {   // S = -inf gives P = 0 and so dS = 0; only the tiles that cross the diagonal
        const int r0 = c.row0 + cw * 64;
        if (MODE == 1 ? j * ATT_COLS < r0 + 64 : (j + 1) * ATT_COLS > r0)
          causal_mask_tile<MODE == 1>(sc, c.row0 + c.rloc, j * ATT_COLS, c.lane);
      }

      // P and dS in place of S and dP.  Columns beyond the sequence get P = 0.
#pragma unroll
      for (int i = 0; i < ATT_COLS / 2; ++i) {
        const int col = 8 * (i >> 2) + 2 * (c.lane & 3) + (i & 1);
        float lse, dl;
        if (MODE == 1) { lse = lse_tile[col]; dl = delta_tile[col]; }
        else { lse = row_lse[(i >> 1) & 1]; dl = row_delta[(i >> 1) & 1]; }
        const float pv = j * ATT_COLS + col < p.n ? exp2f(fmaf(sc[i], p.sc_log2, -lse)) : 0.f;
        sc[i] = pv;
        dp[i] = pv * (dp[i] - dl) * p.scale;
      }
      // Every A fragment is built before the fence: no register an in-flight wgmma reads is written after it.
      uint32_t pf[MODE == 1 ? ATT_COLS / 16 : 1][4], sf[ATT_COLS / 16][4];
#pragma unroll
      for (int kk = 0; kk < ATT_COLS / 16; ++kk) {
        if (MODE == 1) acc_to_a_frag(sc, kk, pf[kk]);
        acc_to_a_frag(dp, kk, sf[kk]);
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < ATT_COLS / 16; ++kk) {
        if (MODE == 1) {
          Wgmma<NO>::rs<1>(acc1, pf[kk], gmma_desc(wa + kk * 2048, ATT_COLS * 128, 1024), 1u);   // dV += P^T dO
          Wgmma<NO>::rs<1>(acc2, sf[kk], gmma_desc(ua + kk * 2048, ATT_COLS * 128, 1024), 1u);   // dK += dS^T Q
        } else {
          Wgmma<NO>::rs<1>(acc1, sf[kk], gmma_desc(ua + kk * 2048, ATT_COLS * 128, 1024), 1u);   // dQ += dS K
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(acc1, NO / 2);
      if (MODE == 1) wgmma_reg_fence(acc2, NO / 2);
      if (c.signal) mbar_arrive(Smem::empty(0, s.st));
    }

    store_rows<NO>(acc1, p.out1, p.ld1, c, p.n, p.d);
    if constexpr (MODE == 1) store_rows<NO>(acc2, p.out2, p.ld2, c, p.n, p.d);
  });
}

template <int MODE, int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmW,
                const AttnBwdParams p) {
  attn_bwd<MODE, KA, NO, KS, false>(tmX, tmY, tmU, tmW, p, nullptr);
}

// rowscale: the attention branch's DropPath factors [B*n]
template <int MODE, int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_plan_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                     const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmW,
                     const AttnBwdParams p, const float* rowscale) {
  attn_bwd<MODE, KA, NO, KS, true>(tmX, tmY, tmU, tmW, p, rowscale);
}

template <int MODE, int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_causal_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                       const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmW,
                       const AttnBwdParams p) {
  attn_bwd<MODE, KA, NO, KS, false, true>(tmX, tmY, tmU, tmW, p, nullptr);
}

}  // namespace ivb

using namespace ivb;

// workspace (floats) needed by ivb_attn_bwd: padded lse2 + delta, [2][B][H][round_up(n,64)]
extern "C" long ivb_attn_bwd_workspace_floats(int B, int n, int H) {
  const long n_pad = (static_cast<long>(n) + ATT_COLS - 1) / ATT_COLS * ATT_COLS;
  return 2 * static_cast<long>(B) * H * n_pad;
}

// ivb_attn_bwd, ivb_attn_bwd_plan (rowscale not null) and ivb_attn_bwd_causal (causal, no rowscale); `fn` names the
// entry point in messages.
static int attn_bwd(const char* fn, const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                    const void* out, long ldo, const void* dout, long lddo, const float* lse2, float* delta_ws, void* dq,
                    long lddq, void* dk, long lddk, void* dv, long lddv, int B, int n, int H, int d,
                    float softmax_scale, const float* rowscale, cudaStream_t stream, bool causal = false) {
  if (B <= 0 || n <= 0) return 0;
  int rc;
  char msg[128];
  auto fail = [&](const char* what) {
    snprintf(msg, sizeof(msg), "%s: %s", fn, what);
    return set_error(msg);
  };
  if ((rc = check_head_args(fn, d, {ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv}))) return rc;
  if (lse2 == nullptr || delta_ws == nullptr) return fail("lse2 and the workspace are required");
  if ((reinterpret_cast<uintptr_t>(delta_ws) & 15) != 0) return fail("workspace must be 16-byte aligned");
  const int n_pad = (n + ATT_COLS - 1) / ATT_COLS * ATT_COLS;
  const long half = static_cast<long>(B) * H * n_pad;
  float* lse2p = delta_ws;
  float* deltap = delta_ws + half;
  if (cudaError_t e = cudaMemsetAsync(delta_ws, 0, 2 * half * sizeof(float), stream))   // zero padding (0 * pad must stay 0)
    return set_error_cuda("cudaMemsetAsync(attn_bwd workspace)", e);
  const long total = static_cast<long>(B) * n * H;
  if ((rc = launch("attn_bwd_prep_kernel", attn_bwd_prep_kernel, (unsigned)((total + 127) / 128), 128, 0, stream, NO_PDL,
                   reinterpret_cast<const __nv_bfloat16*>(out), ldo, reinterpret_cast<const __nv_bfloat16*>(dout),
                   lddo, lse2, lse2p, deltap, B, n, n_pad, H, d)))
    return rc;
  // q, dO, k, v, each with a 128-row box (the rows a CTA owns) and a 64-row box (a streamed tile)
  const void* src[4] = {q, dout, k, v};
  const long ld[4] = {ldq, lddo, ldk, ldv};
  CUtensorMap rows[4], tiles[4];
  for (int i = 0; i < 4; ++i)
    if ((rc = make_head_tmap(&rows[i], src[i], ld[i], B, n, H, d, ATT_ROWS)) ||
        (rc = make_head_tmap(&tiles[i], src[i], ld[i], B, n, H, d, ATT_COLS)))
      return rc;
  const float sc_log2 = softmax_scale * 1.4426950408889634f;
  const auto bf = [](void* x) { return reinterpret_cast<__nv_bfloat16*>(x); };
  const AttnBwdParams pkv{B, n, H, d, n_pad, sc_log2, softmax_scale, lse2p, deltap, bf(dv), lddv, bf(dk), lddk};
  const AttnBwdParams pq{B, n, H, d, n_pad, sc_log2, softmax_scale, lse2p, deltap, bf(dq), lddq, nullptr, 0};
  return dispatch_head_dim(d, [&](auto hd) {
    constexpr int smem = BwdSmem<hd.KA>::BYTES;
    if (causal) {
      const char* attr = "cudaFuncSetAttribute(attn_bwd_causal)";
      if ((rc = launch_attn<attn_bwd_causal_kernel<1, hd.KA, hd.NO, hd.KS>, ALLOW_PDL>(
               attr, "attn_bwd_causal_kernel", smem, B, n, H, stream, rows[2], rows[3], tiles[0], tiles[1], pkv)))
        return rc;
      return launch_attn<attn_bwd_causal_kernel<0, hd.KA, hd.NO, hd.KS>, ALLOW_PDL>(
          attr, "attn_bwd_causal_kernel", smem, B, n, H, stream, rows[0], rows[1], tiles[2], tiles[3], pq);
    }
    if (rowscale != nullptr) {
      const char* attr = "cudaFuncSetAttribute(attn_bwd_plan)";
      if ((rc = launch_attn<attn_bwd_plan_kernel<1, hd.KA, hd.NO, hd.KS>, ALLOW_PDL>(
               attr, "attn_bwd_plan_kernel", smem, B, n, H, stream, rows[2], rows[3], tiles[0], tiles[1], pkv,
               rowscale)))
        return rc;
      return launch_attn<attn_bwd_plan_kernel<0, hd.KA, hd.NO, hd.KS>, ALLOW_PDL>(
          attr, "attn_bwd_plan_kernel", smem, B, n, H, stream, rows[0], rows[1], tiles[2], tiles[3], pq, rowscale);
    }
    const char* attr = "cudaFuncSetAttribute(attn_bwd)";
    if ((rc = launch_attn<attn_bwd_kernel<1, hd.KA, hd.NO, hd.KS>, ALLOW_PDL>(attr, "attn_bwd_kernel", smem, B, n, H,
                                                                               stream, rows[2], rows[3], tiles[0],
                                                                               tiles[1], pkv)))
      return rc;
    return launch_attn<attn_bwd_kernel<0, hd.KA, hd.NO, hd.KS>, ALLOW_PDL>(attr, "attn_bwd_kernel", smem, B, n, H, stream,
                                                                            rows[0], rows[1], tiles[2], tiles[3], pq);
  });
}

extern "C" int ivb_attn_bwd(const void* q, long ldq, const void* k, long ldk, const void* v,
                            long ldv, const void* out, long ldo, const void* dout, long lddo,
                            const float* lse2, float* delta_ws, void* dq, long lddq, void* dk,
                            long lddk, void* dv, long lddv, int B, int n, int H, int d,
                            float softmax_scale, void* stream) {
  return attn_bwd("ivb_attn_bwd", q, ldq, k, ldk, v, ldv, out, ldo, dout, lddo, lse2, delta_ws, dq, lddq, dk, lddk, dv,
                  lddv, B, n, H, d, softmax_scale, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_attn_bwd_plan(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                                 const void* out, long ldo, const void* dout, long lddo, const float* lse2,
                                 float* delta_ws, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv, int B,
                                 int n, int H, int d, float softmax_scale, const float* rowscale, void* stream) {
  if (rowscale == nullptr) return set_error("ivb_attn_bwd_plan: rowscale is null");
  return attn_bwd("ivb_attn_bwd_plan", q, ldq, k, ldk, v, ldv, out, ldo, dout, lddo, lse2, delta_ws, dq, lddq, dk, lddk,
                  dv, lddv, B, n, H, d, softmax_scale, rowscale, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_attn_bwd_causal(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                                   const void* out, long ldo, const void* dout, long lddo, const float* lse2,
                                   float* delta_ws, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv, int B,
                                   int n, int H, int d, float softmax_scale, void* stream) {
  return attn_bwd("ivb_attn_bwd_causal", q, ldq, k, ldk, v, ldv, out, ldo, dout, lddo, lse2, delta_ws, dq, lddq, dk,
                  lddk, dv, lddv, B, n, H, d, softmax_scale, nullptr, reinterpret_cast<cudaStream_t>(stream), true);
}
