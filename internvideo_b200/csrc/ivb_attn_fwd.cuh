// ivb_attn_fwd.cuh — the attention forward, built from the pieces in ivb_attn.cuh: one device body for bf16 and E4M3
// operands, with the compile-time switches of each entry point's kernel, and the host setup the bf16 entry points
// share.  ivb_attn.cu instantiates the plain, DropPath-plan and causal kernels, ivb_attn_keylen.cu the key-length
// kernels, ivb_attn_fp8.cu the E4M3 inference kernel (its operands and scales are described there).
//
// One CTA per (128-query block, head, clip) (ivb_attn.cuh): Q is loaded once, 64-key K/V tiles stream through a ring.
// Per key tile an MMA warpgroup computes S = Q K_j^T with wgmma, runs the online softmax on the accumulator fragments
// (a row lives in the four threads of a quad) and issues O += P V_j with P straight from registers (the fp32
// accumulator layout of S is the bf16 register-A layout of the next wgmma; E4M3 P is permuted into the k32 A layout by
// p_to_e4m3_frags).  TMA zero-fills head_dim 88 and the sequence tail (n = 417, 833, ...).
#pragma once
#include <math.h>

#include <type_traits>

#include "ivb_attn.cuh"
#include "ivb_fp8.cuh"

namespace ivb {

constexpr int ATT_NS = 2;      // bf16 K/V stages
constexpr int F8_NS = 3;       // E4M3 K / V^T stages
constexpr int F8_P_SHIFT = 8;  // E4M3 P is cast as P * 2^8

// Q; the K ring and the V ring, each with its own full/empty barriers.
template <int KA>
using FwdSmem = AttnSmem<KA, 1, ATT_NS, 0, 2>;
// E4M3: the same, with each K tile's 64 column scales in a vector ring.  One 128-byte atom covers an E4M3 row of up to
// 128 columns.
using Fp8Smem = AttnSmem<1, 1, F8_NS, 1, 2>;

struct AttnFwdParams {
  int B, n, H, d;
  float sc_log2;     // softmax_scale * log2(e)
  __nv_bfloat16* out;
  long ldo;
  float* lse2;       // [B, H, n]  log2-domain logsumexp of the scaled scores
};

struct AttnFp8Params {
  int B, n, H, d, dp, n64;  // dp: head_pitch(d), a head's columns in q8 / k8; n64: fp8_scale_pitch(n)
  float sc_log2;           // softmax_scale * log2(e)
  const float* sq;         // [B, H, n64] q scale_inv
  const float* sk;         // [B, H, n64] k scale_inv
  const float* sv;         // [B, H, d]   v scale_inv
  __nv_bfloat16* out;
  long ldo;
};

// The E4M3 A fragments of P's two k32 steps from the fp32 P tile.  The accumulator gives thread t = lane % 4 of a quad
// the column pairs 8 j + 2 t, 8 j + 2 t + 1 of its two rows; the k32 A layout wants columns 4 t .. 4 t + 3 of each
// 16-column half.  Per half, a thread casts its pairs (lo: columns 2t.., hi: 8 + 2t..) to E4M3, rows 0 and 1 in one
// word each, and reads two words inside its quad: thread t takes its first two columns from thread 2 (t % 2) and the
// next two from 2 (t % 2) + 1, the lo words when t < 2 and the hi words otherwise.  In each of the two shuffles every
// thread is read by exactly one other, so it offers the one word that reader wants.  Two byte permutes then split the
// words by row.
__device__ __forceinline__ void p_to_e4m3_frags(const float (&s)[ATT_COLS / 2], int lane, uint32_t (&pa)[2][4]) {
  const int t = lane & 3, quad = lane & ~3;
  const int src1 = quad | (2 * (t & 1) + (t >> 1)), src2 = quad | (2 * (t & 1) + 1 - (t >> 1));
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int j = 4 * kk + 2 * hf;   // 8-column group of the half's lo pairs; j + 1: its hi pairs
      const uint32_t lo = cvt_fp8x2<false>(s[4 * j], s[4 * j + 1]) | (cvt_fp8x2<false>(s[4 * j + 2], s[4 * j + 3]) << 16);
      const uint32_t hi =
          cvt_fp8x2<false>(s[4 * j + 4], s[4 * j + 5]) | (cvt_fp8x2<false>(s[4 * j + 6], s[4 * j + 7]) << 16);
      const uint32_t r1 = __shfl_sync(0xffffffffu, (t & 1) ? hi : lo, src1);
      const uint32_t r2 = __shfl_sync(0xffffffffu, (t & 1) ? lo : hi, src2);
      const uint32_t first = t < 2 ? r1 : r2, second = t < 2 ? r2 : r1;
      pa[kk][2 * hf] = __byte_perm(first, second, 0x5410);       // row 0
      pa[kk][2 * hf + 1] = __byte_perm(first, second, 0x7632);   // row 1
    }
  }
}

// ELT: the operand format.  BF16 takes AttnFwdParams, a two-stage ring and k16 wgmmas; E4M3 (inference only) takes
// AttnFp8Params, a three-stage ring that also carries each K tile's column scales, V^T tiles and k32 wgmmas, scales S
// by its row and column factors before the softmax, and scales O's columns by v's channel scales at the store.
// KA: number of 128-byte atoms covering a head row (bf16: 1 for d<=64, 2 for d<=128; E4M3: 1).  NO: wgmma N of P·V (d
// rounded up to 32).  KS: k steps of S = Q K^T (bf16: ceil(d / 16) of k16; E4M3: NO / 32 of k32).
// PLAN: the CTA of a dropped clip (attn_prologue) writes zeros to its out rows and lse2 0, a finite value, to its rows.
// CAUSAL: key tiles stream up to causal_tile_end, and a warpgroup masks the tiles that cross its diagonal.
// KEYLEN: clip b keeps keys [0, kv_len[b]) for every query.  Its CTAs stream the ceil(kv_len[b] / 64) key tiles that
// hold them and mask the rest of the last one through softmax_tile's `valid`.  kv_len may be written by the kernel
// before (PDL), so it is read after the wait.  An entry outside [1, n] makes the clip's out and lse2 rows NaN.
template <AttnElt ELT, int KA, int NO, int KS, bool PLAN = false, bool CAUSAL = false, bool KEYLEN = false>
__device__ __forceinline__ void attn_fwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                         const std::conditional_t<ELT == AttnElt::E4M3, AttnFp8Params, AttnFwdParams>& p,
                                         const float* rowscale = nullptr, const int* kv_len = nullptr) {
  constexpr bool F8 = ELT == AttnElt::E4M3;
  static_assert(!F8 || (KA == 1 && !PLAN && !CAUSAL && !KEYLEN),
                "the E4M3 forward has no plan, causal or key-length form");
  using Smem = std::conditional_t<F8, Fp8Smem, FwdSmem<KA>>;
  using Slot = RingSlot<Smem::NS>;
  constexpr int PK = F8 ? 32 : 16;   // keys per k step of O += P V
  // E4M3: a K tile lands with its 64 column scales; a V^T tile is NO channel rows of 64 keys under a 64-byte swizzle.
  constexpr int K_BYTES = Smem::TILE_BYTES + (F8 ? Smem::VEC_BYTES : 0);
  constexpr int V_BYTES = F8 ? NO * ATT_COLS : Smem::TILE_BYTES;
  const AttnCta c = attn_prologue<Smem, PLAN>(p.n, rowscale);
  const long hb = static_cast<long>(c.b) * p.H + c.h;   // E4M3: the (clip, head) row of the scale arrays
  if constexpr (PLAN) {
    if (c.dead) {
      zero_rows(p.out, p.ldo, c, p.n, p.d);
      if (p.lse2 != nullptr)
        for (int r = threadIdx.x; r < min(ATT_ROWS, p.n - c.row0); r += ATT_THREADS)
          p.lse2[(static_cast<long>(c.b) * p.H + c.h) * p.n + c.row0 + r] = 0.0f;
      return;
    }
  }
  int keys = p.n;   // the clip's keys
  if constexpr (KEYLEN) {
    pdl_wait();
    keys = kv_len[c.b];
    if (keys < 1 || keys > p.n) {
      fill_rows(p.out, p.ldo, c, p.n, p.d, 0x7FC07FC0u);   // bf16 NaN pairs
      if (p.lse2 != nullptr)
        for (int r = threadIdx.x; r < min(ATT_ROWS, p.n - c.row0); r += ATT_THREADS)
          p.lse2[(static_cast<long>(c.b) * p.H + c.h) * p.n + c.row0 + r] = __int_as_float(0x7FC00000);
      return;
    }
  }
  const int nblk = CAUSAL ? causal_tile_end(c, p.n) : KEYLEN ? (keys + ATT_COLS - 1) / ATT_COLS : c.nblk;
  attn_roles(c, [&] {
    // ===================== TMA producer =====================
    int dp = 0;   // E4M3: the columns of a head in q8 / k8
    if constexpr (F8) dp = p.dp;
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_expect_tx(Smem::bar_row(), Smem::ROW_BYTES);
    load_head_rows<KA, ATT_ROWS, ELT>(Smem::rows(0), &tmQ, c.h, c.row0, c.b, Smem::bar_row(), dp);
    for (int j = 0; j < nblk; ++j) {
      const Slot s(j);
      mbar_wait(Smem::empty(0, s.st), s.ph ^ 1);
      mbar_expect_tx(Smem::full(0, s.st), K_BYTES);
      load_head_rows<KA, ATT_COLS, ELT>(Smem::tile(0, s.st), &tmK, c.h, j * ATT_COLS, c.b, Smem::full(0, s.st), dp);
      if constexpr (F8)
        bulk_load_1d(Smem::vec(0, s.st), p.sk + hb * p.n64 + j * ATT_COLS, Smem::VEC_BYTES, Smem::full(0, s.st));
      mbar_wait(Smem::empty(1, s.st), s.ph ^ 1);
      mbar_expect_tx(Smem::full(1, s.st), V_BYTES);
      if constexpr (F8)
        tma_load_4d(Smem::tile(1, s.st), &tmV, j * ATT_COLS, 0, c.h, c.b, Smem::full(1, s.st));
      else
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
    uint32_t pa[ATT_COLS / PK][4];
    float2 ks[ATT_COLS / 8];   // E4M3: the column scales of the thread's pairs of the current K tile
    float rq[2];               // E4M3: the row factors sq * sc_log2 of the thread's rows
    if constexpr (F8) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = c.row0 + c.rloc + 8 * r;
        rq[r] = row < p.n ? p.sq[hb * p.n64 + row] * p.sc_log2 : 0.f;
      }
    }
    const int q0 = CAUSAL ? c.row0 + c.rloc : 0;   // CAUSAL: this thread's first query row

    // S = Q K_j^T.  E4M3 reads the K tile's column scales first, before the S wgmma that reads the same stage is
    // issued: that wgmma completes only after every warp of the warpgroup issued it, and only then does the stage's
    // `empty` arrive.  Its k32 steps cover a head's dp = NO columns (zeros past d) in one 128-byte atom; the
    // 128-column box reads on into the next head's, which they do not reach.
    auto issue_s = [&](int j) {
      if constexpr (F8) {
        const float* v = Smem::vec(0, Slot(j).st);
#pragma unroll
        for (int jn = 0; jn < ATT_COLS / 8; ++jn) ks[jn] = *reinterpret_cast<const float2*>(v + 8 * jn + 2 * (c.lane & 3));
      }
      const uint32_t ka = smem_u32(Smem::tile(0, Slot(j).st));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        if constexpr (F8) {
          WgmmaF8<ATT_COLS>::ss<false>(s, gmma_desc(qa + kk * 32, 16, 1024), gmma_desc(ka + kk * 32, 16, 1024),
                                       kk > 0 ? 1u : 0u);
        } else {
          const uint32_t off = (kk & 3) * 32;   // steps 4.. lie in the second 64-column atom
          Wgmma<ATT_COLS>::ss<0, 0>(s, gmma_desc(qa + (kk >> 2) * (ATT_ROWS * 128) + off, 16, 1024),
                                    gmma_desc(ka + (kk >> 2) * (ATT_COLS * 128) + off, 16, 1024), kk > 0 ? 1u : 0u);
        }
      }
      wgmma_commit();
    };
    // S of tile j -> P, the columns from `valid` on 0.  E4M3 scales S by its row and column factors first.
    auto softmax = [&](int j, int valid) {
      if constexpr (F8) {
#pragma unroll
        for (int i = 0; i < ATT_COLS / 2; ++i) s[i] *= rq[(i >> 1) & 1] * ((i & 1) ? ks[i >> 2].y : ks[i >> 2].x);
      }
      // CAUSAL: tile j holds a key after one of the warpgroup's queries
      if (CAUSAL && (j + 1) * ATT_COLS > c.row0 + cw * 64) causal_mask_tile<false>(s, q0, j * ATT_COLS, c.lane);
      softmax_tile<F8 ? F8_P_SHIFT : 0>(s, valid, c.lane, F8 ? 1.0f : p.sc_log2, m_run, l_run, alpha);
    };
    auto p_frags = [&] {
      if constexpr (F8) {
        p_to_e4m3_frags(s, c.lane, pa);
      } else {
#pragma unroll
        for (int kk = 0; kk < ATT_COLS / 16; ++kk) acc_to_a_frag(s, kk, pa[kk]);
      }
    };

    mbar_wait(Smem::bar_row(), 0);
    mbar_wait(Smem::full(0, 0), 0);
    issue_s(0);
    wgmma_wait<0>();
    wgmma_reg_fence(s, ATT_COLS / 2);
    if (c.signal) mbar_arrive(Smem::empty(0, 0));
    softmax(0, keys);
    p_frags();

    auto issue_pv = [&](int j) {
      const Slot v(j);
      mbar_wait(Smem::full(1, v.st), v.ph);
      const uint32_t va = smem_u32(Smem::tile(1, v.st));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < ATT_COLS / PK; ++kk) {
        if constexpr (F8)
          WgmmaF8<NO>::rs(o, pa[kk], gmma_desc<2>(va + kk * 32, 16, 512), 1u);
        else
          Wgmma<NO>::rs<1>(o, pa[kk], gmma_desc(va + kk * 2048, ATT_COLS * 128, 1024), 1u);
      }
      wgmma_commit();
    };
    for (int j = 0; j + 1 < nblk; ++j) {
      const Slot k(j + 1);
      mbar_wait(Smem::full(0, k.st), k.ph);
      issue_s(j + 1);
      issue_pv(j);
      wgmma_wait<1>();
      wgmma_reg_fence(s, ATT_COLS / 2);
      if (c.signal) mbar_arrive(Smem::empty(0, k.st));
      softmax(j + 1, keys - (j + 1) * ATT_COLS);
      wgmma_wait<0>();
      wgmma_reg_fence(o, NO / 2);
      if (c.signal) mbar_arrive(Smem::empty(1, Slot(j).st));
#pragma unroll
      for (int i = 0; i < NO / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      p_frags();
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
    if constexpr (F8) {
      store_rows<NO, true>(o, p.out, p.ldo, c, p.n, p.d, inv_l, p.sv + hb * p.d);
    } else {
      store_rows<NO>(o, p.out, p.ldo, c, p.n, p.d, inv_l);
      if (p.lse2 != nullptr && (c.lane & 3) == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int q = c.row0 + c.rloc + 8 * r;
          if (q < p.n) p.lse2[(static_cast<long>(c.b) * p.H + c.h) * p.n + q] = m_run[r] + log2f(l_run[r]);
        }
      }
    }
  });
}

// The host side of every bf16 forward entry point (`fn` names it in messages): B = 0 or n = 0 is a no-op; the head dim
// and pitches are checked before any CUDA call; then launch(hd, tq, tk, tv, p) runs for d's HeadDim hd with the three
// tensor maps and the kernel parameters.
template <class Launch>
int attn_fwd_setup(const char* fn, const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, void* out,
                   long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale, Launch&& launch) {
  if (B <= 0 || n <= 0) return 0;
  int rc;
  if ((rc = check_head_args(fn, d, {ldq, ldk, ldv, ldo}))) return rc;
  CUtensorMap tq, tk, tv;
  if ((rc = make_head_tmap(&tq, q, ldq, B, n, H, d, ATT_ROWS))) return rc;
  if ((rc = make_head_tmap(&tk, k, ldk, B, n, H, d, ATT_COLS))) return rc;
  if ((rc = make_head_tmap(&tv, v, ldv, B, n, H, d, ATT_COLS))) return rc;
  const AttnFwdParams p{B, n, H, d, softmax_scale * 1.4426950408889634f, reinterpret_cast<__nv_bfloat16*>(out), ldo, lse2};
  return dispatch_head_dim(d, [&](auto hd) { return launch(hd, tq, tk, tv, p); });
}

}  // namespace ivb
