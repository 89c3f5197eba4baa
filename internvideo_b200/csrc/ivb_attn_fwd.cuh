// ivb_attn_fwd.cuh — the bf16 attention forward, built from the pieces in ivb_attn.cuh: its device body with the
// compile-time switches of each entry point's kernel, and the host setup every one of those entry points shares.
// ivb_attn.cu instantiates the plain, DropPath-plan and causal kernels, ivb_attn_keylen.cu the key-length kernels.
//
// One CTA per (128-query block, head, clip) (ivb_attn.cuh): Q is loaded once, 64-key K/V tiles stream through a
// two-stage ring.  Per key tile an MMA warpgroup computes S = Q K_j^T with wgmma, runs the online softmax on the
// accumulator fragments (a row lives in the four threads of a quad) and issues O += P V_j with P straight from registers
// (the fp32 accumulator layout of S is the bf16 register-A layout of the next wgmma).  TMA zero-fills head_dim 88 and
// the sequence tail (n = 417, 833, ...).
#pragma once
#include <math.h>

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
// KEYLEN: clip b keeps keys [0, kv_len[b]) for every query.  Its CTAs stream the ceil(kv_len[b] / 64) key tiles that
// hold them and mask the rest of the last one through softmax_tile's `valid`.  kv_len may be written by the kernel
// before (PDL), so it is read after the wait.  An entry outside [1, n] makes the clip's out and lse2 rows NaN.
template <int KA, int NO, int KS, bool PLAN, bool CAUSAL = false, bool KEYLEN = false>
__device__ __forceinline__ void attn_fwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                         const AttnFwdParams& p, const float* rowscale, const int* kv_len = nullptr) {
  using Smem = FwdSmem<KA>;
  const AttnCta c = attn_prologue<Smem, PLAN>(p.n, rowscale);
  if (PLAN && c.dead) {
    zero_rows(p.out, p.ldo, c, p.n, p.d);
    if (p.lse2 != nullptr)
      for (int r = threadIdx.x; r < min(ATT_ROWS, p.n - c.row0); r += ATT_THREADS)
        p.lse2[(static_cast<long>(c.b) * p.H + c.h) * p.n + c.row0 + r] = 0.0f;
    return;
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
    softmax_tile(s, keys, c.lane, p.sc_log2, m_run, l_run, alpha);
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
      softmax_tile(s, keys - (j + 1) * ATT_COLS, c.lane, p.sc_log2, m_run, l_run, alpha);
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
