// ivb_attn_fp8.cu — FP8 (E4M3) attention forward for inference: ivb_attn_fp8_pack casts q, k and v, ivb_attn_fwd_fp8
// computes softmax(scale q k^T) v on the FP8 tensor cores.
//
// Every scale is a power of two from an amax by the ivb_fp8_quantize_rows rule (ivb_fp8.cuh), so dequantisation is exact:
//   q8, k8  [B*n, H*dp]      one scale per (token, head), from the amax of that head's d columns of the row; a head
//                            takes dp = round_up(d, 32) columns, the k32 steps of S = Q K^T, the last dp - d of them
//                            zeros (a TMA box starts 16-byte aligned: an E4M3 head of 88 columns would start at 88 h)
//   vt8     [B, H, d, ldvt]  V^T per (clip, head), one scale per (clip, head, channel), from the amax over the clip's n
//                            tokens; keys n .. round_up(n, 16) are zeros
// fp8 wgmma takes only K-major operands.  For S = Q K^T the K dimension is the head dim, which q8 and k8 rows already
// are; for O += P V it is the key index, hence V^T.
//
// The forward is the CTA of ivb_attn.cu (ivb_attn.cuh) with E4M3 tiles and k32 wgmmas:
//   S_ij = (sq_i scale log2e) sk_j (q8_i . k8_j)   the row factors are loaded once per thread; the 64 column factors of
//                                                   a K tile land in its ring stage under the tile's `full` barrier
//   P    = exp2(S - m + 8)                         the bf16 kernel's online softmax with P scaled by 2^8 (P <= 256 < 448,
//                                                   and small probabilities stay in E4M3's normal range), cast to E4M3
//                                                   and permuted into the k32 A layout in registers
//   O    = (sum P8 V8) sv_c / l                    sv and 1/l are column and row factors of the bf16 store; l sums the
//                                                   same 2^8-scaled P, so the factor cancels
#include <math.h>
#include <stdlib.h>

#include "ivb_attn.cuh"
#include "ivb_fp8.cuh"
#include "ivb_rows.cuh"

namespace ivb {

constexpr int F8_NS = 3;       // K / V^T stages
constexpr int F8_P_SHIFT = 8;  // P is cast to E4M3 as P * 2^8

// Q; the K ring with each tile's 64 column scales, and the V^T ring, each with its own full/empty barriers.  One
// 128-byte atom covers an E4M3 row of up to 128 columns.
using Fp8Smem = AttnSmem<1, 1, F8_NS, 1, 2>;

// Pitch of the per-(clip, head) q and k scale rows: whole 64-key tiles, so a tile's column scales are one 256-byte
// aligned bulk copy.
__host__ __device__ inline int fp8_scale_pitch(int n) { return (n + ATT_COLS - 1) / ATT_COLS * ATT_COLS; }
__host__ __device__ inline long round16(long n) { return (n + 15) / 16 * 16; }
__host__ __device__ inline int head_pitch(int d) { return (d + 31) / 32 * 32; }

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

// NO: the head dim rounded up to 32, the N of O += P V; NO / 32 k32 steps of S = Q K^T.
template <int NO>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_fp8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnFp8Params p) {
  using Smem = Fp8Smem;
  constexpr int KS = NO / 32;
  constexpr int V_BYTES = NO * ATT_COLS;   // a V^T tile: NO channel rows of 64 keys, 64-byte swizzle
  const AttnCta c = attn_prologue<Smem>(p.n);
  const long hb = static_cast<long>(c.b) * p.H + c.h;
  attn_roles(c, [&] {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_expect_tx(Smem::bar_row(), Smem::ROW_BYTES);
    load_head_rows<1, ATT_ROWS, AttnElt::E4M3>(Smem::rows(0), &tmQ, c.h, c.row0, c.b, Smem::bar_row(), p.dp);
    for (int j = 0; j < c.nblk; ++j) {
      const RingSlot<F8_NS> s(j);
      mbar_wait(Smem::empty(0, s.st), s.ph ^ 1);
      mbar_expect_tx(Smem::full(0, s.st), Smem::TILE_BYTES + Smem::VEC_BYTES);
      load_head_rows<1, ATT_COLS, AttnElt::E4M3>(Smem::tile(0, s.st), &tmK, c.h, j * ATT_COLS, c.b,
                                                  Smem::full(0, s.st), p.dp);
      bulk_load_1d(Smem::vec(0, s.st), p.sk + hb * p.n64 + j * ATT_COLS, Smem::VEC_BYTES, Smem::full(0, s.st));
      mbar_wait(Smem::empty(1, s.st), s.ph ^ 1);
      mbar_expect_tx(Smem::full(1, s.st), V_BYTES);
      tma_load_4d(Smem::tile(1, s.st), &tmV, j * ATT_COLS, 0, c.h, c.b, Smem::full(1, s.st));
    }
  }, [&](int cw) {
    // ===================== MMA + softmax warpgroups =====================
    // The pipeline of ivb_attn.cu: S_{j+1} is issued before O += P_j V_j.
    const uint32_t qa = smem_u32(Smem::rows(0)) + cw * 8192;   // query rows [64*cw, 64*cw + 64) of the block
    float o[NO / 2];
#pragma unroll
    for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};
    float s[ATT_COLS / 2];
    float alpha[2];
    float2 ks[ATT_COLS / 8];   // the column scales of the thread's pairs of the current K tile
    uint32_t pa[2][4];
    float rq[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = c.row0 + c.rloc + 8 * r;
      rq[r] = row < p.n ? p.sq[hb * p.n64 + row] * p.sc_log2 : 0.f;
    }

    // The k32 steps cover a head's dp = NO columns (zeros past d); the 128-column box reads on into the next head's,
    // which they do not reach.
    mbar_wait(Smem::bar_row(), 0);

    // The column scales are read before the S wgmma that reads the same stage is issued: that wgmma completes only
    // after every warp of the warpgroup issued it, and only then does the stage's `empty` arrive.
    auto load_ks = [&](int j) {
      const float* v = Smem::vec(0, RingSlot<F8_NS>(j).st);
#pragma unroll
      for (int jn = 0; jn < ATT_COLS / 8; ++jn) ks[jn] = *reinterpret_cast<const float2*>(v + 8 * jn + 2 * (c.lane & 3));
    };
    auto issue_s = [&](int j) {
      const uint32_t ka = smem_u32(Smem::tile(0, RingSlot<F8_NS>(j).st));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KS; ++kk)
        WgmmaF8<ATT_COLS>::ss<false>(s, gmma_desc(qa + kk * 32, 16, 1024), gmma_desc(ka + kk * 32, 16, 1024),
                                     kk > 0 ? 1u : 0u);
      wgmma_commit();
    };
    auto scale_s = [&] {
#pragma unroll
      for (int i = 0; i < ATT_COLS / 2; ++i) s[i] *= rq[(i >> 1) & 1] * ((i & 1) ? ks[i >> 2].y : ks[i >> 2].x);
    };

    mbar_wait(Smem::full(0, 0), 0);
    load_ks(0);
    issue_s(0);
    wgmma_wait<0>();
    wgmma_reg_fence(s, ATT_COLS / 2);
    if (c.signal) mbar_arrive(Smem::empty(0, 0));
    scale_s();
    softmax_tile<F8_P_SHIFT>(s, p.n, c.lane, 1.0f, m_run, l_run, alpha);
    p_to_e4m3_frags(s, c.lane, pa);

    auto issue_pv = [&](int j) {
      const RingSlot<F8_NS> v(j);
      mbar_wait(Smem::full(1, v.st), v.ph);
      const uint32_t va = smem_u32(Smem::tile(1, v.st));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) WgmmaF8<NO>::rs(o, pa[kk], gmma_desc<2>(va + kk * 32, 16, 512), 1u);
      wgmma_commit();
    };
    for (int j = 0; j + 1 < c.nblk; ++j) {
      const RingSlot<F8_NS> k(j + 1);
      mbar_wait(Smem::full(0, k.st), k.ph);
      load_ks(j + 1);
      issue_s(j + 1);
      issue_pv(j);
      wgmma_wait<1>();
      wgmma_reg_fence(s, ATT_COLS / 2);
      if (c.signal) mbar_arrive(Smem::empty(0, k.st));
      scale_s();
      softmax_tile<F8_P_SHIFT>(s, p.n - (j + 1) * ATT_COLS, c.lane, 1.0f, m_run, l_run, alpha);
      wgmma_wait<0>();
      wgmma_reg_fence(o, NO / 2);
      if (c.signal) mbar_arrive(Smem::empty(1, RingSlot<F8_NS>(j).st));
#pragma unroll
      for (int i = 0; i < NO / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      p_to_e4m3_frags(s, c.lane, pa);
    }
    issue_pv(c.nblk - 1);
    wgmma_wait<0>();
    wgmma_reg_fence(o, NO / 2);

    float inv_l[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) inv_l[r] = 1.0f / quad_sum(l_run[r]);
    store_rows<NO, true>(o, p.out, p.ldo, c, p.n, p.d, inv_l, p.sv + hb * p.d);
  });
}

// ------------------------------------------------------------------ the pack
// One CTA per (head, tensor, clip): blockIdx.y 0 and 1 cast the head's q and k rows, 2 casts and transposes its v.
// q / k: 16 lanes per row, lane i < d / 8 holding columns 8i .. 8i + 7; the row's amax is a 16-lane shuffle max, and
// lanes d / 8 .. dp / 8 write the head's zero columns.
// v: the same lanes first take each channel's amax over the clip's tokens (col_amax: no atomics), then 64-token tiles
// are cast with the channel scales and transposed through shared memory.
constexpr int PK_THREADS = 256;

struct AttnPackParams {
  const __nv_bfloat16 *q, *k, *v;
  long ldq, ldk, ldv;
  int B, n, H, d, dp, n64;
  uint8_t *q8, *k8;
  long ld8;
  float *sq, *sk;
  uint8_t* vt8;
  long ldvt;
  float* sv;
};

__global__ void __launch_bounds__(PK_THREADS) attn_fp8_pack_kernel(const AttnPackParams p) {
  __shared__ unsigned red[PK_THREADS / 32][128];
  __shared__ float vscale[128];
  __shared__ Fp8TileT<128, ATT_COLS> tile;
  const int h = blockIdx.x, which = blockIdx.y, b = blockIdx.z;
  const int G = p.d / 8, l16 = threadIdx.x & 15, grp = threadIdx.x >> 4;
  const long hb = static_cast<long>(b) * p.H + h;
  const long row0 = static_cast<long>(b) * p.n;
  if (which < 2) {
    const __nv_bfloat16* src = (which == 0 ? p.q : p.k) + h * p.d + 8 * l16;
    const long ld = which == 0 ? p.ldq : p.ldk;
    uint8_t* dst = (which == 0 ? p.q8 : p.k8) + h * p.dp + 8 * l16;
    float* sinv_row = (which == 0 ? p.sq : p.sk) + hb * p.n64;
    for (int t = grp; t < p.n64; t += PK_THREADS / 16) {   // the same trip count for every lane (n64 % 16 == 0)
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (t < p.n && l16 < G) v = *reinterpret_cast<const uint4*>(src + (row0 + t) * ld);
      unsigned m = bf16_mag_max(v);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
      float scale, sinv;
      fp8_scale(m << 16, 8, scale, sinv);
      if (l16 == 0) sinv_row[t] = t < p.n ? sinv : 0.0f;
      if (t < p.n && l16 < p.dp / 8) {
        float f[8];
        unpack8(v, f);   // zeros past d
        *reinterpret_cast<uint2*>(dst + (row0 + t) * p.ld8) = cvt_e4m3x8(f, scale);
      }
    }
    return;
  }
  const __nv_bfloat16* src = p.v + h * p.d;
  unsigned m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
  if (l16 < G) {
    for (int t = grp; t < p.n; t += PK_THREADS / 16)
      bf16_mag_cols(*reinterpret_cast<const uint4*>(src + (row0 + t) * p.ldv + 8 * l16), m);
  }
  const unsigned mx = col_amax<16, PK_THREADS>(m, red);
  if (threadIdx.x < p.d) {
    float sinv;
    fp8_scale(mx << 16, 8, vscale[threadIdx.x], sinv);
    p.sv[hb * p.d + threadIdx.x] = sinv;
  }
  __syncthreads();
  const int n16 = static_cast<int>(round16(p.n));
  uint8_t* vt = p.vt8 + hb * p.d * p.ldvt;
  for (int t0 = 0; t0 < n16; t0 += ATT_COLS) {
    for (int i = threadIdx.x; i < ATT_COLS * G; i += PK_THREADS) {
      const int tt = i / G, c8 = i % G, t = t0 + tt;   // keys n .. n16 are zeros
      tile.put(8 * c8, tt, t < p.n ? *reinterpret_cast<const uint4*>(src + (row0 + t) * p.ldv + 8 * c8)
                                   : make_uint4(0u, 0u, 0u, 0u), vscale + 8 * c8);
    }
    __syncthreads();
    const int tn = min(ATT_COLS, n16 - t0);   // a multiple of 16
    for (int i = threadIdx.x; i < p.d * (ATT_COLS / 16); i += PK_THREADS) {
      const int row = i / (ATT_COLS / 16), q16 = (i % (ATT_COLS / 16)) * 16;
      tile.store<16>(row, q16, vt + row * p.ldvt + t0 + q16, tn - q16);
    }
    __syncthreads();
  }
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_attn_fp8_scale_pitch(int n) { return fp8_scale_pitch(n); }

extern "C" int ivb_attn_fp8_pack(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, int B, int n,
                                 int H, int d, void* q8, void* k8, long ld8, float* q_scale_inv, float* k_scale_inv,
                                 void* vt8, long ldvt, float* v_scale_inv, void* stream) {
  const char* fn = "ivb_attn_fp8_pack";
  if (B <= 0 || n <= 0) return 0;
  if (int rc = check_head_args(fn, d, {ldq, ldk, ldv})) return rc;
  if (q == nullptr || k == nullptr || v == nullptr || q8 == nullptr || k8 == nullptr || vt8 == nullptr ||
      q_scale_inv == nullptr || k_scale_inv == nullptr || v_scale_inv == nullptr)
    return set_error("ivb_attn_fp8_pack: an operand is null");
  if ((ld8 & 15) || ld8 < static_cast<long>(H) * head_pitch(d))
    return set_error("ivb_attn_fp8_pack: ld8 must be a multiple of 16 and >= H*round_up(d, 32)");
  if ((ldvt & 15) || ldvt < round16(n))
    return set_error("ivb_attn_fp8_pack: ldvt must be a multiple of 16 and >= round_up(n, 16)");
  if (misaligned(16, q, k, v, q8, k8, vt8)) return set_error("ivb_attn_fp8_pack: q, k, v, q8, k8 and vt8 must be 16-byte aligned");
  if (misaligned(16, q_scale_inv, k_scale_inv) || misaligned(4, v_scale_inv))
    return set_error("ivb_attn_fp8_pack: q_scale_inv and k_scale_inv must be 16-byte aligned, v_scale_inv 4-byte");
  const AttnPackParams pp{reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k),
                          reinterpret_cast<const __nv_bfloat16*>(v), ldq, ldk, ldv, B, n, H, d,
                          head_pitch(d), fp8_scale_pitch(n),
                          reinterpret_cast<uint8_t*>(q8), reinterpret_cast<uint8_t*>(k8), ld8, q_scale_inv, k_scale_inv,
                          reinterpret_cast<uint8_t*>(vt8), ldvt, v_scale_inv};
  return launch("attn_fp8_pack_kernel", attn_fp8_pack_kernel, dim3(H, 3, B), PK_THREADS, 0,
                reinterpret_cast<cudaStream_t>(stream), NO_PDL, pp);
}

extern "C" int ivb_attn_fwd_fp8(const void* q8, const void* k8, long ld8, const float* q_scale_inv,
                                const float* k_scale_inv, const void* vt8, long ldvt, const float* v_scale_inv, void* out,
                                long ldo, int B, int n, int H, int d, float softmax_scale, void* stream) {
  const char* fn = "ivb_attn_fwd_fp8";
  if (B <= 0 || n <= 0) return 0;
  if (int rc = check_head_args(fn, d, {ldo})) return rc;
  if (q8 == nullptr || k8 == nullptr || vt8 == nullptr || out == nullptr || q_scale_inv == nullptr ||
      k_scale_inv == nullptr || v_scale_inv == nullptr)
    return set_error("ivb_attn_fwd_fp8: an operand is null");
  if ((ld8 & 15) || ld8 < static_cast<long>(H) * head_pitch(d))
    return set_error("ivb_attn_fwd_fp8: ld8 must be a multiple of 16 and >= H*round_up(d, 32)");
  if ((ldvt & 15) || ldvt < round16(n))
    return set_error("ivb_attn_fwd_fp8: ldvt must be a multiple of 16 and >= round_up(n, 16)");
  if (misaligned(16, q8, k8, vt8, q_scale_inv, k_scale_inv))
    return set_error("ivb_attn_fwd_fp8: q8, k8, vt8, q_scale_inv and k_scale_inv must be 16-byte aligned");
  if (misaligned(8, v_scale_inv) || misaligned(4, out))
    return set_error("ivb_attn_fwd_fp8: v_scale_inv must be 8-byte aligned, out 4-byte");
  int rc;
  CUtensorMap tq, tk, tv;
  const int dp = head_pitch(d);
  if ((rc = make_head_tmap<AttnElt::E4M3>(&tq, q8, ld8, B, n, H, dp, ATT_ROWS))) return rc;
  if ((rc = make_head_tmap<AttnElt::E4M3>(&tk, k8, ld8, B, n, H, dp, ATT_COLS))) return rc;
  const AttnFp8Params p{B, n, H, d, dp, fp8_scale_pitch(n), softmax_scale * 1.4426950408889634f, q_scale_inv, k_scale_inv,
                        v_scale_inv, reinterpret_cast<__nv_bfloat16*>(out), ldo};
  return dispatch_head_dim(d, [&](auto hd) {
    // V^T of (clip, head) as (key, channel, head, clip): keys past round_up(n, 16) and channels past d load as zeros
    const uint64_t dims[4] = {static_cast<uint64_t>(round16(n)), static_cast<uint64_t>(d), static_cast<uint64_t>(H),
                              static_cast<uint64_t>(B)};
    const long strides[3] = {ldvt, static_cast<long>(d) * ldvt, static_cast<long>(H) * d * ldvt};
    const uint32_t box[4] = {ATT_COLS, static_cast<uint32_t>(hd.NO), 1, 1};
    if (int rc2 = make_tmap_4d(&tv, vt8, dims, strides, box, 1, 64)) return rc2;
    return launch_attn<attn_fwd_fp8_kernel<hd.NO>, NO_PDL>("cudaFuncSetAttribute(attn_fwd_fp8)", "attn_fwd_fp8_kernel",
                                                          Fp8Smem::BYTES, B, n, H, reinterpret_cast<cudaStream_t>(stream),
                                                          tq, tk, tv, p);
  });
}
