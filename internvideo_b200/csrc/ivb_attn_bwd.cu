// ivb_attn_bwd.cu — attention backward on Hopper wgmma (two passes, no atomics, recompute of P from lse).
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
// Warp roles (384 threads): warpgroup 0 = the TMA producer (one elected thread), warpgroups 1 and 2 own 64 of the
// 128 rows each.  mbarriers only:
//   bar_row     TMA -> MMA        X,Y (the 128 owned rows) landed
//   full[s]     TMA -> MMA        streamed tiles U_j, W_j of stage s landed (tx)
//   empty[s]    MMA -> TMA        both warpgroups retired every MMA that reads stage s
#include <math.h>
#include <stdlib.h>

#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

int make_head_tmap(CUtensorMap* tm, const void* base, long ld, int B, int n, int H, int d,
                   int box_tokens);

constexpr int BWD_ROWS = 128;  // rows owned by the CTA (two warpgroups of 64)
constexpr int BWD_COLS = 64;   // streamed tile

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

constexpr int BWD_NST = 2;  // streamed-tile stages

// KA: 64-wide atoms covering head_dim (1: d <= 64, 2: d <= 128); NO: wgmma N of the accumulate MMAs.
template <int MODE, int KA, int NO>
__global__ void __launch_bounds__(384, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmW,
                const AttnBwdParams p) {
  constexpr int ROW_BYTES = KA * BWD_ROWS * 128;   // one owned-row operand
  constexpr int COL_BYTES = KA * BWD_COLS * 128;   // one streamed tile
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sX = smem;
  uint8_t* sY = sX + ROW_BYTES;
  uint8_t* sU = sY + ROW_BYTES;                 // BWD_NST stages
  uint8_t* sW = sU + BWD_NST * COL_BYTES;       // BWD_NST stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sW + BWD_NST * COL_BYTES);
  uint64_t* bar_row = bars;
  uint64_t* full = bars + 1;
  uint64_t* empty = full + BWD_NST;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = tid >> 7;
  const int r0 = blockIdx.x * BWD_ROWS;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int nblk = (p.n + BWD_COLS - 1) / BWD_COLS;
  const int ksteps = (p.d + 15) / 16;

  if (tid == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();
    mbar_init(bar_row, 1);
    for (int i = 0; i < BWD_NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (wg == 0) {
    setmaxnreg_dec<24>();
    // ===================== TMA producer =====================
    if (warp == 0 && elect_one()) {
      tma_prefetch_desc(&tmX); tma_prefetch_desc(&tmY); tma_prefetch_desc(&tmU); tma_prefetch_desc(&tmW);
      mbar_expect_tx(bar_row, 2 * ROW_BYTES);
#pragma unroll
      for (int a = 0; a < KA; ++a) {
        tma_load_4d(sX + a * (BWD_ROWS * 128), &tmX, a * 64, h, r0, b, bar_row);
        tma_load_4d(sY + a * (BWD_ROWS * 128), &tmY, a * 64, h, r0, b, bar_row);
      }
      for (int j = 0; j < nblk; ++j) {
        const int st = j % BWD_NST;
        mbar_wait(&empty[st], ((j / BWD_NST) & 1) ^ 1);
        mbar_expect_tx(&full[st], 2 * COL_BYTES);
#pragma unroll
        for (int a = 0; a < KA; ++a) {
          tma_load_4d(sU + st * COL_BYTES + a * (BWD_COLS * 128), &tmU, a * 64, h, j * BWD_COLS, b, &full[st]);
          tma_load_4d(sW + st * COL_BYTES + a * (BWD_COLS * 128), &tmW, a * 64, h, j * BWD_COLS, b, &full[st]);
        }
      }
    }
  } else {
    setmaxnreg_inc<240>();
    // ===================== MMA + math warpgroups =====================
    const int cw = wg - 1;
    const bool signal = (tid & 127) == 0;
    const int rloc = cw * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows: rloc, rloc + 8
    const uint32_t xa = smem_u32(sX) + cw * 8192, ya = smem_u32(sY) + cw * 8192;
    const long hb = (static_cast<long>(b) * p.H + h) * p.n_pad;
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
        const int q = r0 + rloc + 8 * r;
        if (q < p.n_pad) { row_lse[r] = p.lse2p[hb + q]; row_delta[r] = p.deltap[hb + q]; }
      }
    }

    mbar_wait(bar_row, 0);
    for (int j = 0; j < nblk; ++j) {
      const int st = j % BWD_NST;
      mbar_wait(&full[st], (j / BWD_NST) & 1);
      const uint32_t ua = smem_u32(sU + st * COL_BYTES), wa = smem_u32(sW + st * COL_BYTES);
      float sc[BWD_COLS / 2], dp[BWD_COLS / 2];
      wgmma_fence();
      for (int kk = 0; kk < ksteps; ++kk) {
        const uint32_t off = (kk & 3) * 32;
        const uint32_t ro = (kk >> 2) * (BWD_ROWS * 128) + off, co = (kk >> 2) * (BWD_COLS * 128) + off;
        Wgmma<BWD_COLS>::ss<0, 0>(sc, gmma_desc(xa + ro, 16, 1024), gmma_desc(ua + co, 16, 1024), kk > 0 ? 1u : 0u);
        Wgmma<BWD_COLS>::ss<0, 0>(dp, gmma_desc(ya + ro, 16, 1024), gmma_desc(wa + co, 16, 1024), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(sc, BWD_COLS / 2);
      wgmma_reg_fence(dp, BWD_COLS / 2);

      // P and dS in place of S and dP.  Columns beyond the sequence get P = 0.
#pragma unroll
      for (int i = 0; i < BWD_COLS / 2; ++i) {
        const int col = j * BWD_COLS + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        float lse, dl;
        if (MODE == 1) { lse = p.lse2p[hb + col]; dl = p.deltap[hb + col]; }
        else { lse = row_lse[(i >> 1) & 1]; dl = row_delta[(i >> 1) & 1]; }
        const float pv = col < p.n ? exp2f(fmaf(sc[i], p.sc_log2, -lse)) : 0.f;
        sc[i] = pv;
        dp[i] = pv * (dp[i] - dl) * p.scale;
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BWD_COLS / 16; ++kk) {
        uint32_t fa[4];
        if (MODE == 1) {
          acc_to_a_frag(sc, kk, fa);
          Wgmma<NO>::rs<1>(acc1, fa, gmma_desc(wa + kk * 2048, BWD_COLS * 128, 1024), 1u);   // dV += P^T dO
          acc_to_a_frag(dp, kk, fa);
          Wgmma<NO>::rs<1>(acc2, fa, gmma_desc(ua + kk * 2048, BWD_COLS * 128, 1024), 1u);   // dK += dS^T Q
        } else {
          acc_to_a_frag(dp, kk, fa);
          Wgmma<NO>::rs<1>(acc1, fa, gmma_desc(ua + kk * 2048, BWD_COLS * 128, 1024), 1u);   // dQ += dS K
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(acc1, NO / 2);
      if (MODE == 1) wgmma_reg_fence(acc2, NO / 2);
      if (signal) mbar_arrive(&empty[st]);
    }

#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r0 + rloc + 8 * r;
      if (row >= p.n) continue;
      __nv_bfloat16* o1 = p.out1 + (static_cast<long>(b) * p.n + row) * p.ld1 + h * p.d;
      __nv_bfloat16* o2 = MODE == 1 ? p.out2 + (static_cast<long>(b) * p.n + row) * p.ld2 + h * p.d : nullptr;
#pragma unroll
      for (int jn = 0; jn < NO / 8; ++jn) {
        const int c = 8 * jn + 2 * (lane & 3);
        if (c < p.d) {
          *reinterpret_cast<uint32_t*>(o1 + c) = pack_bf16(acc1[4 * jn + 2 * r], acc1[4 * jn + 2 * r + 1]);
          if (MODE == 1)
            *reinterpret_cast<uint32_t*>(o2 + c) = pack_bf16(acc2[4 * jn + 2 * r], acc2[4 * jn + 2 * r + 1]);
        }
      }
    }
  }
}

template <int MODE, int KA, int NO>
static int launch_attn_bwd(const CUtensorMap& tx, const CUtensorMap& ty, const CUtensorMap& tu,
                           const CUtensorMap& tw, const AttnBwdParams& p, cudaStream_t stream) {
  constexpr int SMEM = 2 * KA * BWD_ROWS * 128 + 2 * BWD_NST * KA * BWD_COLS * 128 + 128;
  static_assert(SMEM <= 227 * 1024, "attention backward: shared-memory budget");
  auto kern = attn_bwd_kernel<MODE, KA, NO>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(attn_bwd)", e);
  }
  dim3 grid((p.n + BWD_ROWS - 1) / BWD_ROWS, p.H, p.B);
  cudaError_t le = launch_pdl(kern, grid, dim3(384), SMEM, stream, tx, ty, tu, tw, p);
  if (le != cudaSuccess) return set_error_cuda("launch(attn_bwd_kernel)", le);
  count_launch();
  return check_launch("attn_bwd_kernel");
}

template <int MODE>
static int dispatch_bwd(int d, const CUtensorMap& tx, const CUtensorMap& ty, const CUtensorMap& tu,
                        const CUtensorMap& tw, const AttnBwdParams& p, cudaStream_t stream) {
  const int no = (d + 31) / 32 * 32;
  if (d <= 64) {
    if (no <= 32) return launch_attn_bwd<MODE, 1, 32>(tx, ty, tu, tw, p, stream);
    return launch_attn_bwd<MODE, 1, 64>(tx, ty, tu, tw, p, stream);
  }
  if (no <= 96) return launch_attn_bwd<MODE, 2, 96>(tx, ty, tu, tw, p, stream);
  return launch_attn_bwd<MODE, 2, 128>(tx, ty, tu, tw, p, stream);
}

}  // namespace ivb

using namespace ivb;

// workspace (floats) needed by ivb_attn_bwd: padded lse2 + delta, [2][B][H][round_up(n,64)]
extern "C" long ivb_attn_bwd_workspace_floats(int B, int n, int H) {
  const long n_pad = (static_cast<long>(n) + BWD_COLS - 1) / BWD_COLS * BWD_COLS;
  return 2 * static_cast<long>(B) * H * n_pad;
}

extern "C" int ivb_attn_bwd(const void* q, long ldq, const void* k, long ldk, const void* v,
                            long ldv, const void* out, long ldo, const void* dout, long lddo,
                            const float* lse2, float* delta_ws, void* dq, long lddq, void* dk,
                            long lddk, void* dv, long lddv, int B, int n, int H, int d,
                            float softmax_scale, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || n <= 0) return 0;
  if (d % 8 != 0 || d > 128 || d < 16) return set_error("ivb_attn_bwd: head_dim must be a multiple of 8 in [16,128]");
  if ((ldq & 7) || (ldk & 7) || (ldv & 7) || (ldo & 7) || (lddo & 7) || (lddq & 7) || (lddk & 7) || (lddv & 7))
    return set_error("ivb_attn_bwd: pitches must be multiples of 8");
  if (lse2 == nullptr || delta_ws == nullptr) return set_error("ivb_attn_bwd: lse2 and the workspace are required");
  if ((reinterpret_cast<uintptr_t>(delta_ws) & 15) != 0) return set_error("ivb_attn_bwd: workspace must be 16-byte aligned");
  const int n_pad = (n + BWD_COLS - 1) / BWD_COLS * BWD_COLS;
  const long half = static_cast<long>(B) * H * n_pad;
  float* lse2p = delta_ws;
  float* deltap = delta_ws + half;
  {
    cudaError_t e = cudaMemsetAsync(delta_ws, 0, 2 * half * sizeof(float), stream);   // zero padding (0 * pad must stay 0)
    if (e != cudaSuccess) return set_error_cuda("cudaMemsetAsync(attn_bwd workspace)", e);
    const long total = static_cast<long>(B) * n * H;
    const int threads = 128;
    attn_bwd_prep_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(out), ldo, reinterpret_cast<const __nv_bfloat16*>(dout),
        lddo, lse2, lse2p, deltap, B, n, n_pad, H, d);
    count_launch();
    int rc = check_launch("attn_bwd_prep_kernel");
    if (rc) return rc;
  }
  CUtensorMap tq128, tdo128, tk128, tv128, tq64, tdo64, tk64, tv64;
  int rc;
  if ((rc = make_head_tmap(&tq128, q, ldq, B, n, H, d, BWD_ROWS))) return rc;
  if ((rc = make_head_tmap(&tdo128, dout, lddo, B, n, H, d, BWD_ROWS))) return rc;
  if ((rc = make_head_tmap(&tk128, k, ldk, B, n, H, d, BWD_ROWS))) return rc;
  if ((rc = make_head_tmap(&tv128, v, ldv, B, n, H, d, BWD_ROWS))) return rc;
  if ((rc = make_head_tmap(&tq64, q, ldq, B, n, H, d, BWD_COLS))) return rc;
  if ((rc = make_head_tmap(&tdo64, dout, lddo, B, n, H, d, BWD_COLS))) return rc;
  if ((rc = make_head_tmap(&tk64, k, ldk, B, n, H, d, BWD_COLS))) return rc;
  if ((rc = make_head_tmap(&tv64, v, ldv, B, n, H, d, BWD_COLS))) return rc;
  AttnBwdParams p;
  p.B = B; p.n = n; p.H = H; p.d = d; p.n_pad = n_pad;
  p.scale = softmax_scale;
  p.sc_log2 = softmax_scale * 1.4426950408889634f;
  p.lse2p = lse2p; p.deltap = deltap;
  // dK, dV
  p.out1 = reinterpret_cast<__nv_bfloat16*>(dv); p.ld1 = lddv;
  p.out2 = reinterpret_cast<__nv_bfloat16*>(dk); p.ld2 = lddk;
  if ((rc = dispatch_bwd<1>(d, tk128, tv128, tq64, tdo64, p, stream))) return rc;
  // dQ
  p.out1 = reinterpret_cast<__nv_bfloat16*>(dq); p.ld1 = lddq;
  p.out2 = nullptr; p.ld2 = 0;
  return dispatch_bwd<0>(d, tq128, tdo128, tk64, tv64, p, stream);
}
