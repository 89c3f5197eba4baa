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
// The forward is attn_fwd<AttnElt::E4M3> of ivb_attn_fwd.cuh, the body of the bf16 forward with E4M3 tiles, k32
// wgmmas and a three-stage ring:
//   S_ij = (sq_i scale log2e) sk_j (q8_i . k8_j)   the row factors are loaded once per thread; the 64 column factors of
//                                                   a K tile land in its ring stage under the tile's `full` barrier
//   P    = exp2(S - m + 8)                         the bf16 kernel's online softmax with P scaled by 2^8 (P <= 256 < 448,
//                                                   and small probabilities stay in E4M3's normal range), cast to E4M3
//                                                   and permuted into the k32 A layout in registers
//   O    = (sum P8 V8) sv_c / l                    sv and 1/l are column and row factors of the bf16 store; l sums the
//                                                   same 2^8-scaled P, so the factor cancels
#include <math.h>
#include <stdlib.h>

#include "ivb_attn_fwd.cuh"
#include "ivb_fp8.cuh"
#include "ivb_rows.cuh"

namespace ivb {

// Pitch of the per-(clip, head) q and k scale rows: whole 64-key tiles, so a tile's column scales are one 256-byte
// aligned bulk copy.
__host__ __device__ inline int fp8_scale_pitch(int n) { return (n + ATT_COLS - 1) / ATT_COLS * ATT_COLS; }
__host__ __device__ inline long round16(long n) { return (n + 15) / 16 * 16; }
__host__ __device__ inline int head_pitch(int d) { return (d + 31) / 32 * 32; }

// NO: the head dim rounded up to 32, the N of O += P V; NO / 32 k32 steps of S = Q K^T.
template <int NO>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_fp8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnFp8Params p) {
  attn_fwd<AttnElt::E4M3, 1, NO, NO / 32>(tmQ, tmK, tmV, p);
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
