// ivb_fp8.cu — per-tensor current-scaling FP8 quantisation of bf16 tensors (the operands of ivb_gemm_fp8).
//
//   amax      = max |x| over the [M, K] tensor (an integer atomicMax on the float bits: order-independent, so
//               every run gives the same bits)
//   scale     = 2^floor(log2(fmax / amax)),  fmax = 448 (E4M3) or 57 344 (E5M2);  amax = 0 gives 1
//   out       = round_rn(x * scale)  (cvt.rn.satfinite), out_t = out^T (optional), scale_inv = 1 / scale
//
// A power-of-two scale makes x * scale and the dequantisation exact in fp32, and amax * scale <= fmax means the
// cast never saturates.  A non-finite amax writes scale_inv = NaN: satfinite alone would clamp an Inf to fmax and
// hide the overflow, while NaN reaches the GEMM output and the training step's finiteness check.
//
// ivb_fp8_quantize_rows applies the same rule to each row on its own (E4M3 only): a row's scale comes from the row's
// amax, so a row's grid is never coarser than the whole tensor's, and the cast error of an element never larger.
//
// ivb_fp8_quantize_cols_t applies it to each column of a weight and writes the transposed copy (the input-gradient
// GEMM's B operand, one scale per input channel): a column amax (integer atomicMax, order-independent), then the
// cast kernel's 64 x 64 transposing tile with one scale per column.
//
// ivb_fp8_quantize_blocks_t applies it to each column of each 128-row block of activations or gradients [tokens, C]
// and writes the transposed copy (the K-major operands of the FP8 weight gradient over tokens): one kernel, one read.
#include <cstdio>

#include "ivb_fp8.cuh"
#include "ivb_internal.h"
#include "ivb_rows.cuh"

namespace ivb {

constexpr int Q_TILE = 64;         // the cast kernel's tile: 64 rows x 64 columns, 16 elements per thread
constexpr int Q_THREADS = 256;
constexpr int Q_PITCH = Q_TILE + 16;   // bytes per row of the transposing tile (16-byte aligned rows)

__global__ void __launch_bounds__(256) fp8_amax_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M, int K,
                                                       unsigned* amax_bits) {
  pdl_wait();
  pdl_launch_dependents();
  const long kc = (K + 7) / 8;
  const long chunks = static_cast<long>(M) * kc;
  unsigned m = 0;   // bf16 magnitude bits: NaN > Inf > every finite value
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < chunks;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long row = i / kc;
    const int c = static_cast<int>(i % kc) * 8;
    const __nv_bfloat16* src = x + row * ldx + c;
    if (c + 8 <= K) {
      const uint4 v = *reinterpret_cast<const uint4*>(src);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) m = max(m, max(w[k] & 0x7fffu, (w[k] >> 16) & 0x7fffu));
    } else {
      const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src);
      for (int k = 0; k < K - c; ++k) m = max(m, static_cast<unsigned>(s16[k]) & 0x7fffu);
    }
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(amax_bits, m << 16);
}

// One 64 x 64 tile per CTA: thread t converts 16 elements of row t / 4 and writes them to `out`; with out_t, the tile
// is transposed through shared memory and thread t writes 16 elements of row t / 4 of out_t's tile.
// COLS (E4M3 only): one scale per column, from amax_bits[K] and written to scale_inv[K]; only out_t is written.
template <bool E5M2, bool COLS>
__device__ __forceinline__ void fp8_cast_tile(const __nv_bfloat16* __restrict__ x, long ldx, int M, int K,
                                              const unsigned* amax_bits, uint8_t* out, long ldo, uint8_t* out_t,
                                              long ldt, float* scale_inv) {
  __shared__ __align__(16) uint8_t tile[Q_TILE * Q_PITCH];
  float scale, sinv;
  if constexpr (!COLS) {
    fp8_scale(*amax_bits, E5M2 ? 15 : 8, scale, sinv);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv = sinv;
  }
  const int m0 = blockIdx.y * Q_TILE, k0 = blockIdx.x * Q_TILE;
  const int r = threadIdx.x >> 2, c = (threadIdx.x & 3) * 16;
  const int row = m0 + r, col = k0 + c;
  const int nv = row < M ? min(16, K - col) : 0;   // elements of this thread's segment inside the tensor
  float v[16];
  if (nv == 16) {
    const uint4* src = reinterpret_cast<const uint4*>(x + static_cast<long>(row) * ldx + col);
    const uint4 a = src[0], b = src[1];
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) { const float2 f = unpack_bf16(w[k]); v[2 * k] = f.x; v[2 * k + 1] = f.y; }
  } else {
#pragma unroll
    for (int k = 0; k < 16; ++k)
      v[k] = k < nv ? __bfloat162float(x[static_cast<long>(row) * ldx + col + k]) : 0.0f;
  }
  uint32_t q[4];
  if constexpr (COLS) {
    const int nc = min(16, K - col);   // columns of this thread's segment inside the tensor
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      fp8_scale(k < nc ? amax_bits[col + k] : 0u, 8, scale, sinv);
      v[k] *= scale;
      if (blockIdx.y == 0 && r == 0 && k < nc) scale_inv[col + k] = sinv;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      q[k] = cvt_fp8x2<false>(v[4 * k], v[4 * k + 1]) | (cvt_fp8x2<false>(v[4 * k + 2], v[4 * k + 3]) << 16);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      q[k] = cvt_fp8x2<E5M2>(v[4 * k] * scale, v[4 * k + 1] * scale) |
             (cvt_fp8x2<E5M2>(v[4 * k + 2] * scale, v[4 * k + 3] * scale) << 16);
    uint8_t* dst = out + static_cast<long>(row) * ldo + col;
    if (nv == 16) {
      *reinterpret_cast<uint4*>(dst) = make_uint4(q[0], q[1], q[2], q[3]);
    } else {
      for (int k = 0; k < nv; ++k) dst[k] = static_cast<uint8_t>(q[k >> 2] >> (8 * (k & 3)));
    }
    if (out_t == nullptr) return;
  }
#pragma unroll
  for (int k = 0; k < 16; ++k) tile[(c + k) * Q_PITCH + r] = static_cast<uint8_t>(q[k >> 2] >> (8 * (k & 3)));
  __syncthreads();
  // out_t row k0 + r holds column k0 + r of the tile: tensor rows m0 + c .. m0 + c + 15
  const int trow = k0 + r, tcol = m0 + c;
  const int tn = trow < K ? min(16, M - tcol) : 0;
  if (tn <= 0) return;
  const uint4 t = *reinterpret_cast<const uint4*>(tile + r * Q_PITCH + c);
  uint8_t* tdst = out_t + static_cast<long>(trow) * ldt + tcol;
  if (tn == 16) {
    *reinterpret_cast<uint4*>(tdst) = t;
  } else {
    const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
    for (int k = 0; k < tn; ++k) tdst[k] = static_cast<uint8_t>(tw[k >> 2] >> (8 * (k & 3)));
  }
}

template <bool E5M2>
__global__ void __launch_bounds__(Q_THREADS) fp8_cast_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                             int K, const unsigned* amax_bits, uint8_t* out, long ldo,
                                                             uint8_t* out_t, long ldt, float* scale_inv) {
  pdl_wait();
  pdl_launch_dependents();
  fp8_cast_tile<E5M2, false>(x, ldx, M, K, amax_bits, out, ldo, out_t, ldt, scale_inv);
}

// ------------------------------------------------------------------ per-column scaling (ivb_fp8_quantize_cols_t)
// The column amax of a 64-column strip over Q_COL_ROWS rows per CTA: thread t reads the 8-column chunk t % 8 of rows
// t / 8, t / 8 + 32, ...; the 32 row lanes of a chunk are reduced by shuffles and shared memory, then one integer
// atomicMax per column (order-independent: the same bits on every run).
constexpr int Q_COL_ROWS = 256;

__global__ void __launch_bounds__(Q_THREADS) fp8_col_amax_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                                 int K, unsigned* col_amax_bits) {
  __shared__ unsigned red[Q_THREADS / 32][Q_TILE];
  pdl_wait();
  pdl_launch_dependents();
  const int c = blockIdx.x * Q_TILE + (threadIdx.x & 7) * 8;
  const int r1 = min(M, (blockIdx.y + 1) * Q_COL_ROWS);
  unsigned m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};   // bf16 magnitude bits: NaN > Inf > every finite value
  if (c < K) {
    for (int row = blockIdx.y * Q_COL_ROWS + (threadIdx.x >> 3); row < r1; row += Q_THREADS / 8) {
      const __nv_bfloat16* src = x + static_cast<long>(row) * ldx + c;
      if (c + 8 <= K) {
        const uint4 v = *reinterpret_cast<const uint4*>(src);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          m[2 * k] = max(m[2 * k], w[k] & 0x7fffu);
          m[2 * k + 1] = max(m[2 * k + 1], (w[k] >> 16) & 0x7fffu);
        }
      } else {
        const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src);
        for (int k = 0; k < K - c; ++k) m[k] = max(m[k], static_cast<unsigned>(s16[k]) & 0x7fffu);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {   // lanes l, l ^ 8, l ^ 16, l ^ 24 hold the same chunk
    m[k] = max(m[k], __shfl_xor_sync(0xffffffffu, m[k], 8));
    m[k] = max(m[k], __shfl_xor_sync(0xffffffffu, m[k], 16));
  }
  const int lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) red[threadIdx.x >> 5][lane * 8 + k] = m[k];
  }
  __syncthreads();
  if (threadIdx.x < Q_TILE) {
    unsigned mx = 0;
#pragma unroll
    for (int w = 0; w < Q_THREADS / 32; ++w) mx = max(mx, red[w][threadIdx.x]);
    const int col = blockIdx.x * Q_TILE + threadIdx.x;
    if (col < K && mx != 0) atomicMax(col_amax_bits + col, mx << 16);
  }
}

__global__ void __launch_bounds__(Q_THREADS) fp8_cast_cols_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                                  int K, const unsigned* col_amax_bits, uint8_t* out_t,
                                                                  long ldt, float* col_scale_inv) {
  pdl_wait();
  pdl_launch_dependents();
  fp8_cast_tile<false, true>(x, ldx, M, K, col_amax_bits, nullptr, 0, out_t, ldt, col_scale_inv);
}

// ------------------------------------------------------------------ per-row scaling (ivb_fp8_quantize_rows)
// One CTA per row: thread t holds the row's 8-element chunks t, t + 128, ... in registers (NV of them, packed bf16),
// so the row is read from HBM once; the row's amax is a max over integer magnitude bits (no atomics, the same bits on
// every run), then each chunk is scaled, cast and stored.
constexpr int R_THREADS = 128;

template <int NV>
__global__ void __launch_bounds__(R_THREADS) fp8_rows_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int K,
                                                            uint8_t* __restrict__ out, long ldo,
                                                            float* __restrict__ scale_inv) {
  __shared__ unsigned red[R_THREADS / 32];
  pdl_wait();
  pdl_launch_dependents();
  const long row = blockIdx.x;
  const __nv_bfloat16* src = x + row * ldx;
  uint4 v[NV];
  unsigned m = 0;   // bf16 magnitude bits: NaN > Inf > every finite value
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (threadIdx.x + R_THREADS * i) * 8;
    v[i] = make_uint4(0u, 0u, 0u, 0u);
    if (c + 8 <= K) {
      v[i] = *reinterpret_cast<const uint4*>(src + c);
    } else if (c < K) {   // the row's last, partial chunk: no read past element K - 1
      const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src + c);
      uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (c + k < K) w[k >> 1] |= static_cast<uint32_t>(s16[k]) << (16 * (k & 1));
      v[i] = make_uint4(w[0], w[1], w[2], w[3]);
    }
    const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
    for (int k = 0; k < 4; ++k) m = max(m, max(w[k] & 0x7fffu, (w[k] >> 16) & 0x7fffu));
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < R_THREADS / 32; ++w) m = max(m, red[w]);
  float scale, sinv;
  fp8_scale(m << 16, 8, scale, sinv);
  if (threadIdx.x == 0) scale_inv[row] = sinv;
  uint8_t* dst = out + row * ldo;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (threadIdx.x + R_THREADS * i) * 8;
    if (c >= K) continue;
    float f[8];
    unpack8(v[i], f);
    const uint2 q = cvt_e4m3x8(f, scale);
    if (c + 8 <= K) {
      *reinterpret_cast<uint2*>(dst + c) = q;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (c + k < K) dst[c + k] = static_cast<uint8_t>((k < 4 ? q.x : q.y) >> (8 * (k & 3)));
    }
  }
}

// ------------------------------------------------------------------ per-(128-token block, channel) scaling
// (ivb_fp8_quantize_blocks_t: the operands of the FP8 weight gradient, ivb_gemm_fp8_wgrad)
// One CTA per 128 tokens x 64 channels: thread t reads the 8-channel chunk t % 8 of tokens t / 8, t / 8 + 32, ...
// into registers (x is read once), the column amax goes through shuffles and shared memory (no atomics: the same bits
// on every run), then each element is scaled by its column's factor, cast and transposed through shared memory, and
// thread t writes 32 tokens of channel t / 4.  rowscale (optional): tokens whose factor is 0 are cast as zeros.
constexpr int B_TOK = 128, B_CH = 64;
constexpr int B_PITCH = B_TOK + 16;    // bytes per channel row of the transposing tile (16-byte aligned rows)

__global__ void __launch_bounds__(Q_THREADS) fp8_blocks_t_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                                 int C, const float* __restrict__ rowscale,
                                                                 uint8_t* __restrict__ out_t, long ldt,
                                                                 float* __restrict__ scale_inv) {
  __shared__ unsigned red[Q_THREADS / 32][B_CH];
  __shared__ __align__(16) uint8_t tile[B_CH * B_PITCH];
  pdl_wait();
  pdl_launch_dependents();
  const int m0 = blockIdx.y * B_TOK, c0 = blockIdx.x * B_CH;
  const int cc = (threadIdx.x & 7) * 8, r0 = threadIdx.x >> 3;   // chunk column in the strip, first token
  const int col = c0 + cc;
  uint4 v[B_TOK / 32];
  unsigned m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};   // bf16 magnitude bits: NaN > Inf > every finite value
#pragma unroll
  for (int i = 0; i < B_TOK / 32; ++i) {
    const int row = m0 + r0 + 32 * i;
    v[i] = make_uint4(0u, 0u, 0u, 0u);
    if (row < M && col < C && (rowscale == nullptr || rowscale[row] != 0.0f))
      v[i] = *reinterpret_cast<const uint4*>(x + static_cast<long>(row) * ldx + col);
    const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      m[2 * k] = max(m[2 * k], w[k] & 0x7fffu);
      m[2 * k + 1] = max(m[2 * k + 1], (w[k] >> 16) & 0x7fffu);
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {   // lanes l, l ^ 8, l ^ 16, l ^ 24 hold the same chunk
    m[k] = max(m[k], __shfl_xor_sync(0xffffffffu, m[k], 8));
    m[k] = max(m[k], __shfl_xor_sync(0xffffffffu, m[k], 16));
  }
  const int lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) red[threadIdx.x >> 5][lane * 8 + k] = m[k];
  }
  __syncthreads();
  float scale[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    unsigned mx = 0;
#pragma unroll
    for (int w = 0; w < Q_THREADS / 32; ++w) mx = max(mx, red[w][cc + k]);
    float sinv;
    fp8_scale(mx << 16, 8, scale[k], sinv);
    if (r0 == 0 && col < C) scale_inv[static_cast<long>(blockIdx.y) * C + col + k] = sinv;
  }
#pragma unroll
  for (int i = 0; i < B_TOK / 32; ++i) {
    float f[8];
    unpack8(v[i], f);
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
      const uint32_t q = cvt_fp8x2<false>(f[k] * scale[k], f[k + 1] * scale[k + 1]);
      tile[(cc + k) * B_PITCH + r0 + 32 * i] = static_cast<uint8_t>(q);
      tile[(cc + k + 1) * B_PITCH + r0 + 32 * i] = static_cast<uint8_t>(q >> 8);
    }
  }
  __syncthreads();
  // out_t row c0 + t / 4 holds channel c0 + t / 4: tokens m0 + 32 (t % 4) .. + 31
  const int trow = c0 + (threadIdx.x >> 2), tok = 32 * (threadIdx.x & 3);
  const int tn = trow < C ? min(32, M - m0 - tok) : 0;
  if (tn <= 0) return;
  const uint8_t* src = tile + (threadIdx.x >> 2) * B_PITCH + tok;
  uint8_t* dst = out_t + static_cast<long>(trow) * ldt + m0 + tok;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (tn >= 16 * (h + 1)) {
      reinterpret_cast<uint4*>(dst)[h] = reinterpret_cast<const uint4*>(src)[h];
    } else {
      for (int k = 16 * h; k < tn; ++k) dst[k] = src[k];
    }
  }
}

}  // namespace ivb

using namespace ivb;

// ivb_fp8_quantize_blocks_t and ivb_fp8_quantize_blocks_t_plan; `fn` names the entry point in messages.
static int quantize_blocks_t(const char* fn, const void* x, long ldx, int M, int C, void* out_t, long ldt,
                             float* scale_inv, const float* rowscale, cudaStream_t stream) {
  char msg[128];
  auto fail = [&](const char* what) {
    std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
    return set_error(msg);
  };
  if (M <= 0 || C <= 0) return fail("empty tensor");
  if (C & 7) return fail("C must be a multiple of 8");
  if (x == nullptr || out_t == nullptr || scale_inv == nullptr) return fail("x, out_t or scale_inv is null");
  if ((ldx & 7) || ldx < C) return fail("ldx must be a multiple of 8 elements and >= C");
  if ((ldt & 15) || ldt < M) return fail("ldt must be a multiple of 16 elements and >= M");
  if (misaligned(16, x, out_t)) return fail("x and out_t must be 16-byte aligned");
  if (misaligned(4, scale_inv, rowscale)) return fail("scale_inv and rowscale must be 4-byte aligned");
  const dim3 grid((C + B_CH - 1) / B_CH, (M + B_TOK - 1) / B_TOK);
  return launch("fp8_blocks_t_kernel", fp8_blocks_t_kernel, grid, Q_THREADS, 0, stream, ALLOW_PDL,
                reinterpret_cast<const __nv_bfloat16*>(x), ldx, M, C, rowscale, reinterpret_cast<uint8_t*>(out_t), ldt,
                scale_inv);
}

extern "C" int ivb_fp8_quantize_blocks_t(const void* x, long ldx, int M, int C, void* out_t, long ldt,
                                         float* scale_inv, void* stream) {
  return quantize_blocks_t("ivb_fp8_quantize_blocks_t", x, ldx, M, C, out_t, ldt, scale_inv, nullptr,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_fp8_quantize_blocks_t_plan(const void* x, long ldx, int M, int C, void* out_t, long ldt,
                                              float* scale_inv, const float* rowscale, void* stream) {
  if (rowscale == nullptr) return set_error("ivb_fp8_quantize_blocks_t_plan: rowscale is null");
  return quantize_blocks_t("ivb_fp8_quantize_blocks_t_plan", x, ldx, M, C, out_t, ldt, scale_inv, rowscale,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_fp8_quantize_rows(const void* x, long ldx, int M, int K, void* out, long ldo, float* row_scale_inv,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || K <= 0) return set_error("ivb_fp8_quantize_rows: empty tensor");
  if (K > IVB_FP8_ROWS_MAX_K) return set_error("ivb_fp8_quantize_rows: K > IVB_FP8_ROWS_MAX_K");
  if (x == nullptr || out == nullptr || row_scale_inv == nullptr)
    return set_error("ivb_fp8_quantize_rows: x, out or row_scale_inv is null");
  if ((ldx & 7) || ldx < K) return set_error("ivb_fp8_quantize_rows: ldx must be a multiple of 8 elements and >= K");
  if ((ldo & 15) || ldo < K) return set_error("ivb_fp8_quantize_rows: ldo must be a multiple of 16 elements and >= K");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15)
    return set_error("ivb_fp8_quantize_rows: x and out must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(row_scale_inv) & 3)
    return set_error("ivb_fp8_quantize_rows: row_scale_inv must be 4-byte aligned");
  const auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* o = reinterpret_cast<uint8_t*>(out);
  const int chunks = (K + 7) / 8;   // per row; each thread holds NV of them
  const auto kern = chunks <= R_THREADS * 2 ? fp8_rows_kernel<2>
                  : chunks <= R_THREADS * 4 ? fp8_rows_kernel<4>
                  : chunks <= R_THREADS * 8 ? fp8_rows_kernel<8> : fp8_rows_kernel<16>;
  return launch("fp8_rows_kernel", kern, M, R_THREADS, 0, stream, ALLOW_PDL, xb, ldx, K, o, ldo, row_scale_inv);
}

extern "C" int ivb_fp8_quantize_cols_t(const void* x, long ldx, int M, int K, void* out_t, long ldt, float* col_amax,
                                       float* col_scale_inv, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || K <= 0) return set_error("ivb_fp8_quantize_cols_t: empty tensor");
  if (x == nullptr || out_t == nullptr || col_amax == nullptr || col_scale_inv == nullptr)
    return set_error("ivb_fp8_quantize_cols_t: x, out_t, col_amax or col_scale_inv is null");
  if ((ldx & 7) || ldx < K) return set_error("ivb_fp8_quantize_cols_t: ldx must be a multiple of 8 elements and >= K");
  if ((ldt & 15) || ldt < M) return set_error("ivb_fp8_quantize_cols_t: ldt must be a multiple of 16 elements and >= M");
  if (misaligned(16, x, out_t)) return set_error("ivb_fp8_quantize_cols_t: x and out_t must be 16-byte aligned");
  if (misaligned(4, col_amax, col_scale_inv))
    return set_error("ivb_fp8_quantize_cols_t: col_amax and col_scale_inv must be 4-byte aligned");
  cudaError_t e = cudaMemsetAsync(col_amax, 0, sizeof(float) * static_cast<size_t>(K), stream);
  if (e != cudaSuccess) return set_error_cuda("ivb_fp8_quantize_cols_t: cudaMemsetAsync", e);
  const auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  unsigned* bits = reinterpret_cast<unsigned*>(col_amax);
  const unsigned strips = (K + Q_TILE - 1) / Q_TILE;
  if (int rc = launch("fp8_col_amax_kernel", fp8_col_amax_kernel, dim3(strips, (M + Q_COL_ROWS - 1) / Q_COL_ROWS),
                      Q_THREADS, 0, stream, ALLOW_PDL, xb, ldx, M, K, bits))
    return rc;
  return launch("fp8_cast_cols_kernel", fp8_cast_cols_kernel, dim3(strips, (M + Q_TILE - 1) / Q_TILE), Q_THREADS, 0,
                stream, ALLOW_PDL, xb, ldx, M, K, bits, reinterpret_cast<uint8_t*>(out_t), ldt, col_scale_inv);
}

extern "C" int ivb_fp8_quantize(const void* x, long ldx, int M, int K, int format, void* out, long ldo, void* out_t,
                                long ldt, float* amax, float* scale_inv, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || K <= 0) return set_error("ivb_fp8_quantize: empty tensor");
  if (format != IVB_FP8_E4M3 && format != IVB_FP8_E5M2) return set_error("ivb_fp8_quantize: unknown format");
  if (x == nullptr || out == nullptr) return set_error("ivb_fp8_quantize: x or out is null");
  if (amax == nullptr || scale_inv == nullptr) return set_error("ivb_fp8_quantize: amax or scale_inv is null");
  if ((ldx & 7) || ldx < K) return set_error("ivb_fp8_quantize: ldx must be a multiple of 8 elements and >= K");
  if ((ldo & 15) || ldo < K) return set_error("ivb_fp8_quantize: ldo must be a multiple of 16 elements and >= K");
  if (out_t != nullptr && ((ldt & 15) || ldt < M))
    return set_error("ivb_fp8_quantize: ldt must be a multiple of 16 elements and >= M");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(out_t)) & 15)
    return set_error("ivb_fp8_quantize: x, out and out_t must be 16-byte aligned");
  if ((reinterpret_cast<uintptr_t>(amax) | reinterpret_cast<uintptr_t>(scale_inv)) & 3)
    return set_error("ivb_fp8_quantize: amax and scale_inv must be 4-byte aligned");
  cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), stream);
  if (e != cudaSuccess) return set_error_cuda("ivb_fp8_quantize: cudaMemsetAsync", e);
  const auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  unsigned* bits = reinterpret_cast<unsigned*>(amax);
  const long chunks = static_cast<long>(M) * ((K + 7) / 8);
  const int grid = persistent_grid(chunks, 256, 8);
  if (int rc = launch("fp8_amax_kernel", fp8_amax_kernel, grid, 256, 0, stream, ALLOW_PDL, xb, ldx, M, K, bits))
    return rc;
  const dim3 cast_grid((K + Q_TILE - 1) / Q_TILE, (M + Q_TILE - 1) / Q_TILE);
  return launch("fp8_cast_kernel", format == IVB_FP8_E5M2 ? fp8_cast_kernel<true> : fp8_cast_kernel<false>, cast_grid,
                Q_THREADS, 0, stream, ALLOW_PDL, xb, ldx, M, K, bits, reinterpret_cast<uint8_t*>(out), ldo,
                reinterpret_cast<uint8_t*>(out_t), ldt, scale_inv);
}
