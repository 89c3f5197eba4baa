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
//
// Every kernel is built from the pieces of ivb_fp8.cuh: load_chunk, bf16_mag_max / bf16_mag_cols, col_amax, the
// transposing Fp8TileT and store_fp8.
#include <cstdio>

#include "ivb_fp8.cuh"
#include "ivb_internal.h"
#include "ivb_rows.cuh"

namespace ivb {

constexpr int Q_TILE = 64;         // the cast kernels' tile: 64 rows x 64 columns, 16 elements per thread
constexpr int Q_THREADS = 256;
using QTile = Fp8TileT<Q_TILE, Q_TILE>;

__global__ void __launch_bounds__(256) fp8_amax_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M, int K,
                                                       unsigned* amax_bits) {
  pdl_wait();
  pdl_launch_dependents();
  const long kc = (K + 7) / 8;
  const long chunks = static_cast<long>(M) * kc;
  unsigned m = 0;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < chunks;
       i += static_cast<long>(gridDim.x) * blockDim.x)
    m = max(m, bf16_mag_max(load_chunk(x + (i / kc) * ldx, static_cast<int>(i % kc) * 8, K)));
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(amax_bits, m << 16);
}

// Chunk h of thread t's 16 elements of the cast kernels' tile: row t / 4 of the tile, columns 16 (t % 4) + 8 h ..;
// zeros outside the tensor.
__device__ __forceinline__ uint4 q_tile_chunk(const __nv_bfloat16* x, long ldx, int M, int K, int row, int col, int h) {
  return row < M ? load_chunk(x + static_cast<long>(row) * ldx, col + 8 * h, K) : make_uint4(0u, 0u, 0u, 0u);
}

// One 64 x 64 tile per CTA: thread t casts 16 elements of row t / 4 and writes them to `out`; with out_t, the tile is
// transposed through shared memory and thread t writes 16 elements of row t / 4 of out_t's tile.
template <bool E5M2>
__global__ void __launch_bounds__(Q_THREADS) fp8_cast_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                             int K, const unsigned* amax_bits, uint8_t* out, long ldo,
                                                             uint8_t* out_t, long ldt, float* scale_inv) {
  __shared__ QTile tile;
  pdl_wait();
  pdl_launch_dependents();
  float scale, sinv;
  fp8_scale(*amax_bits, E5M2 ? 15 : 8, scale, sinv);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv = sinv;
  const int m0 = blockIdx.y * Q_TILE, k0 = blockIdx.x * Q_TILE;
  const int r = threadIdx.x >> 2, c = (threadIdx.x & 3) * 16;
  const int row = m0 + r, col = k0 + c;
  uint32_t q[4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float f[8];
    unpack8(q_tile_chunk(x, ldx, M, K, row, col, h), f);
#pragma unroll
    for (int k = 0; k < 2; ++k)
      q[2 * h + k] = cvt_fp8x2<E5M2>(f[4 * k] * scale, f[4 * k + 1] * scale) |
                     (cvt_fp8x2<E5M2>(f[4 * k + 2] * scale, f[4 * k + 3] * scale) << 16);
  }
  store_fp8(out + static_cast<long>(row) * ldo + col, make_uint4(q[0], q[1], q[2], q[3]), row < M ? K - col : 0);
  if (out_t == nullptr) return;
  tile.put8(c, r, make_uint2(q[0], q[1]));
  tile.put8(c + 8, r, make_uint2(q[2], q[3]));
  __syncthreads();
  // out_t row k0 + r holds column k0 + r of the tile: tensor rows m0 + c .. m0 + c + 15
  if (k0 + r < K) tile.store<16>(r, c, out_t + static_cast<long>(k0 + r) * ldt + m0 + c, M - m0 - c);
}

// ------------------------------------------------------------------ per-column scaling (ivb_fp8_quantize_cols_t)
// The column amax of a 64-column strip over Q_COL_ROWS rows per CTA: thread t reads the 8-column chunk t % 8 of rows
// t / 8, t / 8 + 32, ...; col_amax reduces the CTA's strip, then one integer atomicMax per column (order-independent:
// the same bits on every run).
constexpr int Q_COL_ROWS = 256;

__global__ void __launch_bounds__(Q_THREADS) fp8_col_amax_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                                 int K, unsigned* col_amax_bits) {
  __shared__ unsigned red[Q_THREADS / 32][Q_TILE];
  pdl_wait();
  pdl_launch_dependents();
  const int c = blockIdx.x * Q_TILE + (threadIdx.x & 7) * 8;
  const int r1 = min(M, (blockIdx.y + 1) * Q_COL_ROWS);
  unsigned m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
  if (c < K) {
    for (int row = blockIdx.y * Q_COL_ROWS + (threadIdx.x >> 3); row < r1; row += Q_THREADS / 8)
      bf16_mag_cols(load_chunk(x + static_cast<long>(row) * ldx, c, K), m);
  }
  const unsigned mx = col_amax<8, Q_THREADS>(m, red);
  const int col = blockIdx.x * Q_TILE + threadIdx.x;
  if (threadIdx.x < Q_TILE && col < K && mx != 0) atomicMax(col_amax_bits + col, mx << 16);
}

// The cast kernel's tile with one scale per column, from col_amax_bits[K] and written to col_scale_inv[K]; only the
// transposed copy is written.
__global__ void __launch_bounds__(Q_THREADS) fp8_cast_cols_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                                  int K, const unsigned* col_amax_bits, uint8_t* out_t,
                                                                  long ldt, float* col_scale_inv) {
  __shared__ QTile tile;
  pdl_wait();
  pdl_launch_dependents();
  const int m0 = blockIdx.y * Q_TILE, k0 = blockIdx.x * Q_TILE;
  const int r = threadIdx.x >> 2, c = (threadIdx.x & 3) * 16;
  const int row = m0 + r, col = k0 + c;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float scale[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int ck = col + 8 * h + k;
      float sinv;
      fp8_scale(ck < K ? col_amax_bits[ck] : 0u, 8, scale[k], sinv);
      if (blockIdx.y == 0 && r == 0 && ck < K) col_scale_inv[ck] = sinv;
    }
    tile.put(c + 8 * h, r, q_tile_chunk(x, ldx, M, K, row, col, h), scale);
  }
  __syncthreads();
  if (k0 + r < K) tile.store<16>(r, c, out_t + static_cast<long>(k0 + r) * ldt + m0 + c, M - m0 - c);
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
  unsigned m = 0;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i] = load_chunk(src, (threadIdx.x + R_THREADS * i) * 8, K);
    m = max(m, bf16_mag_max(v[i]));
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
    store_fp8(dst + c, cvt_e4m3x8(f, scale), K - c);
  }
}

// ------------------------------------------------------------------ per-(128-token block, channel) scaling
// (ivb_fp8_quantize_blocks_t: the operands of the FP8 weight gradient, ivb_gemm_fp8_wgrad)
// One CTA per 128 tokens x 64 channels: thread t reads the 8-channel chunk t % 8 of tokens t / 8, t / 8 + 32, ...
// into registers (x is read once), col_amax reduces the column amax (no atomics: the same bits on every run), then
// each element is scaled by its column's factor, cast and transposed through shared memory, and thread t writes 32
// tokens of channel t / 4.  rowscale (optional): tokens whose factor is 0 are cast as zeros.
constexpr int B_TOK = 128, B_CH = 64;

__global__ void __launch_bounds__(Q_THREADS) fp8_blocks_t_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                                 int C, const float* __restrict__ rowscale,
                                                                 uint8_t* __restrict__ out_t, long ldt,
                                                                 float* __restrict__ scale_inv) {
  __shared__ unsigned red[Q_THREADS / 32][B_CH];
  __shared__ Fp8TileT<B_CH, B_TOK> tile;
  pdl_wait();
  pdl_launch_dependents();
  const int m0 = blockIdx.y * B_TOK, c0 = blockIdx.x * B_CH;
  const int cc = (threadIdx.x & 7) * 8, r0 = threadIdx.x >> 3;   // chunk column in the strip, first token
  const int col = c0 + cc;
  uint4 v[B_TOK / 32];
  unsigned m[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
#pragma unroll
  for (int i = 0; i < B_TOK / 32; ++i) {
    const int row = m0 + r0 + 32 * i;
    v[i] = make_uint4(0u, 0u, 0u, 0u);
    if (row < M && col < C && (rowscale == nullptr || rowscale[row] != 0.0f))
      v[i] = *reinterpret_cast<const uint4*>(x + static_cast<long>(row) * ldx + col);
    bf16_mag_cols(v[i], m);
  }
  col_amax<8, Q_THREADS>(m, red);
  float scale[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    float sinv;
    fp8_scale(red[0][cc + k] << 16, 8, scale[k], sinv);
    if (r0 == 0 && col < C) scale_inv[static_cast<long>(blockIdx.y) * C + col + k] = sinv;
  }
#pragma unroll
  for (int i = 0; i < B_TOK / 32; ++i) tile.put(cc, r0 + 32 * i, v[i], scale);
  __syncthreads();
  // out_t row c0 + t / 4 holds channel c0 + t / 4: tokens m0 + 32 (t % 4) .. + 31
  const int trow = c0 + (threadIdx.x >> 2), tok = 32 * (threadIdx.x & 3);
  if (trow < C) tile.store<32>(threadIdx.x >> 2, tok, out_t + static_cast<long>(trow) * ldt + m0 + tok, M - m0 - tok);
}

}  // namespace ivb

using namespace ivb;

// Sets the error text "<fn>: <what>"; returns set_error's status.
static int fail(const char* fn, const char* what) {
  char msg[128];
  std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
  return set_error(msg);
}

// ivb_fp8_quantize_blocks_t and ivb_fp8_quantize_blocks_t_plan; `fn` names the entry point in messages.
static int quantize_blocks_t(const char* fn, const void* x, long ldx, int M, int C, void* out_t, long ldt,
                             float* scale_inv, const float* rowscale, cudaStream_t stream) {
  if (M <= 0 || C <= 0) return fail(fn, "empty tensor");
  if (C & 7) return fail(fn, "C must be a multiple of 8");
  if (x == nullptr || out_t == nullptr || scale_inv == nullptr) return fail(fn, "x, out_t or scale_inv is null");
  if ((ldx & 7) || ldx < C) return fail(fn, "ldx must be a multiple of 8 elements and >= C");
  if ((ldt & 15) || ldt < M) return fail(fn, "ldt must be a multiple of 16 elements and >= M");
  if (misaligned(16, x, out_t)) return fail(fn, "x and out_t must be 16-byte aligned");
  if (misaligned(4, scale_inv, rowscale)) return fail(fn, "scale_inv and rowscale must be 4-byte aligned");
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
  const char* fn = "ivb_fp8_quantize_blocks_t_plan";
  if (rowscale == nullptr) return fail(fn, "rowscale is null");
  return quantize_blocks_t(fn, x, ldx, M, C, out_t, ldt, scale_inv, rowscale, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_fp8_quantize_rows(const void* x, long ldx, int M, int K, void* out, long ldo, float* row_scale_inv,
                                     void* stream) {
  const char* fn = "ivb_fp8_quantize_rows";
  if (M <= 0 || K <= 0) return fail(fn, "empty tensor");
  if (K > IVB_FP8_ROWS_MAX_K) return fail(fn, "K > IVB_FP8_ROWS_MAX_K");
  if (x == nullptr || out == nullptr || row_scale_inv == nullptr) return fail(fn, "x, out or row_scale_inv is null");
  if ((ldx & 7) || ldx < K) return fail(fn, "ldx must be a multiple of 8 elements and >= K");
  if ((ldo & 15) || ldo < K) return fail(fn, "ldo must be a multiple of 16 elements and >= K");
  if (misaligned(16, x, out)) return fail(fn, "x and out must be 16-byte aligned");
  if (misaligned(4, row_scale_inv)) return fail(fn, "row_scale_inv must be 4-byte aligned");
  const int chunks = (K + 7) / 8;   // per row; each thread holds NV of them
  const auto kern = chunks <= R_THREADS * 2 ? fp8_rows_kernel<2>
                  : chunks <= R_THREADS * 4 ? fp8_rows_kernel<4>
                  : chunks <= R_THREADS * 8 ? fp8_rows_kernel<8> : fp8_rows_kernel<16>;
  return launch("fp8_rows_kernel", kern, M, R_THREADS, 0, reinterpret_cast<cudaStream_t>(stream), ALLOW_PDL,
                reinterpret_cast<const __nv_bfloat16*>(x), ldx, K, reinterpret_cast<uint8_t*>(out), ldo, row_scale_inv);
}

extern "C" int ivb_fp8_quantize_cols_t(const void* x, long ldx, int M, int K, void* out_t, long ldt, float* col_amax,
                                       float* col_scale_inv, void* stream_) {
  const char* fn = "ivb_fp8_quantize_cols_t";
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || K <= 0) return fail(fn, "empty tensor");
  if (x == nullptr || out_t == nullptr || col_amax == nullptr || col_scale_inv == nullptr)
    return fail(fn, "x, out_t, col_amax or col_scale_inv is null");
  if ((ldx & 7) || ldx < K) return fail(fn, "ldx must be a multiple of 8 elements and >= K");
  if ((ldt & 15) || ldt < M) return fail(fn, "ldt must be a multiple of 16 elements and >= M");
  if (misaligned(16, x, out_t)) return fail(fn, "x and out_t must be 16-byte aligned");
  if (misaligned(4, col_amax, col_scale_inv)) return fail(fn, "col_amax and col_scale_inv must be 4-byte aligned");
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
  const char* fn = "ivb_fp8_quantize";
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || K <= 0) return fail(fn, "empty tensor");
  if (format != IVB_FP8_E4M3 && format != IVB_FP8_E5M2) return fail(fn, "unknown format");
  if (x == nullptr || out == nullptr) return fail(fn, "x or out is null");
  if (amax == nullptr || scale_inv == nullptr) return fail(fn, "amax or scale_inv is null");
  if ((ldx & 7) || ldx < K) return fail(fn, "ldx must be a multiple of 8 elements and >= K");
  if ((ldo & 15) || ldo < K) return fail(fn, "ldo must be a multiple of 16 elements and >= K");
  if (out_t != nullptr && ((ldt & 15) || ldt < M)) return fail(fn, "ldt must be a multiple of 16 elements and >= M");
  if (misaligned(16, x, out, out_t)) return fail(fn, "x, out and out_t must be 16-byte aligned");
  if (misaligned(4, amax, scale_inv)) return fail(fn, "amax and scale_inv must be 4-byte aligned");
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
