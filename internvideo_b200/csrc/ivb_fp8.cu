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
#include "ivb_internal.h"
#include "ivb_ptx.cuh"

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

// scale = 2^e with e the largest integer such that amax * 2^e <= fmax = 1.75 * 2^F, from the bits of amax (exact, no
// rounding of fmax / amax); e is clamped to [-126, 126] so that scale and 1 / scale are normal floats.
__device__ __forceinline__ void fp8_scale(unsigned amax_bits, int F, float& scale, float& scale_inv) {
  if ((amax_bits & 0x7f800000u) == 0x7f800000u) {   // Inf or NaN
    scale = 1.0f;
    scale_inv = __int_as_float(0x7fc00000);
    return;
  }
  if (amax_bits == 0) {
    scale = scale_inv = 1.0f;
    return;
  }
  const int E = static_cast<int>((amax_bits >> 23) & 0xff) - 127;
  int e = F - E - ((amax_bits & 0x7fffffu) > 0x600000u ? 1 : 0);
  e = min(126, max(-126, e));
  scale = __int_as_float((e + 127) << 23);
  scale_inv = __int_as_float((127 - e) << 23);
}

template <bool E5M2>
__device__ __forceinline__ uint32_t cvt_fp8x2(float lo, float hi) {
  uint16_t r;
  if constexpr (E5M2)
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// One 64 x 64 tile per CTA: thread t converts 16 elements of row t / 4 and writes them to `out`; with out_t, the tile
// is transposed through shared memory and thread t writes 16 elements of row t / 4 of out_t's tile.
template <bool E5M2>
__global__ void __launch_bounds__(Q_THREADS) fp8_cast_kernel(const __nv_bfloat16* __restrict__ x, long ldx, int M,
                                                             int K, const unsigned* amax_bits, uint8_t* out, long ldo,
                                                             uint8_t* out_t, long ldt, float* scale_inv) {
  __shared__ __align__(16) uint8_t tile[Q_TILE * Q_PITCH];
  pdl_wait();
  pdl_launch_dependents();
  float scale, sinv;
  fp8_scale(*amax_bits, E5M2 ? 15 : 8, scale, sinv);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv = sinv;
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

}  // namespace ivb

using namespace ivb;

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
  e = launch_pdl(fp8_amax_kernel, dim3(grid), dim3(256), 0, stream, xb, ldx, M, K, bits);
  if (e != cudaSuccess) return set_error_cuda("launch(fp8_amax_kernel)", e);
  count_launch();
  if (int rc = check_launch("fp8_amax_kernel")) return rc;
  const dim3 cast_grid((K + Q_TILE - 1) / Q_TILE, (M + Q_TILE - 1) / Q_TILE);
  auto* o = reinterpret_cast<uint8_t*>(out);
  auto* ot = reinterpret_cast<uint8_t*>(out_t);
  if (format == IVB_FP8_E5M2)
    e = launch_pdl(fp8_cast_kernel<true>, cast_grid, dim3(Q_THREADS), 0, stream, xb, ldx, M, K, bits, o, ldo, ot, ldt,
                   scale_inv);
  else
    e = launch_pdl(fp8_cast_kernel<false>, cast_grid, dim3(Q_THREADS), 0, stream, xb, ldx, M, K, bits, o, ldo, ot, ldt,
                   scale_inv);
  if (e != cudaSuccess) return set_error_cuda("launch(fp8_cast_kernel)", e);
  count_launch();
  return check_launch("fp8_cast_kernel");
}
