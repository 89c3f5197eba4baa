// ivb_gemm_common.cuh — GEMM parameter block and the fused epilogue of the wgmma GEMM (ivb_gemm.cu).
//
// Epilogue data path: the MMA warps stage their accumulator fragments through a small per-warp shared-memory
// tile so that every thread ends up with a contiguous row segment (16 columns); the thread applies the fused
// epilogue and writes the segment straight to global memory with 128-bit accesses.
#pragma once
#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

struct GemmParams {
  int M, N, K;
  int epi;      // IVB_EPI_*
  int flags;    // IVB_FLAG_*
  void* out0;
  long ld0;
  void* out1;
  long ld1;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* gamma;
  const void* aux;
  long ldaux;
  const float* rowscale;  // EPI_RESID: optional per-row multiplier of the branch (DropPath keep/scale)
};

// 32-byte row pieces as two 128-bit accesses (sm_90 has no 256-bit global load / store).
__device__ __forceinline__ void st_global_256(void* p, const uint32_t r[8]) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(r[0], r[1], r[2], r[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(r[4], r[5], r[6], r[7]);
}
__device__ __forceinline__ void ld_global_256(const void* p, uint32_t r[8]) {
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}

// Row-segment I/O: W elements starting at `ptr`; `nvalid` (multiple of 8) of them are inside the matrix.
template <int W>
__device__ __forceinline__ void store_row_bf16(__nv_bfloat16* ptr, const float* v, int nvalid) {
  const bool wide = (reinterpret_cast<uintptr_t>(ptr) & 31) == 0;
#pragma unroll
  for (int i = 0; i < W; i += 16) {
    uint32_t r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = pack_bf16(v[i + 2 * k], v[i + 2 * k + 1]);
    if (wide && i + 16 <= nvalid) {
      st_global_256(ptr + i, r);
    } else {
      if (i < nvalid) *reinterpret_cast<uint4*>(ptr + i) = make_uint4(r[0], r[1], r[2], r[3]);
      if (i + 8 < nvalid) *reinterpret_cast<uint4*>(ptr + i + 8) = make_uint4(r[4], r[5], r[6], r[7]);
    }
  }
}
template <int W>
__device__ __forceinline__ void load_row_bf16(const __nv_bfloat16* ptr, float* v, int nvalid) {
  const bool wide = (reinterpret_cast<uintptr_t>(ptr) & 31) == 0;
#pragma unroll
  for (int i = 0; i < W; i += 16) {
    uint32_t r[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    if (wide && i + 16 <= nvalid) {
      ld_global_256(ptr + i, r);
    } else {
      if (i < nvalid) { const uint4 a = *reinterpret_cast<const uint4*>(ptr + i); r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; }
      if (i + 8 < nvalid) { const uint4 a = *reinterpret_cast<const uint4*>(ptr + i + 8); r[4] = a.x; r[5] = a.y; r[6] = a.z; r[7] = a.w; }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) { const float2 f = unpack_bf16(r[k]); v[i + 2 * k] = f.x; v[i + 2 * k + 1] = f.y; }
  }
}
template <int W>
__device__ __forceinline__ void store_row_f32(float* ptr, const float* v, int nvalid) {
  const bool wide = (reinterpret_cast<uintptr_t>(ptr) & 31) == 0;
#pragma unroll
  for (int i = 0; i < W; i += 8) {
    if (i < nvalid) {
      if (wide) {
        uint32_t r[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) r[k] = __float_as_uint(v[i + k]);
        st_global_256(ptr + i, r);
      } else {
        *reinterpret_cast<float4*>(ptr + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
        *reinterpret_cast<float4*>(ptr + i + 4) = make_float4(v[i + 4], v[i + 5], v[i + 6], v[i + 7]);
      }
    }
  }
}
template <int W>
__device__ __forceinline__ void load_row_f32(const float* ptr, float* v, int nvalid) {
  const bool wide = (reinterpret_cast<uintptr_t>(ptr) & 31) == 0;
#pragma unroll
  for (int i = 0; i < W; i += 8) {
    if (i < nvalid) {
      if (wide) {
        uint32_t r[8];
        ld_global_256(ptr + i, r);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[i + k] = __uint_as_float(r[k]);
      } else {
        const float4 a = *reinterpret_cast<const float4*>(ptr + i), b = *reinterpret_cast<const float4*>(ptr + i + 4);
        v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
        v[i + 4] = b.x; v[i + 5] = b.y; v[i + 6] = b.z; v[i + 7] = b.w;
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[i + k] = 0.f;
    }
  }
}

// ------------------------------------------------------------------ epilogue for W columns of one row
// acc_bits: W fp32 accumulators of (row, col0 .. col0+W-1).  W is a multiple of 16.
template <int W>
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, const uint32_t* acc_bits, long row, int col0) {
  int nvalid = p.N - col0;
  if (nvalid <= 0) return;
  if (nvalid > W) nvalid = W;
  float v[W];
#pragma unroll
  for (int i = 0; i < W; ++i) v[i] = __uint_as_float(acc_bits[i]);
  if (p.bias != nullptr) {
    float bv[W];
    load_row_bf16<W>(p.bias + col0, bv, nvalid);
#pragma unroll
    for (int i = 0; i < W; ++i) v[i] += bv[i];
  }
  const bool accum = (p.flags & IVB_FLAG_ACCUM) != 0;
  const bool tanh_mode = (p.flags & IVB_FLAG_GELU_TANH) != 0;
  switch (p.epi) {
    case IVB_EPI_BF16: {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + col0;
      if (accum) {
        float old[W];
        load_row_bf16<W>(o, old, nvalid);
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] += old[i];
      }
      store_row_bf16<W>(o, v, nvalid);
    } break;
    case IVB_EPI_F32: {
      float* o = reinterpret_cast<float*>(p.out0) + row * p.ld0 + col0;
      if (accum) {
        float old[W];
        load_row_f32<W>(o, old, nvalid);
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] += old[i];
      }
      store_row_f32<W>(o, v, nvalid);
    } break;
    case IVB_EPI_BIAS_GELU: {
      // NOTE: the erf/tanh choice is hoisted out of the element loops on purpose.  With the branch inside,
      // every element became its own basic block and the MUFU latency chains of the 32 elements could not
      // be interleaved: the epilogue ran at ~8K cycles per 32-column chunk instead of ~1K.
      if (p.out1 != nullptr && (p.flags & IVB_FLAG_GELU_SAVE_GRAD) != 0) {
        // save gelu'(h) (shares the exponential with gelu(h)) so the backward epilogue is one multiply
        float dv[W];
        if (tanh_mode) {
#pragma unroll
          for (int i = 0; i < W; ++i) { dv[i] = gelu_tanh_grad(v[i]); v[i] = gelu_tanh(v[i]); }
        } else {
#pragma unroll
          for (int i = 0; i < W; ++i) {
            float cdf, pdf;
            gelu_cdf_pdf(v[i], cdf, pdf);
            dv[i] = fmaf(v[i], pdf, cdf);
            v[i] *= cdf;
          }
        }
        store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out1) + row * p.ld1 + col0, dv, nvalid);
      } else {
        if (p.out1 != nullptr)
          store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out1) + row * p.ld1 + col0, v, nvalid);
        if (tanh_mode) {
#pragma unroll
          for (int i = 0; i < W; ++i) v[i] = gelu_tanh(v[i]);
        } else {
#pragma unroll
          for (int i = 0; i < W; ++i) v[i] = gelu_erf(v[i]);
        }
      }
      store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    case IVB_EPI_RESID: {
      // y = acc + bias ; out1(bf16) = y (optional, kept for the LayerScale gamma gradient)
      // out0(fp32) = aux(fp32 residual stream) + rowscale * gamma * y
      if (p.out1 != nullptr)
        store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out1) + row * p.ld1 + col0, v, nvalid);
      const float rs = p.rowscale ? p.rowscale[row] : 1.0f;
      float res[W];
      load_row_f32<W>(reinterpret_cast<const float*>(p.aux) + row * p.ldaux + col0, res, nvalid);
      if (p.gamma != nullptr) {
        float gm[W];
        load_row_bf16<W>(p.gamma + col0, gm, nvalid);
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] = fmaf(gm[i] * rs, v[i], res[i]);
      } else {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] = fmaf(rs, v[i], res[i]);
      }
      store_row_f32<W>(reinterpret_cast<float*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    case IVB_EPI_GELU_BWD: {
      // out0(bf16) = acc * gelu'(aux(bf16 pre-activation))   [or acc * aux with GELU_SAVE_GRAD]
      float hv[W];
      load_row_bf16<W>(reinterpret_cast<const __nv_bfloat16*>(p.aux) + row * p.ldaux + col0, hv, nvalid);
      if ((p.flags & IVB_FLAG_GELU_SAVE_GRAD) != 0) {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= hv[i];
      } else if (tanh_mode) {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= gelu_tanh_grad(hv[i]);
      } else {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= gelu_erf_grad(hv[i]);
      }
      store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    default:
      break;
  }
}

}  // namespace ivb
