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
  const float* a_scale_inv;  // fp8 operands: device scalars, the accumulator is multiplied by their product
  const float* b_scale_inv;
  // DropPath plan (ivb_droppath_plan), planned kernels only (PLANNED, ivb_gemm.cu); null: every tile, every k-block.
  // m_plan: the ceil(M/128) row tiles, live ones first, then their count; a dead tile runs dead_tile instead of its MMAs.
  // k_plan: the ascending live 64-row k-blocks, then their count; the k-blocks it leaves out are skipped.
  const int* m_plan;
  const int* k_plan;
};

// The epilogue's outputs for a tile whose rows all have DropPath factor 0, with no MMA: EPI_RESID passes the residual
// through (out0 = aux, out1 = 0), every other epilogue writes zeros (EPI_GELU_BWD without reading aux).  Also every
// tile of a K plan that lists no k-block (EPI_BF16 / EPI_F32 without bias): zeros, or under IVB_FLAG_ACCUM nothing.
// Rows [row0, row0 + rows) and columns [n0, n0 + BN) inside the matrix, in 16-byte vectors by the 128 threads of a
// warpgroup.
template <int BN>
__device__ __forceinline__ void dead_tile(const GemmParams& p, long row0, int rows, int n0) {
  if (p.flags & IVB_FLAG_ACCUM) return;
  const int units = min(BN, p.N - n0) / 8;   // 8-column pieces per row (N is a multiple of 8)
  const long nrows = min(static_cast<long>(rows), p.M - row0);
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (long i = threadIdx.x & 127; i < nrows * units; i += 128) {
    const long row = row0 + i / units;
    const int col = n0 + static_cast<int>(i % units) * 8;
    if (p.epi == IVB_EPI_RESID || p.epi == IVB_EPI_F32) {
      uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<float*>(p.out0) + row * p.ld0 + col);
      if (p.epi == IVB_EPI_RESID) {
        const uint4* a = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.aux) + row * p.ldaux + col);
        o[0] = a[0]; o[1] = a[1];
      } else {
        o[0] = z; o[1] = z;
      }
    } else {
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + col) = z;
    }
    if (p.out1 != nullptr && (p.epi == IVB_EPI_RESID || p.epi == IVB_EPI_BIAS_GELU))
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out1) + row * p.ld1 + col) = z;
  }
}

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
// Raw bits of W bf16 (W / 2 words) starting at `ptr`; words of elements past `nvalid` are zero.
template <int W>
__device__ __forceinline__ void load_bits_bf16(const __nv_bfloat16* ptr, uint32_t* r, int nvalid) {
  const bool wide = (reinterpret_cast<uintptr_t>(ptr) & 31) == 0;
#pragma unroll
  for (int i = 0; i < W; i += 16) {
    uint32_t* q = r + i / 2;
    if (wide && i + 16 <= nvalid) {
      ld_global_256(ptr + i, q);
    } else {
      uint4 a = make_uint4(0u, 0u, 0u, 0u), b = a;
      if (i < nvalid) a = *reinterpret_cast<const uint4*>(ptr + i);
      if (i + 8 < nvalid) b = *reinterpret_cast<const uint4*>(ptr + i + 8);
      q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
    }
  }
}
template <int W>
__device__ __forceinline__ void unpack_row_bf16(const uint32_t* r, float* v) {
#pragma unroll
  for (int k = 0; k < W / 2; ++k) { const float2 f = unpack_bf16(r[k]); v[2 * k] = f.x; v[2 * k + 1] = f.y; }
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
// Raw bits of W fp32 starting at `ptr`; words of elements past `nvalid` are zero.
template <int W>
__device__ __forceinline__ void load_bits_f32(const float* ptr, uint32_t* r, int nvalid) {
  const bool wide = (reinterpret_cast<uintptr_t>(ptr) & 31) == 0;
#pragma unroll
  for (int i = 0; i < W; i += 8) {
    if (i < nvalid) {
      if (wide) {
        ld_global_256(ptr + i, r + i);
      } else {
        const uint4 a = *reinterpret_cast<const uint4*>(ptr + i), b = *reinterpret_cast<const uint4*>(ptr + i + 4);
        r[i] = a.x; r[i + 1] = a.y; r[i + 2] = a.z; r[i + 3] = a.w;
        r[i + 4] = b.x; r[i + 5] = b.y; r[i + 6] = b.z; r[i + 7] = b.w;
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) r[i + k] = 0u;
    }
  }
}

// ------------------------------------------------------------------ epilogue for W columns of one row
// What one row segment reads from global memory besides bias and gamma: aux (EPI_RESID: the fp32 residual stream;
// EPI_GELU_BWD: the bf16 pre-activation or saved GELU'), out0's old values under IVB_FLAG_ACCUM, and the EPI_RESID row
// scale.  epilogue_tile loads it a chunk ahead, so its HBM latency is not on the epilogue's critical path.
template <int W>
struct EpiIn {
  uint32_t x[W];   // raw bits: W fp32, or W bf16 in the first W / 2 words
  float rs;
};

template <int W>
__device__ __forceinline__ void epilogue_load(const GemmParams& p, bool accum, EpiIn<W>& in, long row, int col0,
                                              int nvalid) {
  switch (p.epi) {
    case IVB_EPI_BF16:
      if (accum) load_bits_bf16<W>(reinterpret_cast<const __nv_bfloat16*>(p.out0) + row * p.ld0 + col0, in.x, nvalid);
      break;
    case IVB_EPI_F32:
      if (accum) load_bits_f32<W>(reinterpret_cast<const float*>(p.out0) + row * p.ld0 + col0, in.x, nvalid);
      break;
    case IVB_EPI_RESID:
      in.rs = p.rowscale ? p.rowscale[row] : 1.0f;
      load_bits_f32<W>(reinterpret_cast<const float*>(p.aux) + row * p.ldaux + col0, in.x, nvalid);
      break;
    case IVB_EPI_GELU_BWD:
      load_bits_bf16<W>(reinterpret_cast<const __nv_bfloat16*>(p.aux) + row * p.ldaux + col0, in.x, nvalid);
      break;
    default:
      break;
  }
}

// v: the W fp32 accumulators of (row, col0 .. col0+W-1), 0 < nvalid <= W of them inside the matrix.  in: what
// epilogue_load read for them.  bias_bits / gamma_bits: the W bf16 of bias / gamma at col0 (when the GEMM has them).
// SWIGLU: build the IVB_EPI_SWIGLU case (the bf16 kernels).  The FP8 kernels, whose entry points refuse it, leave it
// out: compiled in, it costs the cooperative E4M3 kernel at BN 192 an 8-byte spill.
template <int W, bool SWIGLU>
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, bool accum, bool tanh_mode, bool quick_mode,
                                               bool save_grad, float* v, const EpiIn<W>& in, const uint32_t* bias_bits,
                                               const uint32_t* gamma_bits, long row, int col0, int nvalid) {
  if (p.bias != nullptr) {
    float bv[W];
    unpack_row_bf16<W>(bias_bits, bv);
#pragma unroll
    for (int i = 0; i < W; ++i) v[i] += bv[i];
  }
  switch (p.epi) {
    case IVB_EPI_BF16: {
      if (accum) {
        float old[W];
        unpack_row_bf16<W>(in.x, old);
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] += old[i];
      }
      store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    case IVB_EPI_F32: {
      if (accum) {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] += __uint_as_float(in.x[i]);
      }
      store_row_f32<W>(reinterpret_cast<float*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    case IVB_EPI_BIAS_GELU: {
      // NOTE: the erf/tanh/quick choice is hoisted out of the element loops on purpose.  With the branch inside,
      // every element became its own basic block and the MUFU latency chains of the 32 elements could not
      // be interleaved: the epilogue ran at ~8K cycles per 32-column chunk instead of ~1K.
      if (p.out1 != nullptr && save_grad) {
        // save gelu'(h) (shares the exponential with gelu(h)) so the backward epilogue is one multiply
        float dv[W];
        if (tanh_mode) {
#pragma unroll
          for (int i = 0; i < W; ++i) { dv[i] = gelu_tanh_grad(v[i]); v[i] = gelu_tanh(v[i]); }
        } else if (quick_mode) {
#pragma unroll
          for (int i = 0; i < W; ++i) {
            const float s = gelu_quick_sig(v[i]);
            dv[i] = fmaf(1.702f * v[i] * s, 1.0f - s, s);
            v[i] *= s;
          }
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
        } else if (quick_mode) {
#pragma unroll
          for (int i = 0; i < W; ++i) v[i] = gelu_quick(v[i]);
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
      const float rs = in.rs;
      if (p.gamma != nullptr) {
        float gm[W];
        unpack_row_bf16<W>(gamma_bits, gm);
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] = fmaf(gm[i] * rs, v[i], __uint_as_float(in.x[i]));
      } else {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] = fmaf(rs, v[i], __uint_as_float(in.x[i]));
      }
      store_row_f32<W>(reinterpret_cast<float*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    case IVB_EPI_GELU_BWD: {
      // out0(bf16) = acc * gelu'(aux(bf16 pre-activation))   [or acc * aux with GELU_SAVE_GRAD]
      float hv[W];
      unpack_row_bf16<W>(in.x, hv);
      if (save_grad) {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= hv[i];
      } else if (tanh_mode) {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= gelu_tanh_grad(hv[i]);
      } else if (quick_mode) {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= gelu_quick_grad(hv[i]);
      } else {
#pragma unroll
        for (int i = 0; i < W; ++i) v[i] *= gelu_erf_grad(hv[i]);
      }
      store_row_bf16<W>(reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + col0, v, nvalid);
    } break;
    case IVB_EPI_SWIGLU: if constexpr (SWIGLU) {
      // The B tile interleaves gate and up rows in groups of 8 (ivb_gemm.cu, launch_gemm), so each 16 columns of the
      // segment are the gate (v[i .. i+8)) and up (v[i+8 .. i+16)) products of the 8 output columns from (col0 + i) / 2:
      // out0(bf16) [M, N/2] = silu(gate) * up, one 16-byte piece each.
#pragma unroll
      for (int i = 0; i < W; i += 16) {
        if (i >= nvalid) break;
        uint32_t r[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          r[k] = pack_bf16(silu(v[i + 2 * k]) * v[i + 8 + 2 * k], silu(v[i + 2 * k + 1]) * v[i + 9 + 2 * k]);
        *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out0) + row * p.ld0 + (col0 + i) / 2) =
            make_uint4(r[0], r[1], r[2], r[3]);
      }
    } break;
    default:
      break;
  }
}

}  // namespace ivb
