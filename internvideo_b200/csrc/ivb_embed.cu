// ivb_embed.cu — the token front-end of the video ViT as coalesced HBM kernels:
//   * visible-token index list from the boolean mask (bit-exact `x[~mask]` order)
//       internvideo2_pretrain.py:659 ; InternVideo1/Pretrain/VideoMAE/modeling_pretrain.py:136
//   * tubelet im2col of the VISIBLE patches only (PatchEmbed Conv3d k=s=(t,p,p) as a gather-GEMM;
//     the reference embeds all T*L patches then discards 80 %)           internvideo2_pretrain.py:320-331
//   * gather-add of position tables (+cls) into the fp32 residual stream / decoder inputs
//       internvideo2_pretrain.py:635-656, 712-714, 735-737
//   * the scatter-add backward of those gathers.
#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

// One warp per clip: order-preserving compaction of the indices where mask == 0.
__global__ void visible_indices_kernel(const uint8_t* __restrict__ mask, int B, int N, int n_keep,
                                       int* __restrict__ idx, int* __restrict__ err) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  const uint8_t* m = mask + static_cast<long>(b) * N;
  int count = 0;
  for (int base = 0; base < N; base += 32) {
    const int i = base + lane;
    const bool vis = (i < N) && (m[i] == 0);
    const unsigned bal = __ballot_sync(0xffffffffu, vis);
    const int pos = count + __popc(bal & ((1u << lane) - 1u));
    if (vis && pos < n_keep) idx[static_cast<long>(b) * n_keep + pos] = i;
    count += __popc(bal);
  }
  if (count != n_keep) {
    // ragged mask: flag it (the host poisons the loss with NaN, no sync) and point the unwritten tail at a
    // valid patch token so the gathers that follow never index with uninitialised memory
    if (lane == 0) atomicExch(err, 1 + b);
    const int safe = N > 1 ? 1 : 0;
    for (int pos = count + lane; pos < n_keep; pos += 32) idx[static_cast<long>(b) * n_keep + pos] = safe;
  }
}

// im2col rows of the visible patch tokens.  video [B, C, T, H, W] bf16.  Row (b, j) <- token
// idx[b, j0 + j] (token t>=1 is patch t-1, ordered (frame, py, px)); K axis ordered (c, dt, dy, dx)
// like the Conv3d weight; K padded to Kpad with zeros.  One warp per row, 4-byte (2 x bf16) moves.
__global__ void im2col_visible_kernel(const __nv_bfloat16* __restrict__ video, const int* __restrict__ idx,
                                      int idx_stride, int j0, int rows_per_clip, int B, int C, int T,
                                      int H, int W, int tub, int P, int Kpad,
                                      __nv_bfloat16* __restrict__ cols) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const long total = static_cast<long>(B) * rows_per_clip;
  if (row >= total) return;
  const int b = static_cast<int>(row / rows_per_clip);
  const int j = static_cast<int>(row % rows_per_clip);
  const int tok = idx[static_cast<long>(b) * idx_stride + j0 + j] - 1;  // patch index
  const int gw = W / P, gh = H / P;
  const int f = tok / (gh * gw);
  const int py = (tok / gw) % gh;
  const int px = tok % gw;
  const int K = C * tub * P * P;
  const uint32_t* vid32 = reinterpret_cast<const uint32_t*>(video);
  uint32_t* dst = reinterpret_cast<uint32_t*>(cols + row * Kpad);
  const int halfP = P >> 1;
  for (int u = lane; u < (Kpad >> 1); u += 32) {
    uint32_t val = 0;
    const int e = u * 2;
    if (e < K) {
      const int dx = e % P;
      int rest = e / P;
      const int dy = rest % P; rest /= P;
      const int dt = rest % tub;
      const int c = rest / tub;
      const long src = (((static_cast<long>(b) * C + c) * T + (f * tub + dt)) * H + (py * P + dy)) * W +
                       (px * P + dx);
      val = vid32[src >> 1];
    }
    dst[u] = val;
  }
  (void)halfP;
}

// out[b, j, :] = (src ? src[b*src_bstride + j*D ..] : 0) + (table ? table[(idx[b*idx_bstride + j] + idx_off) * D ..] : 0)
template <bool OUT_F32>
__global__ void gather_add_kernel(const float* __restrict__ src, long src_bstride,
                                  const __nv_bfloat16* __restrict__ table, const int* __restrict__ idx,
                                  int idx_bstride, int idx_off, int B, int rows, int D, void* out,
                                  long out_bstride) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<long>(B) * rows) return;
  const int b = static_cast<int>(row / rows);
  const int j = static_cast<int>(row % rows);
  const float* s = src ? src + b * src_bstride + static_cast<long>(j) * D : nullptr;
  const __nv_bfloat16* t = nullptr;
  if (table) {
    const int ti = (idx ? idx[static_cast<long>(b) * idx_bstride + j] : j) + idx_off;
    t = table + static_cast<long>(ti) * D;
  }
  for (int c = lane * 8; c < D; c += 256) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
    if (s) {
      float4 a = *reinterpret_cast<const float4*>(s + c), bb = *reinterpret_cast<const float4*>(s + c + 4);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = bb.x; v[5] = bb.y; v[6] = bb.z; v[7] = bb.w;
    }
    if (t) {
      uint4 u = *reinterpret_cast<const uint4*>(t + c);
      float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
      v[0] += f0.x; v[1] += f0.y; v[2] += f1.x; v[3] += f1.y; v[4] += f2.x; v[5] += f2.y; v[6] += f3.x; v[7] += f3.y;
    }
    if (OUT_F32) {
      float* o = reinterpret_cast<float*>(out) + b * out_bstride + static_cast<long>(j) * D + c;
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out) + b * out_bstride + static_cast<long>(j) * D + c;
      uint4 w;
      w.x = pack_bf16(v[0], v[1]); w.y = pack_bf16(v[2], v[3]);
      w.z = pack_bf16(v[4], v[5]); w.w = pack_bf16(v[6], v[7]);
      *reinterpret_cast<uint4*>(o) = w;
    }
  }
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// table_grad[(idx[b, j] + idx_off), :] += g[b, j, :]   (fp32 atomics; g is fp32 or bf16)
template <bool G_F32>
__global__ void scatter_add_kernel(const void* __restrict__ g, long g_bstride, const int* __restrict__ idx,
                                   int idx_bstride, int idx_off, int B, int rows, int D,
                                   float* __restrict__ table_grad) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<long>(B) * rows) return;
  const int b = static_cast<int>(row / rows);
  const int j = static_cast<int>(row % rows);
  const int ti = (idx ? idx[static_cast<long>(b) * idx_bstride + j] : j) + idx_off;
  float* dst = table_grad + static_cast<long>(ti) * D;
  for (int c = lane * 8; c < D; c += 256) {
    float v[8];
    if (G_F32) {
      const float* s = reinterpret_cast<const float*>(g) + b * g_bstride + static_cast<long>(j) * D + c;
      float4 a = *reinterpret_cast<const float4*>(s), bb = *reinterpret_cast<const float4*>(s + 4);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = bb.x; v[5] = bb.y; v[6] = bb.z; v[7] = bb.w;
    } else {
      const __nv_bfloat16* s = reinterpret_cast<const __nv_bfloat16*>(g) + b * g_bstride + static_cast<long>(j) * D + c;
      uint4 u = *reinterpret_cast<const uint4*>(s);
      float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
      v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y; v[4] = f2.x; v[5] = f2.y; v[6] = f3.x; v[7] = f3.y;
    }
    // two 128-bit vector reductions per 8 columns (red.global.add.v4.f32, sm_90+): a quarter of the atomic
    // operations of scalar atomicAdd — the scalar form ran at 0.12 of the HBM rate (18.8 M atomics per call)
    red_add_v4(dst + c, v[0], v[1], v[2], v[3]);
    red_add_v4(dst + c + 4, v[4], v[5], v[6], v[7]);
  }
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_visible_indices(const void* mask_u8, int B, int N, int n_keep, int* idx,
                                   int* err_flag, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0) return 0;
  const int wpb = 4;
  visible_indices_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, stream>>>(
      reinterpret_cast<const uint8_t*>(mask_u8), B, N, n_keep, idx, err_flag);
  count_launch();
  return check_launch("visible_indices_kernel");
}

extern "C" int ivb_im2col_visible(const void* video, const int* idx, int idx_stride, int j0,
                                  int rows_per_clip, int B, int C, int T, int H, int W, int tubelet,
                                  int patch, int Kpad, void* cols, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows_per_clip <= 0) return 0;
  if ((patch & 1) || (W & 1) || (Kpad & 7) || Kpad < C * tubelet * patch * patch)
    return set_error("ivb_im2col_visible: patch/W must be even, Kpad a multiple of 8 and >= C*t*p*p");
  const long rows = static_cast<long>(B) * rows_per_clip;
  const int wpb = 8;
  im2col_visible_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(video), idx, idx_stride, j0, rows_per_clip, B, C, T, H, W,
      tubelet, patch, Kpad, reinterpret_cast<__nv_bfloat16*>(cols));
  count_launch();
  return check_launch("im2col_visible_kernel");
}

extern "C" int ivb_gather_add(const float* src, long src_bstride, const void* table, const int* idx,
                              int idx_bstride, int idx_off, int B, int rows, int D, void* out,
                              int out_is_f32, long out_bstride, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows <= 0) return 0;
  if (D & 7) return set_error("ivb_gather_add: D must be a multiple of 8");
  const long total = static_cast<long>(B) * rows;
  const int wpb = 8;
  const unsigned grid = (unsigned)((total + wpb - 1) / wpb);
  const __nv_bfloat16* t = reinterpret_cast<const __nv_bfloat16*>(table);
  if (out_is_f32)
    gather_add_kernel<true><<<grid, wpb * 32, 0, stream>>>(src, src_bstride, t, idx, idx_bstride, idx_off, B, rows, D, out, out_bstride);
  else
    gather_add_kernel<false><<<grid, wpb * 32, 0, stream>>>(src, src_bstride, t, idx, idx_bstride, idx_off, B, rows, D, out, out_bstride);
  count_launch();
  return check_launch("gather_add_kernel");
}

extern "C" int ivb_scatter_add(const void* g, int g_is_f32, long g_bstride, const int* idx,
                               int idx_bstride, int idx_off, int B, int rows, int D,
                               float* table_grad, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows <= 0) return 0;
  if (D & 7) return set_error("ivb_scatter_add: D must be a multiple of 8");
  // One launch per clip, in clip order: the rows of one clip name distinct table rows, so every table row receives its
  // contributions in the same order on every run (one launch over all clips would add them in whatever order the
  // clips' warps arrive, and the table's AdamW update would differ from run to run).
  const int wpb = 8;
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  const char* gb = reinterpret_cast<const char*>(g);
  const long gstep = g_bstride * (g_is_f32 ? 4 : 2);
  for (int b = 0; b < B; ++b) {
    const int* ib = idx ? idx + static_cast<long>(b) * idx_bstride : nullptr;
    if (g_is_f32)
      scatter_add_kernel<true><<<grid, wpb * 32, 0, stream>>>(gb + b * gstep, g_bstride, ib, idx_bstride, idx_off, 1, rows, D, table_grad);
    else
      scatter_add_kernel<false><<<grid, wpb * 32, 0, stream>>>(gb + b * gstep, g_bstride, ib, idx_bstride, idx_off, 1, rows, D, table_grad);
    count_launch();
    if (int rc = check_launch("scatter_add_kernel")) return rc;
  }
  return 0;
}
