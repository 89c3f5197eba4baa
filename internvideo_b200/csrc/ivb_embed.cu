// ivb_embed.cu — the token front-end of the video ViT as coalesced HBM kernels:
//   * visible-token index list from the boolean mask (bit-exact `x[~mask]` order)
//       internvideo2_pretrain.py:659 ; InternVideo1/Pretrain/VideoMAE/modeling_pretrain.py:136
//   * tubelet im2col of the VISIBLE patches only (PatchEmbed Conv3d k=s=(t,p,p) as a gather-GEMM;
//     the reference embeds all T*L patches then discards 80 %)           internvideo2_pretrain.py:320-331
//   * gather-add of position tables (+cls) into the fp32 residual stream / decoder inputs
//       internvideo2_pretrain.py:635-656, 712-714, 735-737
//   * the scatter-add backward of those gathers
//   * the token embedding of the MobileCLIP text tower (text_encoder.py:131-147) and its backward, whose table gradient
//     sums each id's rows in a fixed order through a device counting sort of the positions by id.
#include "ivb_internal.h"
#include "ivb_ptx.cuh"
#include "ivb_rows.cuh"

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
    float v[8] = {};
    if (s) load8<true>(s, c, v);
    if (t) {
      float tv[8];
      load8<false>(t, c, tv);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] += tv[k];
    }
    store8<OUT_F32>(out, b * out_bstride + static_cast<long>(j) * D + c, v);
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
    load8<G_F32>(g, b * g_bstride + static_cast<long>(j) * D + c, v);
    // two 128-bit vector reductions per 8 columns (red.global.add.v4.f32, sm_90+): a quarter of the atomic
    // operations of scalar atomicAdd — the scalar form ran at 0.12 of the HBM rate (18.8 M atomics per call)
    red_add_v4(dst + c, v[0], v[1], v[2], v[3]);
    red_add_v4(dst + c + 4, v[4], v[5], v[6], v[7]);
  }
}


// ------------------------------------------------------------------ text-tower token embedding
// out[b*L + l] = E[ids[b, l]] + P[l] (fp32), one warp per row.  An id outside [0, V) sets *err to 1 + the row and reads
// row 0 instead, so nothing reads out of bounds; the backward treats it the same way.
__device__ __forceinline__ int token_id(const long long* ids, long row, int V) {
  const long long id = ids[row];
  return id < 0 || id >= V ? 0 : static_cast<int>(id);
}

__global__ void token_embed_fwd_kernel(const long long* __restrict__ ids, int B, int L,
                                       const __nv_bfloat16* __restrict__ E, int V, const __nv_bfloat16* __restrict__ P,
                                       int D, float* __restrict__ out, long ldo, int* __restrict__ err) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<long>(B) * L) return;
  if (lane == 0 && (ids[row] < 0 || ids[row] >= V)) atomicExch(err, static_cast<int>(1 + row));
  const __nv_bfloat16* e = E + static_cast<long>(token_id(ids, row, V)) * D;
  const __nv_bfloat16* pl = P + static_cast<long>(row % L) * D;
  for (int c = lane * 8; c < D; c += 256) {
    float v[8], pv[8];
    load8<false>(e, c, v);
    load8<false>(pl, c, pv);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] += pv[k];
    store8<true>(out, row * ldo + c, v);
  }
}

// The backward sorts the N = B*L positions by id, stably, in the int32 workspace [count V | start V | rank N | sorted N]:
// count[v] = occurrences of v (integer atomics: exact), start = its exclusive prefix sum (one CTA), rank[p] = the
// positions before p with p's id, sorted[start[id] + rank] = p.  Then the first occurrence of each id sums that id's
// gradient rows in position order, so the same ids and gradient give the same bits on every run.
__global__ void token_count_kernel(const long long* __restrict__ ids, int N, int V, int* __restrict__ count) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < N) atomicAdd(count + token_id(ids, p, V), 1);
}

constexpr int TOK_SCAN_THREADS = 1024;

__global__ void __launch_bounds__(TOK_SCAN_THREADS) token_scan_kernel(const int* __restrict__ count, int V,
                                                                      int* __restrict__ start) {
  __shared__ int part[TOK_SCAN_THREADS];
  const int per = (V + TOK_SCAN_THREADS - 1) / TOK_SCAN_THREADS, v0 = threadIdx.x * per, v1 = min(V, v0 + per);
  int sum = 0;
  for (int v = v0; v < v1; ++v) sum += count[v];
  part[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < TOK_SCAN_THREADS; off <<= 1) {   // inclusive Hillis-Steele scan of the thread sums
    const int add = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += add;
    __syncthreads();
  }
  int run = part[threadIdx.x] - sum;
  for (int v = v0; v < v1; ++v) {
    start[v] = run;
    run += count[v];
  }
}

constexpr int TOK_RANK_THREADS = 256;

__global__ void __launch_bounds__(TOK_RANK_THREADS) token_rank_kernel(const long long* __restrict__ ids, int N, int V,
                                                                      const int* __restrict__ start,
                                                                      int* __restrict__ rank, int* __restrict__ sorted) {
  __shared__ int tile[TOK_RANK_THREADS];
  const int p = blockIdx.x * TOK_RANK_THREADS + threadIdx.x;
  const int id = p < N ? token_id(ids, p, V) : -1;
  int r = 0;
  for (int t0 = 0; t0 <= static_cast<int>(blockIdx.x) * TOK_RANK_THREADS; t0 += TOK_RANK_THREADS) {
    __syncthreads();
    tile[threadIdx.x] = t0 + threadIdx.x < N ? token_id(ids, t0 + threadIdx.x, V) : -2;
    __syncthreads();
    const int lim = min(TOK_RANK_THREADS, p - t0);   // positions t0 + i < p
    for (int i = 0; i < lim; ++i) r += tile[i] == id;
  }
  if (p < N) {
    rank[p] = r;
    sorted[start[id] + r] = p;
  }
}

// dE[v] = the sum of g over the positions of id v in position order, by one warp per position that is its id's first
// occurrence; the other rows of dE are not written.
__global__ void token_table_grad_kernel(const long long* __restrict__ ids, int N, int V, const float* __restrict__ g,
                                        long ldg, int D, const int* __restrict__ count, const int* __restrict__ start,
                                        const int* __restrict__ rank, const int* __restrict__ sorted,
                                        float* __restrict__ dE) {
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= N || rank[p] != 0) return;
  const int id = token_id(ids, p, V), s0 = start[id], cnt = count[id];
  for (int c = lane * 8; c < D; c += 256) {
    float acc[8] = {};
    for (int k = 0; k < cnt; ++k) {
      float v[8];
      load8<true>(g, static_cast<long>(sorted[s0 + k]) * ldg + c, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += v[e];
    }
    store8<true>(dE, static_cast<long>(id) * D + c, acc);
  }
}

// dP[l] = sum over b = 0, 1, .. B-1 of g[b*L + l]: one thread per (l, 4 columns), clips in order.
__global__ void token_pos_grad_kernel(const float* __restrict__ g, long ldg, int B, int L, int D,
                                      float* __restrict__ dP) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int q = D / 4;
  if (i >= static_cast<long>(L) * q) return;
  const int l = static_cast<int>(i / q), c = static_cast<int>(i % q) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int b = 0; b < B; ++b) {
    const float4 v = *reinterpret_cast<const float4*>(g + (static_cast<long>(b) * L + l) * ldg + c);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  *reinterpret_cast<float4*>(dP + static_cast<long>(l) * D + c) = acc;
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_visible_indices(const void* mask_u8, int B, int N, int n_keep, int* idx,
                                   int* err_flag, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0) return 0;
  const int wpb = 4;
  return launch("visible_indices_kernel", visible_indices_kernel, (B + wpb - 1) / wpb, wpb * 32, 0, stream, NO_PDL,
                reinterpret_cast<const uint8_t*>(mask_u8), B, N, n_keep, idx, err_flag);
}

extern "C" int ivb_im2col_visible(const void* video, const int* idx, int idx_stride, int j0,
                                  int rows_per_clip, int B, int C, int T, int H, int W, int tubelet,
                                  int patch, int Kpad, void* cols, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows_per_clip <= 0) return 0;
  if ((patch & 1) || (W & 1) || (Kpad & 7) || Kpad < C * tubelet * patch * patch)
    return set_error("ivb_im2col_visible: patch/W must be even, Kpad a multiple of 8 and >= C*t*p*p");
  if (misaligned(4, video, cols)) return set_error("ivb_im2col_visible: video and cols must be 4-byte aligned");
  const long rows = static_cast<long>(B) * rows_per_clip;
  const int wpb = 8;
  return launch("im2col_visible_kernel", im2col_visible_kernel, (unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, stream,
                NO_PDL, reinterpret_cast<const __nv_bfloat16*>(video), idx, idx_stride, j0, rows_per_clip, B, C, T, H, W,
                tubelet, patch, Kpad, reinterpret_cast<__nv_bfloat16*>(cols));
}

extern "C" int ivb_gather_add(const float* src, long src_bstride, const void* table, const int* idx,
                              int idx_bstride, int idx_off, int B, int rows, int D, void* out,
                              int out_is_f32, long out_bstride, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows <= 0) return 0;
  if (D & 7) return set_error("ivb_gather_add: D must be a multiple of 8");
  if ((src_bstride & 7) || (out_bstride & 7))
    return set_error("ivb_gather_add: src_bstride and out_bstride must be multiples of 8");
  if (misaligned(16, src, table, out)) return set_error("ivb_gather_add: src, table and out must be 16-byte aligned");
  const long total = static_cast<long>(B) * rows;
  const int wpb = 8;
  const unsigned grid = (unsigned)((total + wpb - 1) / wpb);
  const __nv_bfloat16* t = reinterpret_cast<const __nv_bfloat16*>(table);
  return launch("gather_add_kernel", out_is_f32 ? gather_add_kernel<true> : gather_add_kernel<false>, grid, wpb * 32, 0,
                stream, NO_PDL, src, src_bstride, t, idx, idx_bstride, idx_off, B, rows, D, out, out_bstride);
}

extern "C" int ivb_scatter_add(const void* g, int g_is_f32, long g_bstride, const int* idx,
                               int idx_bstride, int idx_off, int B, int rows, int D,
                               float* table_grad, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows <= 0) return 0;
  if (D & 7) return set_error("ivb_scatter_add: D must be a multiple of 8");
  if (g_bstride & 7) return set_error("ivb_scatter_add: g_bstride must be a multiple of 8");
  if (misaligned(16, g, table_grad)) return set_error("ivb_scatter_add: g and table_grad must be 16-byte aligned");
  // One launch per clip, in clip order: the rows of one clip name distinct table rows, so every table row receives its
  // contributions in the same order on every run (one launch over all clips would add them in whatever order the
  // clips' warps arrive, and the table's AdamW update would differ from run to run).
  const int wpb = 8;
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  const char* gb = reinterpret_cast<const char*>(g);
  const long gstep = g_bstride * (g_is_f32 ? 4 : 2);
  const auto kern = g_is_f32 ? scatter_add_kernel<true> : scatter_add_kernel<false>;
  for (int b = 0; b < B; ++b) {
    const int* ib = idx ? idx + static_cast<long>(b) * idx_bstride : nullptr;
    if (int rc = launch("scatter_add_kernel", kern, grid, wpb * 32, 0, stream, NO_PDL, gb + b * gstep, g_bstride, ib,
                        idx_bstride, idx_off, 1, rows, D, table_grad))
      return rc;
  }
  return 0;
}

extern "C" int ivb_token_embed_fwd(const long long* ids, int B, int L, const void* table, int V, const void* pos, int D,
                                   float* out, long ldo, int* err_flag, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || L <= 0) return 0;
  if (V <= 0 || (D & 7) || D <= 0 || (ldo & 7) || ldo < D)
    return set_error("ivb_token_embed_fwd: V > 0, D and ldo multiples of 8, ldo >= D");
  if (misaligned(16, table, pos, out)) return set_error("ivb_token_embed_fwd: table, pos and out must be 16-byte aligned");
  if (misaligned(8, ids) || misaligned(4, err_flag) || err_flag == nullptr)
    return set_error("ivb_token_embed_fwd: ids must be 8-byte aligned and err_flag a 4-byte aligned int");
  const long rows = static_cast<long>(B) * L;
  const int wpb = 8;
  return launch("token_embed_fwd_kernel", token_embed_fwd_kernel, (unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0,
                stream, NO_PDL, ids, B, L, reinterpret_cast<const __nv_bfloat16*>(table), V,
                reinterpret_cast<const __nv_bfloat16*>(pos), D, out, ldo, err_flag);
}

extern "C" long ivb_token_embed_bwd_workspace_ints(int V, int B, int L) {
  return 2L * V + 2L * B * L;
}

extern "C" int ivb_token_embed_bwd(const long long* ids, int B, int L, const float* g, long ldg, int V, int D,
                                   float* dtable, float* dpos, int* ws, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || L <= 0) return 0;
  if (V <= 0 || (D & 7) || D <= 0 || (ldg & 7) || ldg < D)
    return set_error("ivb_token_embed_bwd: V > 0, D and ldg multiples of 8, ldg >= D");
  if (misaligned(16, g, dtable, dpos)) return set_error("ivb_token_embed_bwd: g, dtable and dpos must be 16-byte aligned");
  if (misaligned(8, ids) || misaligned(4, ws) || ws == nullptr)
    return set_error("ivb_token_embed_bwd: ids must be 8-byte aligned and ws a 4-byte aligned int workspace");
  const long N = static_cast<long>(B) * L;
  if (N > (1L << 30)) return set_error("ivb_token_embed_bwd: B*L must fit the int32 position lists");
  int* count = ws;
  int* start = ws + V;
  int* rank = start + V;
  int* sorted = rank + N;
  const int n = static_cast<int>(N);
  int rc;
  if (cudaError_t e = cudaMemsetAsync(count, 0, static_cast<size_t>(V) * sizeof(int), stream))
    return set_error_cuda("cudaMemsetAsync(token_embed_bwd count)", e);
  if ((rc = launch("token_count_kernel", token_count_kernel, (unsigned)((N + 255) / 256), 256, 0, stream, NO_PDL, ids, n,
                   V, count)) ||
      (rc = launch("token_scan_kernel", token_scan_kernel, 1, TOK_SCAN_THREADS, 0, stream, NO_PDL,
                   static_cast<const int*>(count), V, start)) ||
      (rc = launch("token_rank_kernel", token_rank_kernel, (unsigned)((N + TOK_RANK_THREADS - 1) / TOK_RANK_THREADS),
                   TOK_RANK_THREADS, 0, stream, NO_PDL, ids, n, V, static_cast<const int*>(start), rank, sorted)))
    return rc;
  const int wpb = 8;
  if ((rc = launch("token_table_grad_kernel", token_table_grad_kernel, (unsigned)((N + wpb - 1) / wpb), wpb * 32, 0,
                   stream, NO_PDL, ids, n, V, g, ldg, D, static_cast<const int*>(count),
                   static_cast<const int*>(start), static_cast<const int*>(rank), static_cast<const int*>(sorted), dtable)))
    return rc;
  const long threads = static_cast<long>(L) * (D / 4);
  return launch("token_pos_grad_kernel", token_pos_grad_kernel, (unsigned)((threads + 255) / 256), 256, 0, stream,
                NO_PDL, g, ldg, B, L, D, dpos);
}
