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
#include <cstdio>

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

// ------------------------------------------------------------------ pre-norm im2col (dual-RMSNorm patch embed)
// InternVideo-Next's PatchEmbed (InternVideo_next.py:302-342) applies an RMSNorm (`norm_before`) to each patch's
// K = C*t*p*p raw pixels before the Conv3d.  Its weight is indexed in the reference's `(t hp wp c)` order, so the
// column (c, dt, dy, dx) of a row meets weight element pi(c, dt, dy, dx) = ((dt*p + dy)*p + dx)*C + c.  A warp holds
// its row's pixels in registers (word u = lane + 32 i, two pixels per word), so each pixel is read from HBM once.
constexpr int PRENORM_MAX_KPAD = 1536;
constexpr int PRENORM_NU = PRENORM_MAX_KPAD / 64;     // 2-pixel words per lane

struct PatchRow {
  int b, f, py, px;
};

__device__ __forceinline__ PatchRow patch_row(const int* idx, int idx_stride, int j0, int rows_per_clip, long row,
                                              int H, int W, int P) {
  const int b = static_cast<int>(row / rows_per_clip);
  const int j = static_cast<int>(row % rows_per_clip);
  const int tok = idx[static_cast<long>(b) * idx_stride + j0 + j] - 1;
  const int gw = W / P, gh = H / P;
  return {b, tok / (gh * gw), (tok / gw) % gh, tok % gw};
}

// Video element of column e (even: dx and dx + 1 share one 4-byte word) and pi(e); pi(e + 1) = pi(e) + C.
__device__ __forceinline__ long prenorm_col(const PatchRow& r, int e, int C, int T, int H, int W, int tub, int P,
                                            int* wi) {
  const int dx = e % P;
  int rest = e / P;
  const int dy = rest % P; rest /= P;
  const int dt = rest % tub;
  const int c = rest / tub;
  *wi = ((dt * P + dy) * P + dx) * C + c;
  return (((static_cast<long>(r.b) * C + c) * T + (r.f * tub + dt)) * H + (r.py * P + dy)) * W + (r.px * P + dx);
}

__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// Loads the row's pixel words into v (zero past K) and returns r = rsqrt(mean a^2 + eps), the same in every lane
// (a butterfly sum: the same bits on every run).
__device__ __forceinline__ float prenorm_load(const uint32_t* vid32, const PatchRow& pr, int C, int T, int H, int W,
                                              int tub, int P, int K, float eps, int lane, uint32_t v[PRENORM_NU]) {
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < PRENORM_NU; ++i) {
    const int e = (lane + 32 * i) * 2;
    v[i] = 0u;
    if (e < K) {
      int wi;
      v[i] = vid32[prenorm_col(pr, e, C, T, H, W, tub, P, &wi) >> 1];
      const float2 a = unpack_bf16(v[i]);
      ss = fmaf(a.x, a.x, fmaf(a.y, a.y, ss));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  return rsqrtf(ss / static_cast<float>(K) + eps);
}

// cols[row, e] = bf16(w[pi(e)] * bf16(a_e * r)), zero for K <= e < Kpad; rstd[row] = r.  Rows as im2col_visible_kernel.
__global__ void im2col_prenorm_kernel(const __nv_bfloat16* __restrict__ video, const int* __restrict__ idx,
                                      int idx_stride, int j0, int rows_per_clip, int B, int C, int T, int H, int W,
                                      int tub, int P, int Kpad, const __nv_bfloat16* __restrict__ weight, float eps,
                                      __nv_bfloat16* __restrict__ cols, float* __restrict__ rstd) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= static_cast<long>(B) * rows_per_clip) return;
  const PatchRow pr = patch_row(idx, idx_stride, j0, rows_per_clip, row, H, W, P);
  const int K = C * tub * P * P;
  uint32_t v[PRENORM_NU];
  const float r = prenorm_load(reinterpret_cast<const uint32_t*>(video), pr, C, T, H, W, tub, P, K, eps, lane, v);
  uint32_t* dst = reinterpret_cast<uint32_t*>(cols + row * Kpad);
#pragma unroll
  for (int i = 0; i < PRENORM_NU; ++i) {
    const int u = lane + 32 * i;
    if (u >= (Kpad >> 1)) break;
    uint32_t val = 0u;
    if (2 * u < K) {
      int wi;
      prenorm_col(pr, 2 * u, C, T, H, W, tub, P, &wi);
      const float2 a = unpack_bf16(v[i]);
      val = pack_bf16(__bfloat162float(weight[wi]) * bf16_round(a.x * r),
                      __bfloat162float(weight[wi + C]) * bf16_round(a.y * r));
    }
    dst[u] = val;
  }
  if (lane == 0) rstd[row] = r;
}

// Weight gradient of norm_before: dw[pi(e)] = sum over rows of dcols[row, e] * bf16(a_e * rstd[row]), the normalised
// pixels recomputed from the video (cols cannot give them back: w may hold zeros).  CTA c takes rows
// [c * PRENORM_WG_ROWS, (c + 1) * PRENORM_WG_ROWS); warp k of it adds rows k, k + 8, ... in order in registers, the
// warps are added in warp order, and the CTA's K sums go to slot c of the fixed-order column scratch (ivb_colred.cuh),
// whose slots the host then adds in slot order.
constexpr int PRENORM_WG_WARPS = 8, PRENORM_WG_ROWS = 128;

__global__ void __launch_bounds__(PRENORM_WG_WARPS * 32)
    prenorm_wgrad_kernel(const __nv_bfloat16* __restrict__ video, const int* __restrict__ idx, int idx_stride, int j0,
                         int rows_per_clip, int B, int C, int T, int H, int W, int tub, int P, int Kpad,
                         const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dcols, long lddc,
                         float* __restrict__ slots) {
  extern __shared__ float part[];      // [warp][Kpad]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int K = C * tub * P * P;
  const long total = static_cast<long>(B) * rows_per_clip;
  const long r0 = static_cast<long>(blockIdx.x) * PRENORM_WG_ROWS;
  const long r1 = min(total, r0 + PRENORM_WG_ROWS);
  const uint32_t* vid32 = reinterpret_cast<const uint32_t*>(video);
  float acc[2 * PRENORM_NU];
#pragma unroll
  for (int i = 0; i < 2 * PRENORM_NU; ++i) acc[i] = 0.f;
  for (long row = r0 + warp; row < r1; row += PRENORM_WG_WARPS) {
    const PatchRow pr = patch_row(idx, idx_stride, j0, rows_per_clip, row, H, W, P);
    const float r = rstd[row];
    const uint32_t* dc = reinterpret_cast<const uint32_t*>(dcols + row * lddc);
#pragma unroll
    for (int i = 0; i < PRENORM_NU; ++i) {
      const int e = (lane + 32 * i) * 2;
      if (e < K) {
        int wi;
        const float2 a = unpack_bf16(vid32[prenorm_col(pr, e, C, T, H, W, tub, P, &wi) >> 1]);
        const float2 g = unpack_bf16(dc[lane + 32 * i]);
        acc[2 * i] = fmaf(g.x, bf16_round(a.x * r), acc[2 * i]);
        acc[2 * i + 1] = fmaf(g.y, bf16_round(a.y * r), acc[2 * i + 1]);
      }
    }
  }
  float* mine = part + static_cast<long>(warp) * Kpad;
#pragma unroll
  for (int i = 0; i < PRENORM_NU; ++i) {
    const int e = (lane + 32 * i) * 2;
    if (e < K) {
      mine[e] = acc[2 * i];
      mine[e + 1] = acc[2 * i + 1];
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < K; e += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < PRENORM_WG_WARPS; ++k) s += part[static_cast<long>(k) * Kpad + e];
    const int dx = e % P;
    int rest = e / P;
    const int dy = rest % P; rest /= P;
    const int dt = rest % tub;
    slots[static_cast<long>(blockIdx.x) * K + ((dt * P + dy) * P + dx) * C + rest / tub] = s;
  }
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

// The operand rules the two pre-norm entry points share; fn names the entry point in messages.
static int check_prenorm(const char* fn, const void* video, const int* idx, int C, int W, int tubelet, int patch,
                         int Kpad, const float* rstd) {
  char msg[160];
  const char* what = nullptr;
  if (C <= 0 || tubelet <= 0 || patch <= 0 || (patch & 1) || (W & 1))
    what = "C, tubelet and patch must be positive, patch and W even";
  else if ((Kpad & 7) || Kpad < C * tubelet * patch * patch || Kpad > PRENORM_MAX_KPAD)
    what = "Kpad must be a multiple of 8, >= C*t*p*p and <= 1536";
  else if (video == nullptr || idx == nullptr || rstd == nullptr)
    what = "video, idx and rstd must not be null";
  else if (misaligned(4, video, idx, rstd))
    what = "video, idx and rstd must be 4-byte aligned";
  if (what == nullptr) return 0;
  snprintf(msg, sizeof(msg), "%s: %s", fn, what);
  return set_error(msg);
}

extern "C" int ivb_im2col_prenorm(const void* video, const int* idx, int idx_stride, int j0, int rows_per_clip, int B,
                                  int C, int T, int H, int W, int tubelet, int patch, int Kpad, const void* weight,
                                  float eps, void* cols, float* rstd, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows_per_clip <= 0) return 0;
  if (int rc = check_prenorm("ivb_im2col_prenorm", video, idx, C, W, tubelet, patch, Kpad, rstd)) return rc;
  if (weight == nullptr || cols == nullptr) return set_error("ivb_im2col_prenorm: weight and cols must not be null");
  if (misaligned(4, cols) || misaligned(2, weight))
    return set_error("ivb_im2col_prenorm: cols must be 4-byte and weight 2-byte aligned");
  const long rows = static_cast<long>(B) * rows_per_clip;
  const int wpb = 8;
  return launch("im2col_prenorm_kernel", im2col_prenorm_kernel, (unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0,
                stream, NO_PDL, reinterpret_cast<const __nv_bfloat16*>(video), idx, idx_stride, j0, rows_per_clip, B, C,
                T, H, W, tubelet, patch, Kpad, reinterpret_cast<const __nv_bfloat16*>(weight), eps,
                reinterpret_cast<__nv_bfloat16*>(cols), rstd);
}

extern "C" int ivb_prenorm_wgrad(const void* video, const int* idx, int idx_stride, int j0, int rows_per_clip, int B,
                                 int C, int T, int H, int W, int tubelet, int patch, int Kpad, const float* rstd,
                                 const void* dcols, long lddc, float* dweight, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || rows_per_clip <= 0) return 0;
  if (int rc = check_prenorm("ivb_prenorm_wgrad", video, idx, C, W, tubelet, patch, Kpad, rstd)) return rc;
  if (dcols == nullptr || dweight == nullptr) return set_error("ivb_prenorm_wgrad: dcols and dweight must not be null");
  if ((lddc & 7) || lddc < Kpad) return set_error("ivb_prenorm_wgrad: lddc must be a multiple of 8 and >= Kpad");
  if (misaligned(4, dcols, dweight)) return set_error("ivb_prenorm_wgrad: dcols and dweight must be 4-byte aligned");
  const int K = C * tubelet * patch * patch;
  const long rows = static_cast<long>(B) * rows_per_clip;
  const long nslots = (rows + PRENORM_WG_ROWS - 1) / PRENORM_WG_ROWS;
  float* slots = colred_cols(nslots, K, "ivb_prenorm_wgrad: gradient scratch too small");
  if (slots == nullptr) return 1;
  const size_t smem = static_cast<size_t>(PRENORM_WG_WARPS) * Kpad * sizeof(float);
  if (int rc = launch("prenorm_wgrad_kernel", prenorm_wgrad_kernel, (unsigned)nslots, PRENORM_WG_WARPS * 32, smem,
                      stream, NO_PDL, reinterpret_cast<const __nv_bfloat16*>(video), idx, idx_stride, j0,
                      rows_per_clip, B, C, T, H, W, tubelet, patch, Kpad, rstd,
                      reinterpret_cast<const __nv_bfloat16*>(dcols), lddc, slots))
    return rc;
  return colred_cols_finish(static_cast<int>(nslots), K, dweight, stream);
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
