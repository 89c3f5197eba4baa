// ivb_attn.cuh — the pieces the attention forward (ivb_attn_fwd.cuh: bf16 kernels in ivb_attn.cu and
// ivb_attn_keylen.cu, the E4M3 kernel in ivb_attn_fp8.cu) and backward (ivb_attn_bwd.cu) kernels share: one CTA per
// (128-row block, head, clip) that streams 64-row tiles of the other operands through a ring.
#pragma once
#include <math.h>
#include <stdio.h>

#include <initializer_list>

#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

constexpr int ATT_ROWS = 128;     // rows owned by a CTA (two MMA warpgroups of 64)
constexpr int ATT_COLS = 64;      // rows of a streamed tile
constexpr int ATT_THREADS = 384;  // the producer warpgroup and the two MMA warpgroups

// The element type of the head rows a kernel loads: bf16 (64 columns per 128-byte atom) or E4M3 (128; the FP8 forward).
enum class AttnElt { BF16, E4M3 };

// 4-D TMA view of a [B*n, ld] projection buffer starting at `base`, box_tokens rows per load.  bf16: (d, head, token,
// clip); the head dim is its own axis, so the columns past d of a 64-column atom (d = 88) are out of bounds and land as
// zeros.  E4M3 (heads of d columns, d a multiple of 32): (H*d, 1, token, clip), a head addressed by its first column
// h*d; its 128-column box reads on into the next head's columns (out of bounds, zeros, after the last head).
template <AttnElt ELT = AttnElt::BF16>
inline int make_head_tmap(CUtensorMap* tm, const void* base, long ld, int B, int n, int H, int d, int box_tokens) {
  if constexpr (ELT == AttnElt::E4M3) {
    const uint64_t dims[4] = {(uint64_t)H * d, 1, (uint64_t)n, (uint64_t)B};
    const long strides[3] = {ld, ld, (long)n * ld};
    const uint32_t box[4] = {128, 1, (uint32_t)box_tokens, 1};
    return make_tmap_4d(tm, base, dims, strides, box, 1);
  }
  const uint64_t dims[4] = {(uint64_t)d, (uint64_t)H, (uint64_t)n, (uint64_t)B};
  const long strides[3] = {(long)d, ld, (long)n * ld};
  const uint32_t box[4] = {64, 1, (uint32_t)box_tokens, 1};
  return make_tmap_4d(tm, base, dims, strides, box);
}

extern __shared__ __align__(1024) uint8_t attn_smem[];

// Shared memory of a CTA (1024-byte aligned for the 128-byte swizzle): ROWS operands of the CTA's rows, two rings of NS
// streamed tiles, VECS rings of NS x 64 floats, then the barriers: `row`, BARS x NS `full` and BARS x NS `empty`.
template <int KA, int ROWS, int NS_, int VECS, int BARS_>
struct AttnSmem {
  static constexpr int NS = NS_, BARS = BARS_, VEC_BYTES = ATT_COLS * 4;
  static constexpr int ROW_BYTES = KA * ATT_ROWS * 128, TILE_BYTES = KA * ATT_COLS * 128;   // KA 64-column atoms
  static constexpr int RING = ROWS * ROW_BYTES, VEC = RING + 2 * NS * TILE_BYTES, BAR = VEC + VECS * NS * VEC_BYTES;
  static constexpr int BYTES = BAR + 128;
  static_assert((1 + 2 * BARS * NS) * 8 <= 128 && BYTES <= 227 * 1024, "attention: shared-memory budget");

  static __device__ __forceinline__ uint8_t* rows(int i) { return attn_smem + i * ROW_BYTES; }
  static __device__ __forceinline__ uint8_t* tile(int ring, int st) {
    return attn_smem + RING + (ring * NS + st) * TILE_BYTES;
  }
  static __device__ __forceinline__ float* vec(int v, int st) {
    return reinterpret_cast<float*>(attn_smem + VEC + (v * NS + st) * VEC_BYTES);
  }
  static __device__ __forceinline__ uint64_t* bar_row() { return reinterpret_cast<uint64_t*>(attn_smem + BAR); }
  static __device__ __forceinline__ uint64_t* full(int ring, int st) { return bar_row() + 1 + ring * NS + st; }
  static __device__ __forceinline__ uint64_t* empty(int ring, int st) { return bar_row() + 1 + (BARS + ring) * NS + st; }
};

// The j-th use of a ring of NS stages: its stage, and the parity the MMA warpgroups wait for on `full` (the producer
// waits for ph ^ 1 on `empty`, so a stage's first fill does not wait).
template <int NS>
struct RingSlot {
  int st;
  uint32_t ph;
  __device__ __forceinline__ explicit RingSlot(int j) : st(j % NS), ph((j / NS) & 1) {}
};

struct AttnCta {
  int warp, lane, wg, row0, h, b;  // row0: the CTA's first row; h: its head; b: its clip
  int nblk, live;  // streamed tiles; MMA warpgroups that own a row < n (each arrives once on an `empty`)
  int rloc;        // in an MMA warpgroup: this thread's accumulator rows of the CTA are rloc and rloc + 8
  bool signal;     // the thread that arrives on `empty` for its warpgroup
  bool dead;       // PLAN: the clip's DropPath factor is 0; the CTA only stores zero_rows
};

// PLAN (ivb_attn_fwd_plan, ivb_attn_bwd_plan): rowscale holds the attention branch's DropPath factors, one per clip
// repeated over its n rows.  The CTA of a clip whose factor is 0 returns `dead` before it initialises or waits on a
// barrier, so it issues no TMA and no MMA and every barrier count stays that of the live CTAs.  The factors may be
// written by the kernel before (PDL), so they are read after its wait.
template <class Smem, bool PLAN = false>
__device__ __forceinline__ AttnCta attn_prologue(int n, const float* rowscale = nullptr) {
  AttnCta c;
  const int tid = threadIdx.x;
  c.warp = tid >> 5; c.lane = tid & 31; c.wg = tid >> 7;
  c.row0 = blockIdx.x * ATT_ROWS; c.h = blockIdx.y; c.b = blockIdx.z;
  c.nblk = (n + ATT_COLS - 1) / ATT_COLS;
  c.live = min(2, (n - c.row0 + 63) / 64);
  c.rloc = (c.wg - 1) * 64 + (c.warp & 3) * 16 + (c.lane >> 2);
  c.signal = (tid & 127) == 0;
  c.dead = false;
  if constexpr (PLAN) {
    pdl_wait();
    c.dead = rowscale[static_cast<long>(c.b) * n] == 0.0f;
    if (c.dead) return c;
  }
  if (tid == 0) {
    if ((smem_u32(attn_smem) & 1023u) != 0) __trap();
    mbar_init(Smem::bar_row(), 1);
    for (int i = 0; i < Smem::NS; ++i) {
      for (int r = 0; r < Smem::BARS; ++r) mbar_init(Smem::full(r, i), 1);
      for (int r = 0; r < Smem::BARS; ++r) mbar_init(Smem::empty(r, i), c.live);
    }
    fence_mbar_init();
  }
  __syncthreads();
  return c;
}

// Warpgroup 0 gives its registers up and one elected thread runs produce(); each live MMA warpgroup cw takes them and
// runs consume(cw).
template <class Produce, class Consume>
__device__ __forceinline__ void attn_roles(const AttnCta& c, Produce&& produce, Consume&& consume) {
  if (c.wg == 0) {
    setmaxnreg_dec<24>();
    if (c.warp == 0 && elect_one()) produce();
  } else {
    setmaxnreg_inc<240>();
    const int cw = c.wg - 1;
    if (cw >= c.live) return;
    consume(cw);
  }
}

// TMA of rows [row, row + BOX) of head h of clip b (a make_head_tmap<ELT> view with a BOX-row box) into KA 128-byte
// atoms.  d: the E4M3 view's columns per head (make_head_tmap<E4M3>'s d), needed by that view only.
template <int KA, int BOX, AttnElt ELT = AttnElt::BF16>
__device__ __forceinline__ void load_head_rows(uint8_t* dst, const CUtensorMap* tm, int h, int row, int b,
                                               uint64_t* bar, int d = 0) {
#pragma unroll
  for (int a = 0; a < KA; ++a) {
    if constexpr (ELT == AttnElt::E4M3)
      tma_load_4d(dst + a * (BOX * 128), tm, h * d + a * 128, 0, row, b, bar);
    else
      tma_load_4d(dst + a * (BOX * 128), tm, a * 64, h, row, b, bar);
  }
}

// Quad reductions: the four threads (lane & 3) of a quad share an accumulator row.
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Online-softmax update of one S tile in place: S -> P = exp2(S*sc - m_new + P_SHIFT) (columns >= valid get 0); returns
// the rescale factor alpha = exp2(m_old - m_new) of each of the thread's two rows, and folds the row sums into l_run.
// P_SHIFT scales P (and l) by 2^P_SHIFT: the FP8 forward's E4M3 P keeps small probabilities in the normal range.
template <int P_SHIFT = 0>
__device__ __forceinline__ void softmax_tile(float (&s)[ATT_COLS / 2], int valid, int lane, float sc_log2,
                                             float m_run[2], float l_run[2], float alpha[2]) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < ATT_COLS / 2; ++i) {
    const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    float v = s[i] * sc_log2;
    if (col >= valid) v = -INFINITY;
    s[i] = v;
    mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float m_new = fmaxf(m_run[r], quad_max(mx[r]));
    alpha[r] = exp2f(m_run[r] - m_new);
    m_run[r] = m_new;
  }
  float rs[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < ATT_COLS / 2; ++i) {
    const int r = (i >> 1) & 1;
    if constexpr (P_SHIFT == 0)
      s[i] = exp2f(s[i] - m_run[r]);
    else
      s[i] = exp2f(s[i] - (m_run[r] - static_cast<float>(P_SHIFT)));
    rs[r] += s[i];
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + rs[r];
}

// Causal attention (ivb_attn_fwd_causal, ivb_attn_bwd_causal) keeps key <= query.  The streamed tiles a CTA needs:
// [causal_tile_begin, causal_tile_end).  With queries streamed (the dK/dV pass) they start at the first query tile that
// reaches the CTA's first key; with keys streamed (the forward and the dQ pass) they end at the tile that holds the
// CTA's last live query.  A 128-row CTA covers whole 64-row tiles, so the tile holding key == query is always streamed
// and every live row keeps at least one key.
static_assert(ATT_ROWS % ATT_COLS == 0, "causal tile bounds: a CTA's rows are whole streamed tiles");
__device__ __forceinline__ int causal_tile_begin(const AttnCta& c) { return c.row0 / ATT_COLS; }
__device__ __forceinline__ int causal_tile_end(const AttnCta& c, int n) {
  return (min(n, c.row0 + ATT_ROWS) + ATT_COLS - 1) / ATT_COLS;
}

// Causal mask of a 64 x 64 score tile in the accumulator layout softmax_tile reads: S = -inf where key > query, the
// reference's additive -inf upper triangle.  row0: the first row of this thread's fragment rows (the thread holds rows
// row0 and row0 + 8); col0: the tile's first column.  ROWS_ARE_KEYS: the tile is S^T (the dK/dV pass).
template <bool ROWS_ARE_KEYS>
__device__ __forceinline__ void causal_mask_tile(float (&s)[ATT_COLS / 2], int row0, int col0, int lane) {
#pragma unroll
  for (int i = 0; i < ATT_COLS / 2; ++i) {
    const int col = col0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1), row = row0 + 8 * ((i >> 1) & 1);
    if (ROWS_ARE_KEYS ? row > col : col > row) s[i] = -INFINITY;
  }
}

// Writes this thread's rows (< n) of a 64 x NO accumulator, row r times factor[r] (and, with COLF, column j times
// colf[j]), as bf16 to head h of the [B*n, ld] buffer out.  Fragment row r holds columns 8 jn + 2 (lane % 4) + {0, 1} in
// acc[4 jn + 2 r], acc[4 jn + 2 r + 1].
template <int NO, bool COLF = false>
__device__ __forceinline__ void store_rows(const float (&acc)[NO / 2], __nv_bfloat16* out, long ld, const AttnCta& c,
                                           int n, int d, const float (&factor)[2] = {1.f, 1.f},
                                           const float* colf = nullptr) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = c.row0 + c.rloc + 8 * r;
    if (row >= n) continue;
    __nv_bfloat16* orow = out + (static_cast<long>(c.b) * n + row) * ld + c.h * d;
#pragma unroll
    for (int jn = 0; jn < NO / 8; ++jn) {
      const int col = 8 * jn + 2 * (c.lane & 3);
      if (col >= d) continue;
      float f0 = factor[r], f1 = factor[r];
      if constexpr (COLF) {
        const float2 cf = *reinterpret_cast<const float2*>(colf + col);
        f0 *= cf.x;
        f1 *= cf.y;
      }
      *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16(acc[4 * jn + 2 * r] * f0, acc[4 * jn + 2 * r + 1] * f1);
    }
  }
}

// The CTA's rows (< n) of head h of the [B*n, ld] bf16 buffer out, every element pair set to the bits `pair`, by all
// the CTA's threads.
__device__ __forceinline__ void fill_rows(__nv_bfloat16* out, long ld, const AttnCta& c, int n, int d, uint32_t pair) {
  const int rows = min(ATT_ROWS, n - c.row0), pairs = d / 2;
  for (int i = threadIdx.x; i < rows * pairs; i += ATT_THREADS)
    reinterpret_cast<uint32_t*>(out + (static_cast<long>(c.b) * n + c.row0 + i / pairs) * ld + c.h * d)[i % pairs] = pair;
}

// A dead CTA's rows: zeros.
__device__ __forceinline__ void zero_rows(__nv_bfloat16* out, long ld, const AttnCta& c, int n, int d) {
  fill_rows(out, ld, c, n, d, 0u);
}

// ------------------------------------------------------------------ host side
// Refuses, as entry point fn, a head dim that is not a multiple of 8 in [16, 128] and a pitch that is not a multiple of 8.
inline int check_head_args(const char* fn, int d, std::initializer_list<long> pitches) {
  const char* why = d % 8 != 0 || d > 128 || d < 16 ? "head_dim must be a multiple of 8 in [16,128]" : nullptr;
  for (long ld : pitches)
    if (why == nullptr && (ld & 7)) why = "pitches must be multiples of 8";
  if (why == nullptr) return 0;
  char msg[128];
  snprintf(msg, sizeof(msg), "%s: %s", fn, why);
  return set_error(msg);
}

template <int KA_, int NO_, int KS_> struct HeadDim { static constexpr int KA = KA_, NO = NO_, KS = KS_; };

// Calls f(HeadDim<KA, NO, KS>{}) for head dim d: KA 64-column atoms, NO = d rounded up to 32 (the N of the accumulate
// MMAs) and KS = ceil(d / 16) k16 steps of the score MMAs.
template <class F>
int dispatch_head_dim(int d, F&& f) {
  const bool ks_even = (d + 15) / 16 % 2 == 0;
  switch ((d + 31) / 32) {
    case 1: return ks_even ? f(HeadDim<1, 32, 2>{}) : f(HeadDim<1, 32, 1>{});
    case 2: return ks_even ? f(HeadDim<1, 64, 4>{}) : f(HeadDim<1, 64, 3>{});
    case 3: return ks_even ? f(HeadDim<2, 96, 6>{}) : f(HeadDim<2, 96, 5>{});
    default: return ks_even ? f(HeadDim<2, 128, 8>{}) : f(HeadDim<2, 128, 7>{});
  }
}

// Raises Kern's shared-memory limit (`attr` names that call in an error) and launches it on one CTA per (128-row block,
// head, clip); the forward passes NO_PDL and the backward ALLOW_PDL.
template <auto Kern, LaunchPdl PDL, class... Args>
int launch_attn(const char* attr, const char* name, int smem, int B, int n, int H, cudaStream_t stream,
                const Args&... args) {
  if (int rc = raise_smem_limit<Kern>(smem, attr)) return rc;
  return launch(name, Kern, dim3((n + ATT_ROWS - 1) / ATT_ROWS, H, B), ATT_THREADS, smem, stream, PDL, args...);
}

}  // namespace ivb
