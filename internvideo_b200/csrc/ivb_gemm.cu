// ivb_gemm.cu — persistent, warp-specialised bf16 GEMM on Hopper wgmma tensor cores (sm_90a).
//
//   D[M,N] = epilogue( sum_k A(m,k) * B(n,k) ),  fp32 accumulation in registers.
//
// Replaces the reference's cuBLAS / cuBLASLt calls behind nn.Linear and FA2 fused_dense:
//   Attention.qkv / proj      InternVideo2/single_modality/models/internvideo2_pretrain.py:195,211
//   Mlp.fc1 / fc2 (+GELU)     internvideo2_pretrain.py:232-244 (FusedMLP :269)
//   LayerScale + residual     internvideo2_pretrain.py:131-146,284-291   (fused into the epilogue)
//   Linear_Decoder/MLP_Decoder heads  internvideo2_pretrain.py:341,375-379
//   PatchEmbed Conv3d as GEMM internvideo2_pretrain.py:320-331 (im2col done by ivb_embed.cu)
// and their autograd dgrad / wgrad GEMMs (operands read "transposed" straight from the
// row-major tensors through MN-major wgmma descriptors — no transpose copies).
//
// Structure (one CTA per SM, 384 threads = three warpgroups):
//   warpgroup 0   : TMA producer (one elected thread; cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx),
//                   gives its registers to the MMA warpgroups (setmaxnreg)
//   warpgroups 1-2: 64 rows of the 128 x BN tile each: wgmma m64nBNk16 from the smem ring, then the fused epilogue
//                   (accumulator fragments -> per-warp smem staging tile -> row segments -> global)
// The ring keeps streaming the next tile's operands while the MMA warpgroups run the epilogue.
//
// FP8 (ivb_gemm_fp8): the same kernels with the operand format as a template parameter (Op).  A 128-byte swizzle row
// holds 64 bf16 or 128 fp8 elements, so a stage has the same byte layout, a k-block is still four wgmmas (k16 bf16 or
// k32 fp8) 32 B apart, and only the instruction and the k-block's element count change.  FP8 operands are K-major
// (fp8 wgmma has no transpose bits).  The epilogue first multiplies the accumulator by a_scale_inv * b_scale_inv (two
// device scalars read once per CTA, so a captured graph stays valid), then runs the bf16 epilogues unchanged.
// Accumulation: the tensor core's fp8 MMA keeps fewer mantissa bits in its running sum than fp32 (about 14, DeepSeek-V3
// technical report 3.3.2).  The ping-pong kernel accumulates in the tensor core; the FP8 cooperative kernel promotes:
// each 128-element k-block goes into a fresh register tile, which the CUDA cores add to the fp32 accumulator.
// Vector scales (IVB_FLAG_FP8_VECTOR_SCALES, Op = OpVecFp8): a_scale_inv[M] per row and b_scale_inv[N] per column;
// the same in-place dequantisation multiplies each accumulator by its row's and its column's factor.
// Block scales (ivb_gemm_fp8_wgrad, Op = OpBlockFp8: the weight gradient over tokens, DeepSeek-V3 technical report
// 3.3): one scale per row and per column of each 128-element k-block, a_scale_inv [ceil(K/128), M] and b_scale_inv
// [ceil(K/128), N].  They cannot be factored out of the k sum, so the cooperative kernel applies them where it
// promotes: acc += part * a_s[row] * b_s[col] per k-block.  The producer copies a k-block's 128 row and BN column
// scales into the ring stage with its operands, under the stage's full barrier.
//
// Ping-pong form (gemm_bf16_pingpong_kernel, the default for most shapes, see use_pingpong): same producer, ring and
// epilogue, but each MMA warpgroup owns a whole 128 x 128 tile and the two alternate, so one runs its epilogue while
// the other issues its MMAs.
//
// CL = 2 (the CTA-pair form, IVB_FLAG_2CTA / ivb_set_default_2cta): a cluster of two CTAs on neighbouring SMs computes
// a 256 x BN tile.  Each CTA loads its own 128 A rows and HALF of the B tile, which TMA multicasts into both CTAs'
// rings, so B is read from L2 once per 256 rows instead of once per 128.  A stage is refilled only when the MMA
// warpgroups of BOTH CTAs released it (each arrives on its own and on the peer's empty barrier).
//
// DropPath plans (ivb_gemm_bf16_plan: bf16 single-CTA kernels; ivb_gemm_fp8_plan: the OpPlannedFp8 instantiations of
// both FP8 forms): an M plan puts the row tiles holding a kept row first, and the tiles after its live count only store
// (dead_tile); a K plan lists the k-blocks the weight gradient sums (ivb_gemm_bf16_plan, and ivb_gemm_fp8_wgrad with
// 128-token k-blocks).
//
// Both kernels are built from the same pieces (gemm_prologue, produce, mma_kblock, dequantise, epilogue_tile) and keep
// only how their MMA warpgroups consume and release the ring: FP8 promotion and the CTA pair's remote arrivals in the
// cooperative kernel, the token in the ping-pong kernel.  Both C entry points share choose_kernel, dispatch and
// launch_gemm.
#include <cstdio>

#include "ivb_gemm_common.cuh"

namespace ivb {

constexpr int BM = 128;
constexpr int K_MMAS = 4;              // wgmmas per k-block, 32 B apart along the 128-byte swizzle row
constexpr int GEMM_THREADS = 384;
constexpr int A_STAGE_BYTES = BM * 128;     // 16 KB: 128 rows of one 128-byte k-block, either major
constexpr int EPI_PITCH = 36;               // floats per staged row: 32 columns + 4 (bank spread, 16-B rows)
constexpr int EPI_BYTES = 8 * 16 * EPI_PITCH * 4;  // one 16 x 32 fp32 staging tile per MMA warp

// Operand formats: bf16 x bf16, or fp8 (A E4M3 or E5M2, B E4M3).  BK: elements in a 128-byte k-block.
// VEC: per-row / per-column scale vectors instead of two scalars (E4M3 A only).
// PLAN: the single-CTA kernels are built with the DropPath plan code (PLANNED); OpPlannedFp8 is OpVecFp8 with it, so
// ivb_gemm_fp8 keeps kernels without it.
struct OpBf16 {
  static constexpr bool FP8 = false, VEC = false, PLAN = true, BLOCK = false;
  static constexpr int BK = 64;
};
template <bool A_E5M2_>
struct OpFp8 {
  static constexpr bool FP8 = true, A_E5M2 = A_E5M2_, VEC = false, PLAN = false, BLOCK = false;
  static constexpr int BK = 128;
};
struct OpVecFp8 {
  static constexpr bool FP8 = true, A_E5M2 = false, VEC = true, PLAN = false, BLOCK = false;
  static constexpr int BK = 128;
};
struct OpPlannedFp8 : OpVecFp8 {
  static constexpr bool PLAN = true;
};
// BLOCK: per-k-block row and column scales (E4M3 A), applied as each k-block is promoted; built with the plan code for
// its K plan.
struct OpBlockFp8 {
  static constexpr bool FP8 = true, A_E5M2 = false, VEC = false, PLAN = true, BLOCK = true;
  static constexpr int BK = 128;
};

// SCALES (OpBlockFp8): each stage also holds its k-block's BM row and BN column scales, after the barriers.
template <int BN, bool B_MN, bool SCALES = false>
struct GemmCfg {
  static constexpr int B_ATOMS = (BN + 63) / 64;
  static constexpr int B_STAGE_BYTES = B_MN ? B_ATOMS * 64 * 128 : BN * 128;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int SCALE_FLOATS = SCALES ? BM + BN : 0;
  static constexpr int STAGES_RAW = (227 * 1024 - EPI_BYTES - 1024 - 256) / (STAGE_BYTES + 4 * SCALE_FLOATS);
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * (STAGE_BYTES + 4 * SCALE_FLOATS) + EPI_BYTES + 1024 /*align slack*/ +
                                    256 /*barriers*/;
};

// ------------------------------------------------------------------ epilogue of one warpgroup's accumulators
// acc[h] holds rows [row0 + 64h, row0 + 64h + 64) x BN columns: NH = 1 for a cooperative warpgroup's band, NH = 2 for a
// ping-pong warpgroup's whole tile.  The epilogue walks it in chunks of 32 columns of one 64-row band, the band index
// running fastest: fragments -> the warp's 16 x 32 staging tile -> one 16-column row segment per thread.
//
// The chunk loop is rolled, so the kernel holds one copy of the epilogue body.  Unrolled, every chunk carried its own
// copy of all six epilogue forms (17 K instructions per kernel), and the fc1 epilogue ran at the speed of the
// instruction fetch.  Only the fragment -> staging copy is selected per chunk (epilogue_stage), so acc is indexed with
// constants and stays in registers.  Each chunk's global inputs are loaded during the previous chunk; bias and gamma
// are loaded once per 32-column strip, and the NH bands of the strip share them.
template <int BN, int NH>
__device__ __forceinline__ void epilogue_stage(const float (&acc)[NH][BN / 2], float* st, int chunk, int lane) {
#pragma unroll
  for (int k = 0; k < NH * ((BN + 31) / 32); ++k) {
    if (k != chunk) continue;
    const int h = k % NH, c = k / NH;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * c + jj;
      if (j < BN / 8) {
#pragma unroll
        for (int q = 0; q < 2; ++q)
          *reinterpret_cast<float2*>(st + ((lane >> 2) + 8 * q) * EPI_PITCH + 8 * jj + 2 * (lane & 3)) =
              make_float2(acc[h][4 * j + 2 * q], acc[h][4 * j + 2 * q + 1]);
      }
    }
  }
}

template <int BN, int NH, bool SWIGLU>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float (&acc)[NH][BN / 2], float* st, long row0,
                                              int n0) {
  constexpr int CHUNKS = NH * ((BN + 31) / 32);
  const int lane = threadIdx.x & 31;
  const int wr = (threadIdx.x >> 5) & 3;   // warp inside the warpgroup: rows [16*wr, 16*wr + 16) of each band
  const long row_b0 = row0 + wr * 16 + (lane >> 1);
  const int half = lane & 1;
  const bool accum = (p.flags & IVB_FLAG_ACCUM) != 0;
  const bool tanh_mode = (p.flags & IVB_FLAG_GELU_TANH) != 0;
  const bool quick_mode = (p.flags & IVB_FLAG_GELU_QUICK) != 0;
  const bool save_grad = (p.flags & IVB_FLAG_GELU_SAVE_GRAD) != 0;
  // this thread's row, first column (in the tile) and columns inside the matrix in chunk i
  auto row_of = [&](int i) { return row_b0 + 64 * (i % NH); };
  auto col_of = [&](int i) { return (i / NH) * 32 + half * 16; };
  auto nvalid_of = [&](int i) {
    const int col = col_of(i);
    if (col >= BN || row_of(i) >= p.M) return 0;
    return min(16, p.N - n0 - col);
  };
  EpiIn<16> next;
  if (nvalid_of(0) > 0) epilogue_load<16>(p, accum, next, row_of(0), n0 + col_of(0), nvalid_of(0));
  uint32_t bias[8] = {}, gamma[8] = {};
#pragma unroll 1
  for (int i = 0; i < CHUNKS; ++i) {
    const long row = row_of(i);
    const int col = col_of(i), nvalid = nvalid_of(i);
    const EpiIn<16> in = next;
    if (i + 1 < CHUNKS && nvalid_of(i + 1) > 0)
      epilogue_load<16>(p, accum, next, row_of(i + 1), n0 + col_of(i + 1), nvalid_of(i + 1));
    if (i % NH == 0 && col < BN && n0 + col < p.N) {
      const int ncols = min(16, p.N - n0 - col);
      if (p.bias != nullptr) load_bits_bf16<16>(p.bias + n0 + col, bias, ncols);
      if (p.gamma != nullptr) load_bits_bf16<16>(p.gamma + n0 + col, gamma, ncols);
    }
    epilogue_stage<BN, NH>(acc, st, i, lane);
    __syncwarp();
    if (nvalid > 0) {
      float v[16];
      const float* src = st + (lane >> 1) * EPI_PITCH + half * 16;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 f = reinterpret_cast<const float4*>(src)[k];
        v[4 * k] = f.x; v[4 * k + 1] = f.y; v[4 * k + 2] = f.z; v[4 * k + 3] = f.w;
      }
      epilogue_chunk<16, SWIGLU>(p, accum, tanh_mode, quick_mode, save_grad, v, in, bias, gamma, row, n0 + col, nvalid);
    }
    __syncwarp();
  }
}

// fp8: dequantise the accumulators in place before the epilogue.  (Scaling them as the epilogue stages them lets the
// compiler hoist every product out of the rolled chunk loop, which needs a second copy of acc and spills.)
// Vector scales: acc[h][4j + 2q + e] is the accumulator of row row0 + 64h + 16 * (warp in the warpgroup) + lane / 4 +
// 8q and column n0 + 8j + 2 * (lane % 4) + e (the wgmma fragment layout, as epilogue_stage reads it).  A thread
// holds 2 NH rows, whose factors it loads once, and reads each column pair's factors as one 8-byte load.  Rows and
// columns outside the matrix are never stored: they get factor 0 and no load.
template <class Op, int BN, int NH>
__device__ __forceinline__ void dequantise(const GemmParams& p, float (&acc)[NH][BN / 2], float dq, long row0, int n0) {
  if constexpr (Op::VEC) {
    const int lane = threadIdx.x & 31;
    const long r0 = row0 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
    float ra[NH][2];
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int q = 0; q < 2; ++q) ra[h][q] = r0 + 64 * h + 8 * q < p.M ? p.a_scale_inv[r0 + 64 * h + 8 * q] : 0.0f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = n0 + 8 * j + 2 * (lane & 3);
      const float2 cb = col < p.N ? *reinterpret_cast<const float2*>(p.b_scale_inv + col) : make_float2(0.0f, 0.0f);
#pragma unroll
      for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          acc[h][4 * j + 2 * q] *= ra[h][q] * cb.x;
          acc[h][4 * j + 2 * q + 1] *= ra[h][q] * cb.y;
        }
    }
  } else if constexpr (Op::FP8 && !Op::BLOCK) {   // block scales were applied as each k-block was promoted
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[h][i] *= dq;
  }
}

// Block scales: one k-block's partial sums, times their row's and column's scale of that k-block (read from the ring
// stage before it is released: rows row0 .. row0 + 63 of this warpgroup, fragment layout as in dequantise), added to
// the fp32 accumulator.
template <int BN>
struct BlockScales {
  float ra[2];
  float2 cb[BN / 8];
};
template <int BN>
__device__ __forceinline__ void load_block_scales(BlockScales<BN>& bs, const float* sc, int row0) {
  const int lane = threadIdx.x & 31;
  const int r = row0 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  bs.ra[0] = sc[r];
  bs.ra[1] = sc[r + 8];
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) bs.cb[j] = *reinterpret_cast<const float2*>(sc + BM + 8 * j + 2 * (lane & 3));
}
template <int BN>
__device__ __forceinline__ void promote_block(float (&acc)[BN / 2], const float (&part)[BN / 2], const BlockScales<BN>& bs) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      acc[4 * j + 2 * q] = fmaf(part[4 * j + 2 * q], bs.ra[q] * bs.cb[j].x, acc[4 * j + 2 * q]);
      acc[4 * j + 2 * q + 1] = fmaf(part[4 * j + 2 * q + 1], bs.ra[q] * bs.cb[j].y, acc[4 * j + 2 * q + 1]);
    }
}

// ------------------------------------------------------------------ pieces of both kernels
// Shared memory, aligned to 1024 bytes for the 128-byte swizzle: the ring (STAGES A stages, then STAGES B stages), one
// 16 x 32 fp32 staging tile per MMA warp, then each stage's full and empty barrier.
struct Smem {
  uint8_t* a;
  uint8_t* b;
  float* epi;
  uint64_t* full;
  uint64_t* empty;
  float* scales;   // SCALES: STAGES x (BM row + BN column) scales
};

// Carves up shared memory, initialises the barriers and waits for the previous kernel (PDL).  `empty_arrivals`: the
// releases a stage waits for before the producer refills it.
template <int BN, bool B_MN, int CL, bool SCALES = false>
__device__ __forceinline__ Smem gemm_prologue(const CUtensorMap& tmA, const CUtensorMap& tmB, uint32_t empty_arrivals) {
  using Cfg = GemmCfg<BN, B_MN, SCALES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  Smem s;
  s.a = smem;
  s.b = smem + Cfg::STAGES * A_STAGE_BYTES;
  s.epi = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  s.full = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + EPI_BYTES);
  s.empty = s.full + Cfg::STAGES;
  s.scales = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + EPI_BYTES + 256);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&s.full[i], 1);
      mbar_init(&s.empty[i], empty_arrivals);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (CL == 2) cluster_sync_all();   // the peer's barriers exist before any multicast or remote arrive reaches them
  pdl_wait();
  pdl_launch_dependents();
  return s;
}

// The tiles (tile order: row tile, then column tile) and k-blocks a kernel's MMAs run: all of them, or under a DropPath
// plan the live tiles and the listed k-blocks (the counts after each list).  A K plan that lists no k-block leaves no
// live tile: every tile then runs dead_tile, whose zeros are the empty sum.  Read after gemm_prologue's PDL wait.
struct PlanCounts {
  int live_tiles, num_kb;
};
// Only the single-CTA kernels of an Op with PLAN are built with the plan code (PLANNED).
template <class Op, int CL>
constexpr bool PLANNED = Op::PLAN && CL == 1;
// K plans for bf16 and for the block-scaled FP8 weight gradient (over tokens; its K plan lists 128-token k-blocks).
template <class Op, int CL>
constexpr bool K_PLANNED = PLANNED<Op, CL> && (!Op::FP8 || Op::BLOCK);

template <class Op, int BN, int CL>
__device__ __forceinline__ PlanCounts plan_counts(const GemmParams& p) {
  const int num_m = (p.M + CL * BM - 1) / (CL * BM), num_n = (p.N + BN - 1) / BN, num_kb = (p.K + Op::BK - 1) / Op::BK;
  if constexpr (!PLANNED<Op, CL>) return {num_m * num_n, num_kb};
  const int live_kb = K_PLANNED<Op, CL> && p.k_plan != nullptr ? p.k_plan[num_kb] : num_kb;
  return {live_kb > 0 ? (p.m_plan != nullptr ? p.m_plan[num_m] : num_m) * num_n : 0, live_kb};
}

// The row tile the kernels' mt-th tile covers: mt, or under an M plan the plan's mt-th tile.
template <class Op, int CL>
__device__ __forceinline__ int plan_tile(const GemmParams& p, int mt) {
  if constexpr (PLANNED<Op, CL>) return p.m_plan != nullptr ? p.m_plan[mt] : mt;
  return mt;
}

// The TMA producer (one elected thread): every k-block of the tiles first_tile, first_tile + stride, ... below
// num_tiles, in that order.  CL = 2: the cluster's tile has 256 rows; this CTA (rank) loads its own 128 A rows and half
// of the B tile, which TMA multicasts into both CTAs' rings.  Under a DropPath plan (p.m_plan / p.k_plan, CL = 1 only)
// num_tiles counts the live tiles, which come first, and only the listed k-blocks are loaded.
template <class Op, int BN, bool A_MN, bool B_MN, int CL>
__device__ __forceinline__ void produce(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p,
                                        const Smem& s, int first_tile, int stride, int num_tiles, int num_kb,
                                        uint32_t rank) {
  using Cfg = GemmCfg<BN, B_MN, Op::BLOCK>;
  const int num_n = (p.N + BN - 1) / BN;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = first_tile; tile < num_tiles; tile += stride) {
    const int m0 = plan_tile<Op, CL>(p, tile / num_n) * (CL * BM) + rank * BM;
    const int n0 = (tile % num_n) * BN;
    for (int i = 0; i < num_kb; ++i) {
      const int kb = K_PLANNED<Op, CL> && p.k_plan != nullptr ? p.k_plan[i] : i;
      mbar_wait(&s.empty[stage], phase ^ 1);
      // block scales: the rows and columns inside the matrix (M, N multiples of 8: whole 16-byte pieces)
      const uint32_t a_sbytes = Op::BLOCK ? 4u * min(BM, p.M - m0) : 0u;
      const uint32_t b_sbytes = Op::BLOCK ? 4u * min(BN, p.N - n0) : 0u;
      mbar_expect_tx(&s.full[stage], Cfg::STAGE_BYTES + a_sbytes + b_sbytes);
      uint8_t* sa = s.a + stage * A_STAGE_BYTES;
      uint8_t* sb = s.b + stage * Cfg::B_STAGE_BYTES;
      const int k0 = kb * Op::BK;
      if (!A_MN) {
        tma_load_2d(sa, &tmA, k0, m0, &s.full[stage]);
      } else {
#pragma unroll
        for (int i = 0; i < BM / 64; ++i)
          tma_load_2d(sa + i * 8192, &tmA, m0 + i * 64, k0, &s.full[stage]);
      }
      if (CL == 1) {
        if (!B_MN) {
          // IVB_EPI_SWIGLU: tmB is the 4-D (k, row, half, 8-row group) map of launch_gemm, so the tile's BN rows come in
          // as gate rows 8g .. 8g + 7, then the up rows of the same output columns, for each of its BN / 16 groups
          if (!Op::FP8 && p.epi == IVB_EPI_SWIGLU)
            tma_load_4d(sb, &tmB, k0, 0, 0, n0 / 16, &s.full[stage]);
          else
            tma_load_2d(sb, &tmB, k0, n0, &s.full[stage]);
        } else {
#pragma unroll
          for (int i = 0; i < Cfg::B_ATOMS; ++i)
            tma_load_2d(sb + i * 8192, &tmB, n0 + i * 64, k0, &s.full[stage]);
        }
      } else {  // this CTA's half of B, into both CTAs (K-major: BN/2 rows; MN-major: every other 64-wide atom)
        if (!B_MN) {
          tma_load_2d_mc(sb + rank * (BN / 2) * 128, &tmB, k0, n0 + rank * (BN / 2), &s.full[stage], 0x3);
        } else {
#pragma unroll
          for (int i = 0; i < Cfg::B_ATOMS; ++i)
            if ((i & 1) == static_cast<int>(rank))
              tma_load_2d_mc(sb + i * 8192, &tmB, n0 + i * 64, k0, &s.full[stage], 0x3);
        }
      }
      if constexpr (Op::BLOCK) {
        float* sc = s.scales + stage * Cfg::SCALE_FLOATS;
        bulk_load_1d(sc, p.a_scale_inv + static_cast<long>(kb) * p.M + m0, a_sbytes, &s.full[stage]);
        bulk_load_1d(sc + BM, p.b_scale_inv + static_cast<long>(kb) * p.N + n0, b_sbytes, &s.full[stage]);
      }
      if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
  }
}

// Issues and commits one k-block's wgmmas from ring stage `stage`: K_MMAS steps 32 B apart along the k-block, each with
// one wgmma per 64-row band h0, h0 + 1, ..., h0 + NH - 1 of the A stage into d[0 .. NH-1].  accumulate = false: the
// first step overwrites d.
template <class Op, int BN, bool A_MN, bool B_MN, int NH>
__device__ __forceinline__ void mma_kblock(float (&d)[NH][BN / 2], const Smem& s, int stage, int h0, bool accumulate) {
  using Cfg = GemmCfg<BN, B_MN>;
  const uint32_t sa = smem_u32(s.a + stage * A_STAGE_BYTES);
  const uint32_t sb = smem_u32(s.b + stage * Cfg::B_STAGE_BYTES);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < K_MMAS; ++k) {
    const uint64_t bd = B_MN ? gmma_desc(sb + k * 2048, 8192, 1024) : gmma_desc(sb + k * 32, 16, 1024);
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      const uint64_t ad = A_MN ? gmma_desc(sa + (h0 + h) * 8192 + k * 2048, 8192, 1024)
                               : gmma_desc(sa + (h0 + h) * 8192 + k * 32, 16, 1024);
      const uint32_t scale_d = (accumulate || k > 0) ? 1u : 0u;
      if constexpr (Op::FP8)
        WgmmaF8<BN>::template ss<Op::A_E5M2>(d[h], ad, bd, scale_d);
      else
        Wgmma<BN>::template ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(d[h], ad, bd, scale_d);
    }
  }
  wgmma_commit();
}

// ------------------------------------------------------------------ the cooperative kernel
// Op: operand format.  The FP8 form promotes (see the top of the file): each k-block's four wgmmas accumulate into
// `part`, which is added to acc once they retire; BN <= 192 keeps both tiles in the 232 registers of a thread.
template <class Op, int BN, bool A_MN, bool B_MN, int CL>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using Cfg = GemmCfg<BN, B_MN, Op::BLOCK>;
  constexpr int STAGES = Cfg::STAGES;
  const int warp = threadIdx.x >> 5;
  const int wg = threadIdx.x >> 7;

  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0;   // 128-row half of the cluster's tile
  const int cid = blockIdx.x / CL, ncl = gridDim.x / CL;   // tiles are walked per cluster
  const int num_m = (p.M + CL * BM - 1) / (CL * BM);
  const int num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  constexpr bool PROMOTE = Op::FP8;

  const Smem s = gemm_prologue<BN, B_MN, CL, Op::BLOCK>(tmA, tmB, 2 * CL);   // one arrival per MMA warpgroup of the cluster
  const PlanCounts pc = plan_counts<Op, BN, CL>(p);
  const int num_kb = pc.num_kb;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) produce<Op, BN, A_MN, B_MN, CL>(tmA, tmB, p, s, cid, ncl, pc.live_tiles, num_kb, rank);
  } else {
    setmaxnreg_inc<232>();
    // ===================== MMA + epilogue warpgroups =====================
    const int cw = wg - 1;              // rows [64*cw, 64*cw + 64) of the tile
    const bool signal = (threadIdx.x & 127) == 0;
    auto release = [&](int s_) {   // this warpgroup no longer reads stage s_ (of either CTA's ring)
      if (!signal) return;
      mbar_arrive(&s.empty[s_]);
      if (CL == 2) mbar_arrive_cluster(mapa_u32(smem_u32(&s.empty[s_]), rank ^ 1));
    };
    float* st = s.epi + (warp - 4) * 16 * EPI_PITCH;
    float dq = 1.0f;
    if constexpr (Op::FP8 && !Op::VEC && !Op::BLOCK) dq = *p.a_scale_inv * *p.b_scale_inv;
    float acc[1][BN / 2];
    float part[1][PROMOTE ? BN / 2 : 1];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = cid; tile < num_tiles; tile += ncl) {
      const int m0 = plan_tile<Op, CL>(p, tile / num_n) * (CL * BM) + rank * BM;
      const int n0 = (tile % num_n) * BN;
      if (PLANNED<Op, CL> && tile >= pc.live_tiles) {   // M plan: a tile of dropped rows, nothing loaded
        dead_tile<BN>(p, m0 + cw * 64, 64, n0);
        continue;
      }
      int prev = 0;
      if constexpr (PROMOTE) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[0][i] = 0.0f;
      }
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&s.full[stage], phase);
        if constexpr (PROMOTE) {  // this k-block's partial sum, added in fp32; its smem slot is free
          mma_kblock<Op, BN, A_MN, B_MN, 1>(part, s, stage, cw, false);
          if constexpr (Op::BLOCK) {   // the k-block's scales, read while its MMAs run
            BlockScales<BN> bs;
            load_block_scales<BN>(bs, s.scales + stage * Cfg::SCALE_FLOATS, cw * 64);
            wgmma_wait<0>();
            wgmma_reg_fence(part[0], BN / 2);
            release(stage);
            promote_block<BN>(acc[0], part[0], bs);
          } else {
            wgmma_wait<0>();
            wgmma_reg_fence(part[0], BN / 2);
            release(stage);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[0][i] += part[0][i];
          }
        } else {
          mma_kblock<Op, BN, A_MN, B_MN, 1>(acc, s, stage, cw, kb > 0);
          if (kb > 0) {  // the MMAs of the previous k-block retired: its smem slot is free
            wgmma_wait<1>();
            release(prev);
          }
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if constexpr (!PROMOTE) {
        wgmma_wait<0>();
        wgmma_reg_fence(acc[0], BN / 2);
        release(prev);
      }
      dequantise<Op, BN, 1>(p, acc, dq, m0 + cw * 64, n0);
      epilogue_tile<BN, 1, !Op::FP8>(p, acc, st, m0 + cw * 64, n0);
    }
  }
  if (CL == 2) cluster_sync_all();   // the peer may still multicast into / arrive on this CTA's ring
}

// ------------------------------------------------------------------ the ping-pong kernel
// Same producer, ring and epilogue as the cooperative kernel at BN = 128, but each MMA warpgroup owns a whole 128 x 128
// tile: the CTA's j-th tile (static persistent order) goes to warpgroup j & 1, which issues two m64n128k16 wgmmas per
// k16 step, one per 64-row half of the A stage.  The producer streams the tiles' k-blocks in that same order, and a
// token passed between the warpgroups on named barriers 1 and 2 keeps the ring consumed strictly in order: a warpgroup
// takes the token before its first k-block of a tile and hands it on as soon as the tile's last wgmma is committed,
// so the other warpgroup's MMAs queue behind them while this one waits for its MMAs and runs the epilogue.  The
// tensor cores stay busy through every epilogue except the CTA's last.
constexpr int PP_BN = 128;

template <class Op, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_pingpong_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const GemmParams p) {
  constexpr int STAGES = GemmCfg<PP_BN, B_MN>::STAGES;
  const int warp = threadIdx.x >> 5;
  const int wg = threadIdx.x >> 7;
  const int num_n = (p.N + PP_BN - 1) / PP_BN;
  const int num_tiles = ((p.M + BM - 1) / BM) * num_n;

  const Smem s = gemm_prologue<PP_BN, B_MN, 1>(tmA, tmB, 1);   // each stage is read by exactly one MMA warpgroup
  const PlanCounts pc = plan_counts<Op, PP_BN, 1>(p);
  const int num_kb = pc.num_kb;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one())
      produce<Op, PP_BN, A_MN, B_MN, 1>(tmA, tmB, p, s, blockIdx.x, gridDim.x, pc.live_tiles, num_kb, 0);
  } else {
    setmaxnreg_inc<232>();
    // ===================== MMA + epilogue warpgroups, one whole tile each =====================
    const int cw = wg - 1;              // this warpgroup takes the CTA's tiles j with (j & 1) == cw
    const bool signal = (threadIdx.x & 127) == 0;
    float* st = s.epi + (warp - 4) * 16 * EPI_PITCH;
    float dq = 1.0f;
    if constexpr (Op::FP8 && !Op::VEC) dq = *p.a_scale_inv * *p.b_scale_inv;
    float acc[2][PP_BN / 2];            // rows [0, 64) and [64, 128) of the tile
    for (int j = cw, tile = blockIdx.x + cw * gridDim.x; tile < num_tiles; j += 2, tile += 2 * gridDim.x) {
      const int m0 = plan_tile<Op, 1>(p, tile / num_n) * BM;
      const int n0 = (tile % num_n) * PP_BN;
      // M plan: live tiles come first, so the CTA's j-th tile is live exactly when j counts its live tiles; a dead
      // tile takes no token and no ring stage
      if (PLANNED<Op, 1> && tile >= pc.live_tiles) {
        dead_tile<PP_BN>(p, m0, BM, n0);
        continue;
      }
      const int it = j * num_kb;        // ring position of this tile's first k-block
      int stage = it % STAGES;
      uint32_t phase = (it / STAGES) & 1;
      // the token: the other warpgroup has committed every MMA of the previous tile (tile 0 needs none)
      if (j > 0) named_bar_sync(1 + cw, 256);
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&s.full[stage], phase);
        mma_kblock<Op, PP_BN, A_MN, B_MN, 2>(acc, s, stage, 0, kb > 0);
        if (kb > 0) {  // the MMAs of the previous k-block retired: its smem slot is free
          wgmma_wait<1>();
          if (signal) mbar_arrive(&s.empty[prev]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // hand the token on (only if the CTA has a next tile: an arrival nobody waits for would outlive the CTA)
      if (tile + gridDim.x < pc.live_tiles) named_bar_arrive(2 - cw, 256);
      wgmma_wait<0>();
      wgmma_reg_fence(acc[0], PP_BN / 2);
      wgmma_reg_fence(acc[1], PP_BN / 2);
      if (signal) mbar_arrive(&s.empty[prev]);
      dequantise<Op, PP_BN, 2>(p, acc, dq, m0, n0);
      epilogue_tile<PP_BN, 2, !Op::FP8>(p, acc, st, m0, n0);
    }
  }
}

// ------------------------------------------------------------------ host side
template <class Op, bool PINGPONG, int BN, bool A_MN, bool B_MN, int CL>
constexpr auto gemm_kernel() {
  if constexpr (PINGPONG) return gemm_bf16_pingpong_kernel<Op, A_MN, B_MN>;
  else return gemm_bf16_kernel<Op, BN, A_MN, B_MN, CL>;
}

// Launches either kernel form (PINGPONG: BN = PP_BN, CL = 1) on at most one CTA per SM and one cluster per tile.
template <class Op, bool PINGPONG, int BN, bool A_MN, bool B_MN, int CL>
static int launch_gemm(const void* A, long lda, const void* B, long ldb, const GemmParams& p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN, B_MN, Op::BLOCK && !PINGPONG>;
  constexpr int EB = Op::FP8 ? 1 : 2;
  CUtensorMap tmA, tmB;
  int rc;
  if (!A_MN) rc = make_tmap_2d(&tmA, A, (uint64_t)p.K, (uint64_t)p.M, lda, Op::BK, BM, EB);
  else       rc = make_tmap_2d(&tmA, A, (uint64_t)p.M, (uint64_t)p.K, lda, 64, 64);
  if (rc) return rc;
  if (p.epi == IVB_EPI_SWIGLU) {
    // B = [gate; up], [2I, K]: dims (k, row in an 8-row group, half [I rows apart], group [8 rows apart]).  An 8-row
    // group is one 128-byte swizzle atom, so the box lands in shared memory as a 2-D box of the same BN rows would.
    const long I = p.N / 2;
    const uint64_t dims[4] = {(uint64_t)p.K, 8, 2, (uint64_t)(I / 8)};
    const long strides[3] = {ldb, I * ldb, 8 * ldb};
    const uint32_t box[4] = {64, 8, 2, BN / 16};
    rc = make_tmap_4d(&tmB, B, dims, strides, box);
  } else if (!B_MN) {
    rc = make_tmap_2d(&tmB, B, (uint64_t)p.K, (uint64_t)p.N, ldb, Op::BK, BN / CL, EB);
  } else {
    rc = make_tmap_2d(&tmB, B, (uint64_t)p.N, (uint64_t)p.K, ldb, 64, 64);
  }
  if (rc) return rc;
  constexpr auto kern = gemm_kernel<Op, PINGPONG, BN, A_MN, B_MN, CL>();
  if ((rc = raise_smem_limit<kern>(Cfg::SMEM_BYTES, "cudaFuncSetAttribute(gemm)"))) return rc;
  const int num_tiles = ((p.M + CL * BM - 1) / (CL * BM)) * ((p.N + BN - 1) / BN);
  int clusters = num_sms() / CL;
  if (clusters > num_tiles) clusters = num_tiles;
  return launch<CL>(PINGPONG ? "gemm_bf16_pingpong_kernel" : "gemm_bf16_kernel", kern, clusters * CL, GEMM_THREADS,
                    Cfg::SMEM_BYTES, stream, ALLOW_PDL, tmA, tmB, p);
}

// Pick the N tile that wastes the fewest padded columns / partial waves (fp8: of the two tiles its cooperative kernel has).
static int choose_bn(int M, int N, int cl, bool fp8 = false) {
  const int cand[4] = {256, 192, 176, 128};
  const int first = fp8 ? 1 : 0, step = fp8 ? 2 : 1;
  const int sms = num_sms() / cl;
  const int num_m = (M + cl * BM - 1) / (cl * BM);
  double best = 1e30;
  int best_bn = 256;
  for (int i = first; i < 4; i += step) {
    const int bn = cand[i];
    const int num_n = (N + bn - 1) / bn;
    const long tiles = (long)num_m * num_n;
    const long waves = (tiles + sms - 1) / sms;
    // cost ~ waves * per-tile time (proportional to bn; small-N tiles are smem-bandwidth limited)
    double per_tile = bn * (bn >= 176 ? 1.0 : 1.15);
    double cost = (double)waves * per_tile;
    if (cost < best - 1e-9) { best = cost; best_bn = bn; }
  }
  return best_bn;
}

// Ping-pong or cooperative (single-CTA kernels).  The ping-pong kernel hides a tile's epilogue under the next tile's
// MMAs, so it needs at least two tiles per CTA; with one, a single warpgroup issues all the MMAs and the kernel is
// slower (wgrad 1408 x 1408 x 13344: 0.095 against 0.090 ms).  Its price is the 128-wide tile, which reads a third
// more operand bytes from shared memory per flop than a 128 x 256 one: at long K, where the epilogue is a small share
// of a tile, the cooperative kernel with BN = 256 stays ahead (wgrad 1408 x 6144 x 13344: 0.318 against 0.400 ms).
// Every other GEMM of the cfg-2 step is 0.5-28 % faster on the ping-pong kernel (DESIGN.md 4.1, tools/gemm_table.py).
static bool use_pingpong(int M, int N, int K) {
  const long tiles = (long)((M + BM - 1) / BM) * ((N + PP_BN - 1) / PP_BN);
  if (tiles <= num_sms()) return false;
  return !(K >= 8192 && choose_bn(M, N, 1) == 256);
}

static bool g_default_2cta = false;

// Operand rules of the fused epilogue (ivb200.h), shared by both entry points; `fn` names the entry point in messages.
static int check_epilogue_args(const char* fn, int epilogue, int flags, const void* out0, const void* out1, long ld1,
                               const void* aux, long ldaux, const void* bias, const void* gamma) {
  char msg[128];
  auto fail = [&](const char* what) {
    std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
    return set_error(msg);
  };
  if (out0 == nullptr) return fail("out0 is null");
  if ((flags & IVB_FLAG_GELU_TANH) && (flags & IVB_FLAG_GELU_QUICK))
    return fail("IVB_FLAG_GELU_TANH and IVB_FLAG_GELU_QUICK exclude each other");
  if ((epilogue == IVB_EPI_RESID || epilogue == IVB_EPI_GELU_BWD) && aux == nullptr) return fail("epilogue needs aux");
  // the epilogue reads and writes every operand in 16-byte vectors (epilogue_chunk): each row must start on 16 bytes
  if (out1 != nullptr && (ld1 & 7)) return fail("ld1 must be a multiple of 8 elements");
  if (aux != nullptr && (ldaux & (epilogue == IVB_EPI_RESID ? 3 : 7)))
    return fail("ldaux must be a multiple of 8 bf16 or 4 fp32 elements");
  const void* vec_ptrs[5] = {out0, out1, aux, bias, gamma};
  const char* vec_msgs[5] = {"out0 must be 16-byte aligned", "out1 must be 16-byte aligned", "aux must be 16-byte aligned",
                             "bias must be 16-byte aligned", "gamma must be 16-byte aligned"};
  for (int i = 0; i < 5; ++i)
    if (reinterpret_cast<uintptr_t>(vec_ptrs[i]) & 15) return fail(vec_msgs[i]);
  return 0;
}

static GemmParams make_params(int M, int N, int K, int epilogue, int flags, void* out0, long ld0, void* out1, long ld1,
                              const void* bias, const void* gamma, const void* aux, long ldaux, const float* rowscale) {
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.epi = epilogue; p.flags = flags;
  p.out0 = out0; p.ld0 = ld0; p.out1 = out1; p.ld1 = ld1;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.gamma = reinterpret_cast<const __nv_bfloat16*>(gamma);
  p.aux = aux; p.ldaux = ldaux; p.rowscale = rowscale;
  p.a_scale_inv = p.b_scale_inv = nullptr;
  p.m_plan = p.k_plan = nullptr;
  return p;
}

struct KernelChoice {
  bool pingpong;
  int bn, cl;
};

// The kernel of a GEMM whose force flags and tile_n the entry point has checked.  The CTA-pair (cluster) kernel when
// forced, or by default (default_2cta) for problems tall enough to fill 256-row tiles; the ping-pong kernel when forced
// or chosen by use_pingpong; the single-CTA cooperative kernel otherwise / when IVB_FLAG_1CTA is set, at tile_n or
// choose_bn's width.  FP8 has no CTA-pair kernel, and its cooperative kernel promotes each k-block to fp32 (BN 192 or
// 128).  Promotion is not needed for accuracy at the step's shapes: the tensor-core accumulation adds at most 4.5 % of
// the error the fp8 quantisation already carries (fc2, K = 6144;
// tests/test_gemm_fp8_gpu.py::test_accumulation_error_at_step_shapes, DESIGN.md 4.1), and ping-pong is the faster
// form at every one of them, so FP8 selects like bf16.
static KernelChoice choose_kernel(int M, int N, int K, int flags, int tile_n, bool fp8, bool default_2cta) {
  const bool force2 = (flags & IVB_FLAG_2CTA) != 0, force1 = (flags & IVB_FLAG_1CTA) != 0;
  const bool forcepp = (flags & IVB_FLAG_PINGPONG) != 0;
  KernelChoice k;
  k.cl = (force2 || (!force1 && !forcepp && default_2cta && M >= 512)) ? 2 : 1;
  k.pingpong = forcepp || (k.cl == 1 && !force1 && (tile_n == 0 || tile_n == PP_BN) && use_pingpong(M, N, K));
  k.bn = k.pingpong ? PP_BN : tile_n > 0 ? tile_n : choose_bn(M, N, k.cl, fp8);
  return k;
}

// The kernel k names, for operands of format Op and majors A_MN / B_MN.  Together with the entry points' choice of Op
// and majors this instantiates the library's 38 kernels: the ping-pong kernel of every Op and major; the bf16
// cooperative kernel at BN 256 / 192 / 176 / 128 and CL 1 or 2; the FP8 one (K-major only) at BN 192 or 128, CL 1,
// and with a plan (OpPlannedFp8) at BN 128 only.  ivb_gemm_fp8_wgrad adds the 39th, the block-scaled cooperative
// kernel (OpBlockFp8) at BN 128, which it launches itself.
template <class Op, bool A_MN, bool B_MN>
static int dispatch(const KernelChoice& k, const void* A, long lda, const void* B, long ldb, const GemmParams& p,
                    cudaStream_t stream) {
  if (k.pingpong) return launch_gemm<Op, true, PP_BN, A_MN, B_MN, 1>(A, lda, B, ldb, p, stream);
  // the cooperative kernel, by (BN, CL): the bf16-only pairs, then those FP8 has too
  if constexpr (!Op::FP8) {
    switch (k.bn * 4 + k.cl) {
      case 256 * 4 + 1: return launch_gemm<Op, false, 256, A_MN, B_MN, 1>(A, lda, B, ldb, p, stream);
      case 176 * 4 + 1: return launch_gemm<Op, false, 176, A_MN, B_MN, 1>(A, lda, B, ldb, p, stream);
      case 256 * 4 + 2: return launch_gemm<Op, false, 256, A_MN, B_MN, 2>(A, lda, B, ldb, p, stream);
      case 192 * 4 + 2: return launch_gemm<Op, false, 192, A_MN, B_MN, 2>(A, lda, B, ldb, p, stream);
      case 176 * 4 + 2: return launch_gemm<Op, false, 176, A_MN, B_MN, 2>(A, lda, B, ldb, p, stream);
      case 128 * 4 + 2: return launch_gemm<Op, false, 128, A_MN, B_MN, 2>(A, lda, B, ldb, p, stream);
    }
  }
  switch (k.bn * 4 + k.cl) {
    case 192 * 4 + 1:
      // with the plan code the promoting FP8 kernel does not hold 192 columns in registers: plans run it at 128
      if constexpr (!(Op::FP8 && Op::PLAN)) return launch_gemm<Op, false, 192, A_MN, B_MN, 1>(A, lda, B, ldb, p, stream);
      break;
    case 128 * 4 + 1: return launch_gemm<Op, false, 128, A_MN, B_MN, 1>(A, lda, B, ldb, p, stream);
  }
  return set_error("ivb_gemm_bf16: unsupported BN");
}

}  // namespace ivb

using namespace ivb;

extern "C" void ivb_set_default_2cta(int enable) { g_default_2cta = enable != 0; }

// ivb_gemm_bf16 and ivb_gemm_bf16_plan; `fn` names the entry point in messages.
static int gemm_bf16(const char* fn, const void* A, int a_mn_major, long lda, const void* B, int b_mn_major, long ldb,
                     int M, int N, int K, int epilogue, int flags, void* out0, long ld0, void* out1, long ld1,
                     const void* bias, const void* gamma, const void* aux, long ldaux, const float* rowscale,
                     int tile_n, const int* m_plan, const int* k_plan, cudaStream_t stream) {
  char msg[128];
  auto fail = [&](const char* what) {
    std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
    return set_error(msg);
  };
  if (M <= 0 || N <= 0 || K <= 0) return fail("empty problem");
  if ((N & 7) || (lda & 7) || (ldb & 7) || (ld0 & 7)) return fail("N and leading dimensions must be multiples of 8 elements");
  if (int rc = check_epilogue_args(fn, epilogue, flags, out0, out1, ld1, aux, ldaux, bias, gamma)) return rc;
  if (a_mn_major && !b_mn_major) return fail("(A MN-major, B K-major) unused");
  GemmParams p = make_params(M, N, K, epilogue, flags, out0, ld0, out1, ld1, bias, gamma, aux, ldaux, rowscale);
  const bool force2 = (flags & IVB_FLAG_2CTA) != 0, force1 = (flags & IVB_FLAG_1CTA) != 0;
  const bool forcepp = (flags & IVB_FLAG_PINGPONG) != 0;
  if ((int)force2 + (int)force1 + (int)forcepp > 1)
    return fail("IVB_FLAG_1CTA, IVB_FLAG_2CTA and IVB_FLAG_PINGPONG exclude each other");
  if (forcepp && tile_n != 0 && tile_n != PP_BN) return fail("the ping-pong kernel has tile_n 128");
  const bool plan = m_plan != nullptr || k_plan != nullptr;
  if (plan && force2) return fail("a DropPath plan needs a single-CTA kernel (no IVB_FLAG_2CTA)");
  if (m_plan != nullptr && (flags & IVB_FLAG_ACCUM)) return fail("an M plan excludes IVB_FLAG_ACCUM");
  if (k_plan != nullptr && !(a_mn_major && b_mn_major)) return fail("a K plan needs both operands MN-major (wgrad)");
  if (k_plan != nullptr && (bias != nullptr || (epilogue != IVB_EPI_BF16 && epilogue != IVB_EPI_F32)))
    return fail("a K plan needs IVB_EPI_BF16 or IVB_EPI_F32 without bias");
  if (epilogue == IVB_EPI_SWIGLU) {
    if (b_mn_major) return fail("IVB_EPI_SWIGLU needs a K-major B");
    if (N & 15) return fail("IVB_EPI_SWIGLU needs N = 2I with I a multiple of 8");
    if (bias != nullptr || out1 != nullptr) return fail("IVB_EPI_SWIGLU takes no bias and no out1");
    if (flags & (IVB_FLAG_ACCUM | IVB_FLAG_2CTA)) return fail("IVB_EPI_SWIGLU excludes IVB_FLAG_ACCUM and IVB_FLAG_2CTA");
    if (plan) return fail("IVB_EPI_SWIGLU has no DropPath plan form");
  }
  p.m_plan = m_plan;
  p.k_plan = k_plan;
  // a plan and the SwiGLU epilogue run on the single-CTA kernels, whatever the process-wide CTA-pair default
  const KernelChoice k = choose_kernel(M, N, K, flags, tile_n, false,
                                       g_default_2cta && !plan && epilogue != IVB_EPI_SWIGLU);
  if (!a_mn_major && !b_mn_major) return dispatch<OpBf16, false, false>(k, A, lda, B, ldb, p, stream);
  if (!a_mn_major) return dispatch<OpBf16, false, true>(k, A, lda, B, ldb, p, stream);
  return dispatch<OpBf16, true, true>(k, A, lda, B, ldb, p, stream);
}

extern "C" int ivb_gemm_bf16(const void* A, int a_mn_major, long lda, const void* B,
                             int b_mn_major, long ldb, int M, int N, int K, int epilogue,
                             int flags, void* out0, long ld0, void* out1, long ld1,
                             const void* bias, const void* gamma, const void* aux, long ldaux,
                             const float* rowscale, int tile_n, void* stream) {
  return gemm_bf16("ivb_gemm_bf16", A, a_mn_major, lda, B, b_mn_major, ldb, M, N, K, epilogue, flags, out0, ld0, out1,
                   ld1, bias, gamma, aux, ldaux, rowscale, tile_n, nullptr, nullptr,
                   reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_gemm_bf16_plan(const void* A, int a_mn_major, long lda, const void* B, int b_mn_major, long ldb,
                                  int M, int N, int K, int epilogue, int flags, void* out0, long ld0, void* out1,
                                  long ld1, const void* bias, const void* gamma, const void* aux, long ldaux,
                                  const float* rowscale, int tile_n, const int* m_plan, const int* k_plan,
                                  void* stream) {
  return gemm_bf16("ivb_gemm_bf16_plan", A, a_mn_major, lda, B, b_mn_major, ldb, M, N, K, epilogue, flags, out0, ld0,
                   out1, ld1, bias, gamma, aux, ldaux, rowscale, tile_n, m_plan, k_plan,
                   reinterpret_cast<cudaStream_t>(stream));
}

// ivb_gemm_fp8 and ivb_gemm_fp8_plan; `fn` names the entry point in messages.
static int gemm_fp8(const char* fn, const void* A, int a_mn_major, long lda, int a_format, const float* a_scale_inv,
                    const void* B, int b_mn_major, long ldb, const float* b_scale_inv, int M, int N, int K, int epilogue,
                    int flags, void* out0, long ld0, void* out1, long ld1, const void* bias, const void* gamma,
                    const void* aux, long ldaux, const float* rowscale, int tile_n, const int* m_plan,
                    cudaStream_t stream) {
  char msg[128];
  auto fail = [&](const char* what) {
    std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
    return set_error(msg);
  };
  if (M <= 0 || N <= 0 || K <= 0) return fail("empty problem");
  if (a_mn_major || b_mn_major) return fail("both operands must be K-major");
  if ((lda & 15) || (ldb & 15)) return fail("lda and ldb must be multiples of 16 elements");
  if ((N & 7) || (ld0 & 7)) return fail("N and ld0 must be multiples of 8 elements");
  if (a_format != IVB_FP8_E4M3 && a_format != IVB_FP8_E5M2) return fail("unknown a_format");
  if (epilogue == IVB_EPI_SWIGLU) return fail("IVB_EPI_SWIGLU is bf16 only (ivb_gemm_bf16)");
  if (a_scale_inv == nullptr || b_scale_inv == nullptr) return fail("scale_inv pointers are null");
  const bool vec = (flags & IVB_FLAG_FP8_VECTOR_SCALES) != 0;
  if (vec && a_format != IVB_FP8_E4M3) return fail("vector scales need an E4M3 A operand");
  if (vec && ((reinterpret_cast<uintptr_t>(a_scale_inv) | reinterpret_cast<uintptr_t>(b_scale_inv)) & 7))
    return fail("scale vectors must be 8-byte aligned");
  if (int rc = check_epilogue_args(fn, epilogue, flags, out0, out1, ld1, aux, ldaux, bias, gamma)) return rc;
  const bool force1 = (flags & IVB_FLAG_1CTA) != 0, forcepp = (flags & IVB_FLAG_PINGPONG) != 0;
  if (flags & IVB_FLAG_2CTA) return fail("no CTA-pair kernel");
  if (force1 && forcepp) return fail("IVB_FLAG_1CTA and IVB_FLAG_PINGPONG exclude each other");
  if (tile_n != 0 && tile_n != 128 && tile_n != 192) return fail("tile_n must be 0, 128 or 192");
  if (forcepp && tile_n == 192) return fail("the ping-pong kernel has tile_n 128");
  // a per-tensor scale comes from the whole tensor's amax, which the zeroed rows of dropped clips would change
  if (m_plan != nullptr && !vec) return fail("a DropPath plan needs IVB_FLAG_FP8_VECTOR_SCALES");
  if (m_plan != nullptr && (flags & IVB_FLAG_ACCUM)) return fail("an M plan excludes IVB_FLAG_ACCUM");
  if (m_plan != nullptr && tile_n == 192) return fail("a DropPath plan runs the FP8 GEMM at tile_n 128");
  GemmParams p = make_params(M, N, K, epilogue, flags, out0, ld0, out1, ld1, bias, gamma, aux, ldaux, rowscale);
  p.a_scale_inv = a_scale_inv;
  p.b_scale_inv = b_scale_inv;
  p.m_plan = m_plan;
  KernelChoice k = choose_kernel(M, N, K, flags, tile_n, true, false);
  if (m_plan != nullptr) k.bn = 128;   // the cooperative kernel's width under a plan (dispatch); the ping-pong one's
  if (m_plan != nullptr) return dispatch<OpPlannedFp8, false, false>(k, A, lda, B, ldb, p, stream);
  if (vec) return dispatch<OpVecFp8, false, false>(k, A, lda, B, ldb, p, stream);
  if (a_format == IVB_FP8_E5M2) return dispatch<OpFp8<true>, false, false>(k, A, lda, B, ldb, p, stream);
  return dispatch<OpFp8<false>, false, false>(k, A, lda, B, ldb, p, stream);
}

extern "C" int ivb_gemm_fp8(const void* A, int a_mn_major, long lda, int a_format, const float* a_scale_inv,
                            const void* B, int b_mn_major, long ldb, const float* b_scale_inv, int M, int N, int K,
                            int epilogue, int flags, void* out0, long ld0, void* out1, long ld1, const void* bias,
                            const void* gamma, const void* aux, long ldaux, const float* rowscale, int tile_n,
                            void* stream) {
  return gemm_fp8("ivb_gemm_fp8", A, a_mn_major, lda, a_format, a_scale_inv, B, b_mn_major, ldb, b_scale_inv, M, N, K,
                  epilogue, flags, out0, ld0, out1, ld1, bias, gamma, aux, ldaux, rowscale, tile_n, nullptr,
                  reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ivb_gemm_fp8_plan(const void* A, int a_mn_major, long lda, int a_format, const float* a_scale_inv,
                                 const void* B, int b_mn_major, long ldb, const float* b_scale_inv, int M, int N, int K,
                                 int epilogue, int flags, void* out0, long ld0, void* out1, long ld1, const void* bias,
                                 const void* gamma, const void* aux, long ldaux, const float* rowscale, int tile_n,
                                 const int* m_plan, void* stream) {
  return gemm_fp8("ivb_gemm_fp8_plan", A, a_mn_major, lda, a_format, a_scale_inv, B, b_mn_major, ldb, b_scale_inv, M, N,
                  K, epilogue, flags, out0, ld0, out1, ld1, bias, gamma, aux, ldaux, rowscale, tile_n, m_plan,
                  reinterpret_cast<cudaStream_t>(stream));
}

// The weight gradient over tokens from block-scaled E4M3 operands (ivb_fp8_quantize_blocks_t's transposed copies): the
// promoting cooperative kernel at BN = 128 with OpBlockFp8, with or without a K plan.
extern "C" int ivb_gemm_fp8_wgrad(const void* A_t, long lda, const float* a_scale_inv, const void* B_t, long ldb,
                                  const float* b_scale_inv, int M, int N, int K, int epilogue, int flags, void* out0,
                                  long ld0, const int* k_plan, void* stream) {
  const char* fn = "ivb_gemm_fp8_wgrad";
  char msg[128];
  auto fail = [&](const char* what) {
    std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
    return set_error(msg);
  };
  if (M <= 0 || N <= 0 || K <= 0) return fail("empty problem");
  if (A_t == nullptr || B_t == nullptr) return fail("A_t or B_t is null");
  if ((lda & 15) || (ldb & 15) || lda < K || ldb < K) return fail("lda and ldb must be multiples of 16 elements and >= K");
  if ((M & 7) || (N & 7)) return fail("M and N must be multiples of 8");
  if ((ld0 & 7) || ld0 < N) return fail("ld0 must be a multiple of 8 elements and >= N");
  if (a_scale_inv == nullptr || b_scale_inv == nullptr) return fail("scale_inv pointers are null");
  if (misaligned(16, a_scale_inv, b_scale_inv)) return fail("scale vectors must be 16-byte aligned");
  if (epilogue != IVB_EPI_BF16 && epilogue != IVB_EPI_F32) return fail("epilogue must be IVB_EPI_BF16 or IVB_EPI_F32");
  if (flags & ~IVB_FLAG_ACCUM) return fail("the only flag is IVB_FLAG_ACCUM (one kernel form: cooperative, 1 CTA)");
  if (int rc = check_epilogue_args(fn, epilogue, flags, out0, nullptr, 0, nullptr, 0, nullptr, nullptr)) return rc;
  GemmParams p = make_params(M, N, K, epilogue, flags, out0, ld0, nullptr, 0, nullptr, nullptr, nullptr, 0, nullptr);
  p.a_scale_inv = a_scale_inv;
  p.b_scale_inv = b_scale_inv;
  p.k_plan = k_plan;
  return launch_gemm<OpBlockFp8, false, 128, false, false, 1>(A_t, lda, B_t, ldb, p, reinterpret_cast<cudaStream_t>(stream));
}
