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
// CL = 2 (the CTA-pair form, IVB_FLAG_2CTA / ivb_set_default_2cta): a cluster of two CTAs on neighbouring SMs computes
// a 256 x BN tile.  Each CTA loads its own 128 A rows and HALF of the B tile, which TMA multicasts into both CTAs'
// rings, so B is read from L2 once per 256 rows instead of once per 128.  A stage is refilled only when the MMA
// warpgroups of BOTH CTAs released it (each arrives on its own and on the peer's empty barrier).
#include "ivb_gemm_common.cuh"

namespace ivb {

constexpr int BM = 128;
constexpr int BK = 64;                 // 64 bf16 = 128 B = one swizzle atom
constexpr int GEMM_THREADS = 384;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB either major
constexpr int EPI_PITCH = 36;               // floats per staged row: 32 columns + 4 (bank spread, 16-B rows)
constexpr int EPI_BYTES = 8 * 16 * EPI_PITCH * 4;  // one 16 x 32 fp32 staging tile per MMA warp

template <int BN, bool B_MN>
struct GemmCfg {
  static constexpr int B_ATOMS = (BN + 63) / 64;
  static constexpr int B_STAGE_BYTES = B_MN ? B_ATOMS * 64 * 128 : BN * 128;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES_RAW = (227 * 1024 - EPI_BYTES - 1024 - 256) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// ------------------------------------------------------------------ the kernel
template <int BN, bool A_MN, bool B_MN, int CL>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using Cfg = GemmCfg<BN, B_MN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  float* epi = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + EPI_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0;   // 128-row half of the cluster's tile
  const int cid = blockIdx.x / CL, ncl = gridDim.x / CL;   // tiles are walked per cluster
  const int num_m = (p.M + CL * BM - 1) / (CL * BM);
  const int num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2 * CL);  // one arrival per MMA warpgroup of the cluster
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (CL == 2) cluster_sync_all();   // the peer's barriers exist before any multicast or remote arrive reaches them
  pdl_wait();
  pdl_launch_dependents();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ===================== TMA producer =====================
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = cid; tile < num_tiles; tile += ncl) {
        const int m0 = (tile / num_n) * (CL * BM) + rank * BM;
        const int n0 = (tile % num_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
          uint8_t* sb = smem_b + stage * Cfg::B_STAGE_BYTES;
          const int k0 = kb * BK;
          if (!A_MN) {
            tma_load_2d(sa, &tmA, k0, m0, &full[stage]);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              tma_load_2d(sa + i * 8192, &tmA, m0 + i * 64, k0, &full[stage]);
          }
          if (CL == 1) {
            if (!B_MN) {
              tma_load_2d(sb, &tmB, k0, n0, &full[stage]);
            } else {
#pragma unroll
              for (int i = 0; i < Cfg::B_ATOMS; ++i)
                tma_load_2d(sb + i * 8192, &tmB, n0 + i * 64, k0, &full[stage]);
            }
          } else {  // this CTA's half of B, into both CTAs (K-major: BN/2 rows; MN-major: every other 64-wide atom)
            if (!B_MN) {
              tma_load_2d_mc(sb + rank * (BN / 2) * 128, &tmB, k0, n0 + rank * (BN / 2), &full[stage], 0x3);
            } else {
#pragma unroll
              for (int i = 0; i < Cfg::B_ATOMS; ++i)
                if ((i & 1) == static_cast<int>(rank))
                  tma_load_2d_mc(sb + i * 8192, &tmB, n0 + i * 64, k0, &full[stage], 0x3);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================== MMA + epilogue warpgroups =====================
    const int cw = wg - 1;              // rows [64*cw, 64*cw + 64) of the tile
    const int wr = warp & 3;            // warp inside the warpgroup: accumulator rows [16*wr, 16*wr + 16)
    const bool signal = (threadIdx.x & 127) == 0;
    auto release = [&](int s_) {   // this warpgroup no longer reads stage s_ (of either CTA's ring)
      if (!signal) return;
      mbar_arrive(&empty[s_]);
      if (CL == 2) mbar_arrive_cluster(mapa_u32(smem_u32(&empty[s_]), rank ^ 1));
    };
    float* st = epi + (warp - 4) * 16 * EPI_PITCH;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = cid; tile < num_tiles; tile += ncl) {
      const int m0 = (tile / num_n) * (CL * BM) + rank * BM;
      const int n0 = (tile % num_n) * BN;
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES);
        const uint32_t sb = smem_u32(smem_b + stage * Cfg::B_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t ad = A_MN ? gmma_desc(sa + cw * 8192 + k * 2048, 8192, 1024)
                                   : gmma_desc(sa + cw * 8192 + k * 32, 16, 1024);
          const uint64_t bd = B_MN ? gmma_desc(sb + k * 2048, 8192, 1024) : gmma_desc(sb + k * 32, 16, 1024);
          Wgmma<BN>::template ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd, (kb > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        if (kb > 0) {  // the MMAs of the previous k-block retired: its smem slot is free
          wgmma_wait<1>();
          release(prev);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc, BN / 2);
      release(prev);

      // epilogue, 32 columns at a time: fragments -> staging tile -> one 16-column row segment per thread
      const long row = m0 + cw * 64 + wr * 16 + (lane >> 1);
      const int half = lane & 1;
#pragma unroll
      for (int c = 0; c < (BN + 31) / 32; ++c) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * c + jj;
          if (j < BN / 8) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
              *reinterpret_cast<float2*>(st + ((lane >> 2) + 8 * h) * EPI_PITCH + 8 * jj + 2 * (lane & 3)) =
                  make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
        }
        __syncwarp();
        const int col = c * 32 + half * 16;
        if (col < BN && row < p.M) {
          uint32_t bits[16];
          const float* src = st + (lane >> 1) * EPI_PITCH + half * 16;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 v = reinterpret_cast<const float4*>(src)[i];
            bits[4 * i] = __float_as_uint(v.x); bits[4 * i + 1] = __float_as_uint(v.y);
            bits[4 * i + 2] = __float_as_uint(v.z); bits[4 * i + 3] = __float_as_uint(v.w);
          }
          epilogue_chunk<16>(p, bits, row, n0 + col);
        }
        __syncwarp();
      }
    }
  }
  if (CL == 2) cluster_sync_all();   // the peer may still multicast into / arrive on this CTA's ring
}

// ------------------------------------------------------------------ host side
template <int BN, bool A_MN, bool B_MN, int CL>
static int launch_gemm(const void* A, long lda, const void* B, long ldb, const GemmParams& p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN, B_MN>;
  CUtensorMap tmA, tmB;
  int rc;
  if (!A_MN) rc = make_tmap_2d(&tmA, A, (uint64_t)p.K, (uint64_t)p.M, lda, 64, BM);
  else       rc = make_tmap_2d(&tmA, A, (uint64_t)p.M, (uint64_t)p.K, lda, 64, 64);
  if (rc) return rc;
  if (!B_MN) rc = make_tmap_2d(&tmB, B, (uint64_t)p.K, (uint64_t)p.N, ldb, 64, BN / CL);
  else       rc = make_tmap_2d(&tmB, B, (uint64_t)p.N, (uint64_t)p.K, ldb, 64, 64);
  if (rc) return rc;
  auto kern = gemm_bf16_kernel<BN, A_MN, B_MN, CL>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(gemm)", e);
  }
  const int num_tiles = ((p.M + CL * BM - 1) / (CL * BM)) * ((p.N + BN - 1) / BN);
  int clusters = num_sms() / CL;
  if (clusters > num_tiles) clusters = num_tiles;
  cudaError_t le;
  if (CL == 1) {
    le = launch_pdl(kern, dim3(clusters), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, tmA, tmB, p);
  } else {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(clusters * CL);
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    le = cudaLaunchKernelEx(&cfg, kern, tmA, tmB, p);
  }
  if (le != cudaSuccess) return set_error_cuda("launch(gemm_bf16_kernel)", le);
  count_launch();
  return check_launch("gemm_bf16_kernel");
}

template <bool A_MN, bool B_MN, int CL>
static int dispatch_bn(int bn, const void* A, long lda, const void* B, long ldb,
                       const GemmParams& p, cudaStream_t stream) {
  switch (bn) {
    case 256: return launch_gemm<256, A_MN, B_MN, CL>(A, lda, B, ldb, p, stream);
    case 192: return launch_gemm<192, A_MN, B_MN, CL>(A, lda, B, ldb, p, stream);
    case 176: return launch_gemm<176, A_MN, B_MN, CL>(A, lda, B, ldb, p, stream);
    case 128: return launch_gemm<128, A_MN, B_MN, CL>(A, lda, B, ldb, p, stream);
    default: return set_error("ivb_gemm_bf16: unsupported BN");
  }
}

template <int CL>
static int dispatch_major(int bn, bool a_mn, bool b_mn, const void* A, long lda, const void* B, long ldb,
                          const GemmParams& p, cudaStream_t stream) {
  if (!a_mn && !b_mn) return dispatch_bn<false, false, CL>(bn, A, lda, B, ldb, p, stream);
  if (!a_mn && b_mn) return dispatch_bn<false, true, CL>(bn, A, lda, B, ldb, p, stream);
  return dispatch_bn<true, true, CL>(bn, A, lda, B, ldb, p, stream);
}

// Pick the N tile that wastes the fewest padded columns / partial waves.
static int choose_bn(int M, int N, int cl) {
  const int cand[4] = {256, 192, 176, 128};
  const int sms = num_sms() / cl;
  const int num_m = (M + cl * BM - 1) / (cl * BM);
  double best = 1e30;
  int best_bn = 256;
  for (int i = 0; i < 4; ++i) {
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

static bool g_default_2cta = false;

}  // namespace ivb

using namespace ivb;

extern "C" void ivb_set_default_2cta(int enable) { g_default_2cta = enable != 0; }

extern "C" int ivb_gemm_bf16(const void* A, int a_mn_major, long lda, const void* B,
                             int b_mn_major, long ldb, int M, int N, int K, int epilogue,
                             int flags, void* out0, long ld0, void* out1, long ld1,
                             const void* bias, const void* gamma, const void* aux, long ldaux,
                             const float* rowscale, int tile_n, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || N <= 0 || K <= 0) return set_error("ivb_gemm_bf16: empty problem");
  if ((N & 7) || (lda & 7) || (ldb & 7) || (ld0 & 7))
    return set_error("ivb_gemm_bf16: N and leading dimensions must be multiples of 8 elements");
  if (out0 == nullptr) return set_error("ivb_gemm_bf16: out0 is null");
  if ((epilogue == IVB_EPI_RESID || epilogue == IVB_EPI_GELU_BWD) && aux == nullptr)
    return set_error("ivb_gemm_bf16: epilogue needs aux");
  if (a_mn_major && !b_mn_major) return set_error("ivb_gemm_bf16: (A MN-major, B K-major) unused");
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.epi = epilogue; p.flags = flags;
  p.out0 = out0; p.ld0 = ld0; p.out1 = out1; p.ld1 = ld1;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.gamma = reinterpret_cast<const __nv_bfloat16*>(gamma);
  p.aux = aux; p.ldaux = ldaux; p.rowscale = rowscale;
  // kernel selection: the CTA-pair (cluster) kernel when forced, or by default for problems tall enough to fill
  // 256-row tiles; the single-CTA kernel otherwise / when IVB_FLAG_1CTA is set.
  const bool force2 = (flags & IVB_FLAG_2CTA) != 0, force1 = (flags & IVB_FLAG_1CTA) != 0;
  const int cl = (force2 || (!force1 && g_default_2cta && M >= 512)) ? 2 : 1;
  const int bn = tile_n > 0 ? tile_n : choose_bn(M, N, cl);
  if (cl == 2) return dispatch_major<2>(bn, a_mn_major != 0, b_mn_major != 0, A, lda, B, ldb, p, stream);
  return dispatch_major<1>(bn, a_mn_major != 0, b_mn_major != 0, A, lda, B, ldb, p, stream);
}
