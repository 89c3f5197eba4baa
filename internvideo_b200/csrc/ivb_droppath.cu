// ivb_droppath.cu — the DropPath (stochastic depth) plan of a training step: which 128-row tiles and 64-row k-blocks of
// each block branch hold a row whose factor the draw kept, so that the GEMMs (ivb_gemm_bf16_plan) skip the work of the
// rows it dropped.  Read on the device from the same factors the residual epilogues multiply by: no host read, and a
// captured CUDA graph stays valid while the draws change.
#include "ivb_internal.h"

namespace ivb {

constexpr int PLAN_THREADS = 256;

// One CTA per branch.  Each warp marks the k-blocks it owns live or dead (one ballot per 32 rows), then warp 0 lists
// the row tiles and warp 1 the k-blocks.
__global__ void __launch_bounds__(PLAN_THREADS)
droppath_plan_kernel(const float* __restrict__ rowscale, long ld_rs, int M, int* __restrict__ plan, long ld_plan) {
  extern __shared__ uint8_t kb_live[];
  const float* rs = rowscale + blockIdx.x * ld_rs;
  int* out = plan + blockIdx.x * ld_plan;
  const int nm = (M + 127) / 128, nk = (M + 63) / 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int kb = warp; kb < nk; kb += PLAN_THREADS / 32) {
    bool live = false;
    for (int r = kb * 64 + lane; r < min(M, kb * 64 + 64); r += 32) live |= rs[r] != 0.0f;
    live = __any_sync(0xffffffffu, live);
    if (lane == 0) kb_live[kb] = live;
  }
  __syncthreads();
  if (threadIdx.x == 0) {          // row tiles: live ascending, then dead ascending; then the live count
    int c = 0;
    for (int t = 0; t < nm; ++t)
      if (kb_live[2 * t] || (2 * t + 1 < nk && kb_live[2 * t + 1])) out[c++] = t;
    const int live = c;
    for (int t = 0; t < nm; ++t)
      if (!(kb_live[2 * t] || (2 * t + 1 < nk && kb_live[2 * t + 1]))) out[c++] = t;
    out[nm] = live;
  } else if (threadIdx.x == 32) {  // live k-blocks ascending; their count after the nk slots
    int* kl = out + nm + 1;
    int c = 0;
    for (int kb = 0; kb < nk; ++kb)
      if (kb_live[kb]) kl[c++] = kb;
    kl[nk] = c;
  }
}

}  // namespace ivb

using namespace ivb;

extern "C" long ivb_droppath_plan_ints(int M) { return M <= 0 ? 0 : (M + 127) / 128 + (M + 63) / 64 + 2; }

extern "C" int ivb_droppath_plan(const float* rowscale, long ld_rs, int branches, int M, int* plan, long ld_plan,
                                 void* stream) {
  if (branches <= 0 || M <= 0) return 0;
  const long nk = (M + 63) / 64;
  if (ld_rs < M || ld_plan < ivb_droppath_plan_ints(M))
    return set_error("ivb_droppath_plan: ld_rs must be >= M and ld_plan >= ivb_droppath_plan_ints(M)");
  if (nk > 48 * 1024) return set_error("ivb_droppath_plan: M above 48K k-blocks of 64 rows");
  return launch("droppath_plan_kernel", droppath_plan_kernel, branches, PLAN_THREADS, static_cast<size_t>(nk),
                reinterpret_cast<cudaStream_t>(stream), NO_PDL, rowscale, ld_rs, M, plan, ld_plan);
}
