// ivb_internal.h — shared host-side helpers of libivb200 (not part of the public C ABI).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ivb200.h"

namespace ivb {

// error reporting: every entry point returns 0 or a non-zero status; text via ivb_last_error().
int set_error(const char* msg);
int set_error_cuda(const char* what, cudaError_t e);
void count_launch();                 // bumps the library-wide launch counter
int num_sms();
// Raises Kern's dynamic shared-memory limit to `bytes` on the current device, once per device: the device is marked
// only after the call succeeds, so a failed attempt is retried (and reported) by the next launch.
template <auto Kern>
inline int raise_smem_limit(int bytes, const char* what) {
  static bool set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  const bool tracked = dev >= 0 && dev < 64;
  if (tracked && set[dev]) return 0;
  const cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_error_cuda(what, e);
  if (tracked) set[dev] = true;
  return 0;
}
// True when one of the pointers is not a multiple of `bytes` (a power of two); null pointers count as aligned.
template <typename... P>
inline bool misaligned(uintptr_t bytes, const P*... ps) {
  return ((reinterpret_cast<uintptr_t>(ps) & (bytes - 1)) | ... | 0u) != 0;
}
// Grid of a persistent row kernel: one CTA per `rows_per_cta` rows, at most `per_sm` CTAs per SM, at least one.
inline int persistent_grid(long rows, int rows_per_cta, int per_sm) {
  const long blocks = (rows + rows_per_cta - 1) / rows_per_cta;
  const long cap = static_cast<long>(num_sms()) * per_sm;
  return static_cast<int>(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

// Fixed-order scalar sums (the losses and dtemp of ivb_loss.cu) through the one per-device reduction scratch of
// ivb_colred.cuh, which lives in ivb_norm.cu: each CTA of a kernel stores its partial in slot blockIdx.x of
// scalar_slots(n), and scalar_finish(n, dst) then adds slots [0, n) in slot order into *dst (nothing when dst is null).
// scalar_slots returns null, with `who` as the error text, when n slots do not fit or the address cannot be read.
float* scalar_slots(long n, const char* who);
int scalar_finish(int n, float* dst, cudaStream_t stream);
// The same scratch for column sums of another translation unit (ivb_embed.cu): colred_cols(n, D) is the base of n
// partial rows of D fp32 (slot s at s * D; null as scalar_slots), and colred_cols_finish(n, D, dst) adds slots [0, n)
// in slot order into dst[0, D).
float* colred_cols(long n, int D, const char* who);
int colred_cols_finish(int n, int D, float* dst, cudaStream_t stream);

// Programmatic dependent launch (PDL) is opt-in: pdl_enabled() is true only when IVB_PDL is set to a non-zero value.
// A PDL-launched kernel may be scheduled while the previous kernel of the stream is still draining, so it must execute
// pdl_wait() (ivb_ptx.cuh) before its first global-memory access; only such kernels are launched with ALLOW_PDL.
// ~1 100 of the ~1 500 launches of a training step allow it; the launch/drain gap between them was ~5 us each.
bool pdl_enabled();
enum LaunchPdl : bool { NO_PDL = false, ALLOW_PDL = true };

// The one launch path of the library: launches `kern` (in clusters of CLUSTER CTAs along x when CLUSTER > 1), with the
// PDL attribute when `pdl` allows it and pdl_enabled(), and counts it.  Returns 0, or a status whose ivb_last_error()
// text is `name` and the CUDA error.
template <int CLUSTER = 1, typename... KArgs, typename... Args>
inline int launch(const char* name, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                  LaunchPdl pdl, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (CLUSTER > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = CLUSTER; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl && pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
  const cudaError_t last = cudaGetLastError();   // clears the launch's error, and reports one left by earlier work
  if (e == cudaSuccess) e = last;
  if (e != cudaSuccess) return set_error_cuda(name, e);
  count_launch();
  return 0;
}

// cuTensorMapEncodeTiled through cudaGetDriverEntryPoint (no link-time libcuda dependency).
// 2-D bf16 (elem_bytes 2) or fp8 (elem_bytes 1) tensor, dims {inner, outer}, row pitch ld_elems, 128-byte swizzle,
// zero OOB fill.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer,
                 long ld_elems, uint32_t box_inner, uint32_t box_outer, int elem_bytes = 2);
// 4-D bf16 (elem_bytes 2) or fp8 (elem_bytes 1) tensor (dims[0] innermost/contiguous), strides in elements for dims
// 1..3, 128-byte (or, swizzle_bytes 64, 64-byte) swizzle, zero OOB fill.
int make_tmap_4d(CUtensorMap* out, const void* base, const uint64_t dims[4],
                 const long strides_elems[3], const uint32_t box[4], int elem_bytes = 2, int swizzle_bytes = 128);

}  // namespace ivb
