// ivb_runtime.cu — status reporting, launch accounting and TMA tensor-map construction.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>

#include <stdlib.h>

#include "ivb_internal.h"

namespace ivb {

static thread_local char g_err[512] = "";
static std::atomic<long> g_launches{0};

int set_error(const char* msg) {
  std::snprintf(g_err, sizeof(g_err), "%s", msg);
  return 1;
}
int set_error_cuda(const char* what, cudaError_t e) {
  std::snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
  return 2;
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("IVB_PDL"); return e != nullptr && atoi(e) != 0; }();
  return on;
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = (PFN_encodeTiled)p;
  });
  return fn;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer,
                 long ld_elems, uint32_t box_inner, uint32_t box_outer, int elem_bytes) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error("TMA base pointer must be 16-byte aligned");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld_elems) * elem_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dtype = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = enc(out, dtype, 2, const_cast<void*>(base), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    std::snprintf(buf, sizeof(buf),
                  "cuTensorMapEncodeTiled(2d) failed rc=%d dims=(%llu,%llu) ld=%ld box=(%u,%u)",
                  (int)r, (unsigned long long)inner, (unsigned long long)outer, ld_elems,
                  box_inner, box_outer);
    return set_error(buf);
  }
  return 0;
}

int make_tmap_4d(CUtensorMap* out, const void* base, const uint64_t dims_[4],
                 const long strides_elems[3], const uint32_t box_[4], int elem_bytes, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error("TMA base pointer must be 16-byte aligned");
  cuuint64_t dims[4] = {dims_[0], dims_[1], dims_[2], dims_[3]};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(strides_elems[0]) * elem_bytes,
                           static_cast<cuuint64_t>(strides_elems[1]) * elem_bytes,
                           static_cast<cuuint64_t>(strides_elems[2]) * elem_bytes};
  cuuint32_t box[4] = {box_[0], box_[1], box_[2], box_[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapDataType dtype = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const CUtensorMapSwizzle swz = swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(out, dtype, 4, const_cast<void*>(base), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[200];
    std::snprintf(buf, sizeof(buf),
                  "cuTensorMapEncodeTiled(4d) failed rc=%d dims=(%llu,%llu,%llu,%llu)", (int)r,
                  (unsigned long long)dims[0], (unsigned long long)dims[1],
                  (unsigned long long)dims[2], (unsigned long long)dims[3]);
    return set_error(buf);
  }
  return 0;
}

}  // namespace ivb

using namespace ivb;

extern "C" const char* ivb_last_error(void) { return g_err; }
extern "C" int ivb_version(void) { return IVB_VERSION; }
extern "C" long ivb_launch_count(void) { return g_launches.load(); }
extern "C" void ivb_reset_launch_count(void) { g_launches.store(0); }
extern "C" int ivb_device_check(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) return set_error("libivb200: no CUDA device (there is no CPU fallback)");
  int dev = 0, major = 0, minor = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) return set_error("libivb200: device is not compute capability 9.0 (sm_90a only)");
  return 0;
}
