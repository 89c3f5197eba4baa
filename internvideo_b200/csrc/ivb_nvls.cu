// In-switch gradient all-reduce over an NVLink multicast mapping (NVLS), written for the data-parallel engine
// (SURVEY §8 row a19/e: the reference's DDP/DeepSpeed gradient reduction, run_pretraining.py:378 + utils.py:814-834).
//
// Why not ncclAllReduce: on an 8-GPU NVSwitch box NCCL's NVLS all-reduce runs 24 channels = 24 CTAs that each hold an SM
// for the whole bucket; under the persistent one-CTA-per-SM GEMMs of the backward pass those SMs are taken from the GEMMs.  The gradients only need ~2 GB per ~75 ms of backward, so this kernel
// trades bandwidth for footprint: a handful of CTAs, no staging buffers, no protocol — the switch does the arithmetic.
//
// Every rank maps the SAME symmetric buffer (the flat bf16 gradient buffer) through a multicast address `mc`.  Two-shot:
//   1. barrier (every rank's producers of this range have finished — stream order on each rank + the flag exchange here)
//   2. rank r owns the r-th 1/world slice:  v = multimem.ld_reduce.add.acc::f32 [mc + i]   (the switch reads all replicas,
//      adds them in fp32, returns one bf16x2 x4 vector)  ;  multimem.st [mc + i], v       (the switch writes all replicas)
//   3. barrier (every slice has landed everywhere)
// Every replica receives the same bits for every element (one reduction per address, broadcast), so data-parallel
// replicas stay bit-identical by construction.
//
// Flags: `flags[p]` is rank p's flag array (peer-mapped, zero-initialised, one uint32 per (CTA, source rank)).  A signal is
// CAS 0->1 with release.sys on the TARGET's array, a wait is CAS 1->0 with acquire.sys on the OWN array: self-resetting, so
// a captured CUDA graph can replay the kernel.  Launch order of these kernels must be the same on every rank (it is: the
// engine launches buckets in backward order on one communication stream).
#include "ivb_internal.h"

namespace ivb {

constexpr int NVLS_THREADS = 512;
constexpr int NVLS_MAX_BLOCKS = 64;
constexpr int NVLS_MAX_WORLD = 16;
constexpr unsigned long long NVLS_SPIN_LIMIT_NS = 120ull * 1000 * 1000 * 1000;   // a peer 2 minutes late: trap, do not hang

__device__ __forceinline__ unsigned long long nvls_now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ void nvls_flag_put(uint32_t* addr) {     // peer's slot: 0 -> 1
  uint32_t old;
  const unsigned long long t0 = nvls_now_ns();
  do {
    asm volatile("atom.global.release.sys.cas.b32 %0, [%1], 0, 1;" : "=r"(old) : "l"(addr) : "memory");
    if (old != 0 && nvls_now_ns() - t0 > NVLS_SPIN_LIMIT_NS) __trap();
  } while (old != 0);
}
__device__ __forceinline__ void nvls_flag_wait(uint32_t* addr) {    // own slot: 1 -> 0
  uint32_t old;
  const unsigned long long t0 = nvls_now_ns();
  do {
    asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], 1, 0;" : "=r"(old) : "l"(addr) : "memory");
    if (old != 1 && nvls_now_ns() - t0 > NVLS_SPIN_LIMIT_NS) __trap();
  } while (old != 1);
}

// CTA `blockIdx.x` of every rank meets CTA `blockIdx.x` of every other rank.
__device__ __forceinline__ void nvls_barrier(uint32_t* const* flags, int rank, int world) {
  __syncthreads();                       // this CTA's earlier writes happen-before the releasing CAS (cumulativity)
  if (threadIdx.x < world) {
    const int peer = threadIdx.x;
    nvls_flag_put(flags[peer] + blockIdx.x * world + rank);
    nvls_flag_wait(flags[rank] + blockIdx.x * world + peer);
  }
  __syncthreads();
}

__device__ __forceinline__ void mm_ld_reduce(const uint4* mc, uint4& v) {
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
}
__device__ __forceinline__ void mm_st(uint4* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1, %2, %3, %4};"
               ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// mc: multicast address of element 0 of the range; nvec: 16-byte vectors in the range.
__global__ void __launch_bounds__(NVLS_THREADS)
nvls_allreduce_bf16_kernel(uint4* __restrict__ mc, long nvec, uint32_t* const* __restrict__ flags, int rank, int world) {
  nvls_barrier(flags, rank, world);
  const long per = (nvec + world - 1) / world;
  const long v0 = per * rank;
  const long v1 = (v0 + per < nvec) ? v0 + per : nvec;
  const long stride = static_cast<long>(gridDim.x) * NVLS_THREADS;
  long i = v0 + static_cast<long>(blockIdx.x) * NVLS_THREADS + threadIdx.x;
  // four independent reductions in flight per thread: the round trip through the switch is microseconds long
  for (; i + 3 * stride < v1; i += 4 * stride) {
    uint4 a, b, c, d;
    mm_ld_reduce(mc + i, a);
    mm_ld_reduce(mc + i + stride, b);
    mm_ld_reduce(mc + i + 2 * stride, c);
    mm_ld_reduce(mc + i + 3 * stride, d);
    mm_st(mc + i, a);
    mm_st(mc + i + stride, b);
    mm_st(mc + i + 2 * stride, c);
    mm_st(mc + i + 3 * stride, d);
  }
  for (; i < v1; i += stride) {
    uint4 a;
    mm_ld_reduce(mc + i, a);
    mm_st(mc + i, a);
  }
  nvls_barrier(flags, rank, world);
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_nvls_allreduce_bf16(void* mc_base, long elem_off, long numel, const void* flag_ptrs_dev, int rank,
                                       int world, int nblocks, void* stream) {
  if (mc_base == nullptr || flag_ptrs_dev == nullptr) return set_error("ivb_nvls_allreduce_bf16: null multicast / flag pointer");
  if (world < 2 || world > NVLS_MAX_WORLD || rank < 0 || rank >= world)
    return set_error("ivb_nvls_allreduce_bf16: world must be 2..16 and 0 <= rank < world");
  if (nblocks < 1 || nblocks > NVLS_MAX_BLOCKS) return set_error("ivb_nvls_allreduce_bf16: nblocks must be 1..64");
  if (elem_off < 0 || numel < 0 || (elem_off % 8) != 0 || (numel % 8) != 0)
    return set_error("ivb_nvls_allreduce_bf16: range must start and end on 16-byte boundaries (8 bf16 elements)");
  if (numel == 0) return 0;
  uint4* mc = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(mc_base) + elem_off);
  const long nvec = numel / 8;
  uint32_t* const* flags = reinterpret_cast<uint32_t* const*>(flag_ptrs_dev);
  nvls_allreduce_bf16_kernel<<<nblocks, NVLS_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(mc, nvec, flags, rank, world);
  count_launch();
  return check_launch("nvls_allreduce_bf16_kernel");
}

extern "C" int ivb_nvls_flag_words(void) { return NVLS_MAX_BLOCKS * NVLS_MAX_WORLD; }
