// Hopper (sm_90a) plumbing shared by the HE and NN kernels: inline-PTX wrappers for mbarriers, TMA tensor and bulk
// copies, proxy fences and clusters on the device side, and the encoding of TMA tensor maps on the host side.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <initializer_list>
#include <stdexcept>
#include <string>

namespace hefl {
namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// Orders this thread's generic-proxy shared-memory accesses before later TMA (async-proxy) accesses.
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// Wait on the phase parity; traps (instead of hanging the GPU) after ~2 s. The suspend-time hint lets the
// hardware park the warp until the phase completes instead of returning to a software spin loop: with ~30
// waiting warps per SM the spin instructions were competing with the epilogue for issue slots. The clock is
// read once every kMbarClockSpins failed waits.
constexpr uint32_t kMbarSuspendNs = 1000000;
constexpr uint32_t kMbarClockSpins = 0x1000;
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  long long start = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity), "r"(kMbarSuspendNs)
        : "memory");
    if (done) break;
    if ((++spins & (kMbarClockSpins - 1)) == 0) {
      const long long now = clock64();
      if (start == 0) start = now;
      else if (now - start > 4000000000ll) __trap();
    }
  }
}

// One lane of a converged warp.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---- cluster ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- TMA: tensor copies global -> shared complete on an mbarrier --------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
        "r"(smem_u32(bar))
      : "memory");
}
// 2-D tensor copy into the shared memory of every CTA in `mask` (same offsets in each CTA).
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar,
                                               uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%2, %3}], [%4], %5;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(mask)
      : "memory");
}
// Plain (non-tensor) copy of `bytes` contiguous bytes, 16-byte aligned at both ends.
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- TMA: tensor stores shared -> global, tracked by bulk groups ---------------------------
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(src))
               : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// At most N committed groups still read their shared-memory source.
template <int N>
__device__ __forceinline__ void tma_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// At most N committed groups are still in flight.
template <int N>
__device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ---- host: tensor maps --------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// The driver's cuTensorMapEncodeTiled, looked up once through the runtime (no link against libcuda).
inline EncodeTiledFn encode_tiled_fn() {
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      throw std::runtime_error("cuTensorMapEncodeTiled not available");
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// Swizzle span equal to the box's innermost extent in bytes (128, 64, else 32): the layout the swizzled-tile
// readers (tc::swz<>, dev2::swz) expect.
inline CUtensorMapSwizzle swizzle_for(uint32_t inner_box_bytes) {
  return inner_box_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
         : inner_box_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                 : CU_TENSOR_MAP_SWIZZLE_32B;
}

// The driver call needs a current context on the calling thread. A thread that has made no runtime call yet has none
// (autograd's device thread, for one: the first CUDA work of a backward can be a GEMM's tensor-map encode, which then
// failed with CUDA_ERROR_INVALID_CONTEXT), so bind the current device's primary context once per thread.
inline void bind_primary_context() {
  thread_local bool bound = false;
  if (!bound) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaSetDevice(dev);
    bound = true;
  }
}

// Tiled map of the tensor at `ptr`, rank = dims.size(): dims innermost first, strides = the byte strides of
// dims[1..], one box per copy. Element strides 1, no interleave, 128-byte L2 promotion, out-of-bounds elements
// zero-filled. Throws with every parameter when the driver rejects the map.
inline CUtensorMap tensor_map(const void* ptr, CUtensorMapDataType type, std::initializer_list<uint64_t> dims,
                              std::initializer_list<uint64_t> strides, std::initializer_list<uint32_t> box,
                              CUtensorMapSwizzle swizzle) {
  const uint32_t rank = (uint32_t)dims.size();
  CUtensorMap m;
  CUresult r = CUDA_ERROR_INVALID_VALUE;
  bind_primary_context();
  if (rank >= 1 && rank <= 5 && strides.size() == rank - 1 && box.size() == rank) {
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    r = encode_tiled_fn()(&m, type, rank, const_cast<void*>(ptr), dims.begin(), strides.begin(), box.begin(), estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) {
    auto list = [](const auto& v) {
      std::string s = "{";
      for (const auto x : v) s += (s.size() > 1 ? ", " : "") + std::to_string(x);
      return s + "}";
    };
    char p[32];
    snprintf(p, sizeof(p), "%p", ptr);
    throw std::runtime_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + "): ptr=" + p +
                             " type=" + std::to_string((int)type) + " rank=" + std::to_string(rank) +
                             " dims=" + list(dims) + " strides=" + list(strides) + " box=" + list(box) +
                             " swizzle=" + std::to_string((int)swizzle));
  }
  return m;
}

}  // namespace sm90
}  // namespace hefl
