// Helpers of the NN tensor-core kernels (sm_90a): shared-memory budgets, warp-level MMAs (ldmatrix + mma.sync) on the
// swizzled tiles TMA writes, accumulator staging, the deterministic split-K sum and named barriers. The mbarrier, TMA
// and tensor-map plumbing they share with the HE kernels is in common/hopper.cuh.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../common/hopper.cuh"

namespace hefl {
namespace tc {

// Largest dynamic shared memory a block may opt into on H100 (sm_90): 227 KB. An SM has 228 KB and reserves 1 KB per
// resident block, so `nblocks` blocks of `smem` dynamic bytes fit on one SM when blocks_fit(smem, nblocks).
constexpr int kSmemMax = 227 * 1024;
constexpr bool blocks_fit(int smem, int nblocks) { return nblocks * (smem + 1024) <= 228 * 1024; }

// ---- warp-level tensor-core MMA on TMA-written shared-memory tiles (sm_90) ---------------------
// TMA writes a tile with a swizzle span of SW bytes (32, 64 or 128, equal to the tile's row length): the 16-byte
// chunk index inside a span is XORed with address bits 7.. . The pattern is a function of the absolute shared-memory
// address (tile bases are aligned to the pattern's repeat), so a tile may be read starting at ANY row: the halo
// kernels read shifted row windows of one loaded tile instead of loading every tap separately.
template <int SW>
__device__ __forceinline__ uint32_t swz(uint32_t addr) {
  constexpr uint32_t M = SW == 128 ? 7u : (SW == 64 ? 3u : 1u);
  return addr ^ (((addr >> 7) & M) << 4);
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_u16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
// d (m16 x n8, fp32) += a (m16 x k16, bf16, row) * b (k16 x n8, bf16, col)
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// d (m16 x n8, fp32) += a (m16 x k32, e4m3, row) * b (k32 x n8, e4m3, col)
__device__ __forceinline__ void mma_e4m3(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// A fragment (m16 x 32 bytes of K) of a K-major tile: row r of the fragment is tile row row0 + r, K bytes kb0..kb0+31.
template <int SW>
__device__ __forceinline__ void ld_a_kmajor(uint32_t tile, int row0, int kb0, int lane, uint32_t (&a)[4]) {
  ldsm_x4(swz<SW>(tile + (uint32_t)((row0 + (lane & 15)) * SW + kb0 + ((lane >> 4) << 4))), a);
}
// B fragments of two n8 tiles (rows n0 and n1 of a K-major [N][K] tile), 32 bytes of K: b[0..1] tile n0, b[2..3] n1.
template <int SW>
__device__ __forceinline__ void ld_b_kmajor(uint32_t tile, int n0, int n1, int kb0, int lane, uint32_t (&b)[4]) {
  const int n = ((lane >> 4) ? n1 : n0) + (lane & 7);
  ldsm_x4(swz<SW>(tile + (uint32_t)(n * SW + kb0 + (((lane >> 3) & 1) << 4))), b);
}
// Accumulator staging: a warp's two m16 x n8 fragments (rows 0-15, 16-31 of its 32 rows) -> row `lane`, 8 columns.
// `scr` is the warp's private 1 KB of shared memory.
__device__ __forceinline__ void frag_rows(float* scr, const float (&c0)[4], const float (&c1)[4], int lane, float* v) {
  const int r = lane >> 2, c = (lane & 3) * 2;
  __syncwarp();
  *reinterpret_cast<float2*>(scr + r * 8 + c) = make_float2(c0[0], c0[1]);
  *reinterpret_cast<float2*>(scr + (r + 8) * 8 + c) = make_float2(c0[2], c0[3]);
  *reinterpret_cast<float2*>(scr + (r + 16) * 8 + c) = make_float2(c1[0], c1[1]);
  *reinterpret_cast<float2*>(scr + (r + 24) * 8 + c) = make_float2(c1[2], c1[3]);
  __syncwarp();
  const float4 x = *reinterpret_cast<const float4*>(scr + lane * 8);
  const float4 y = *reinterpret_cast<const float4*>(scr + lane * 8 + 4);
  v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; v[4] = y.x; v[5] = y.y; v[6] = y.z; v[7] = y.w;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// Deterministic split-K reduction: returns sum over p = 0 .. parts-1 of ws[p * n + i] for element i = blockIdx.x * 32 +
// lane, with a fixed summation tree (warp j of the 256-thread block sums p = j, j + 8, ... in order, then the eight
// warp sums are added in warp order), so the result is the same bits on every run. Call with blockDim.x == 256;
// `red` is 256 floats of shared memory; the result is valid in warp 0.
__device__ __forceinline__ float sum_partials(const float* __restrict__ ws, int parts, int64_t n, float* red) {
  const int lane = threadIdx.x & 31, j = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * 32 + lane;
  float s = 0.f;
  if (i < n)
    for (int p = j; p < parts; p += 8) s += ws[(int64_t)p * n + i];
  red[threadIdx.x] = s;
  __syncthreads();
  float t = 0.f;
  if (j == 0)
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w * 32 + lane];
  return t;
}

__device__ __forceinline__ void named_barrier_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_barrier_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace tc
}  // namespace hefl
