// Layer-1 (3 input channels) weight gradient straight from the POOLED gradient — no un-pooling pass and
// no 132 MB conv-grid gradient tensor.
//
// After ReLU + 2x2 max-pool the conv-grid gradient has exactly one non-zero per window and channel (at the
// arg-max, if the unit is active), so
//     dW[r,s,ci,co] = sum over windows  g[window,co] * X[argmax_pos(window,co) + (r,s), ci]
// is a gather with 27 MACs per (window, channel) instead of a dense GEMM over 4x as many pixels padded to
// 16 channels. The tensor-core path spent 47 us (unpool) + 88 us (wgrad) on this layer; the position
// depends on the channel, so the work is not GEMM-shaped — it runs on the FP32 pipes (bf16 operands widened
// to fp32 by a shift, fp32 FMA):
//   * lane = output channel (Co = 32), a warp walks the windows of one pooled row;
//   * the 4 input rows under a pooled row are staged once per strip in shared memory as 4 x bf16 per pixel
//     (row pitch padded by 16 B so the 4 candidate positions of a window hit distinct banks). Shared-memory
//     wavefronts are the floor of this kernel: with fp32x4 pixels every lane-divergent LDS.128 cost 4+
//     wavefronts and the kernel ran slower than the tensor-core path (measured); LDS.64 halves that;
//   * g / argmax of all the warp's windows of the strip are fetched up front (16 loads in flight per lane);
//   * the next strip's rows are prefetched into registers while the current strip is processed;
//   * 27 + 1 (bias) accumulators per lane, reduced across warps in shared memory in warp order, then one
//     partial per CTA, added into the split-K buffer in CTA order (wgrad0_reduce).
// Reference semantics: Keras Conv2D/MaxPooling2D backward of the first block (FLPyfhelin.py:120-121).
#include <cuda_bf16.h>

#include "../he/kernels.h"
#include "launch.cuh"
#include "nn.h"

namespace hefl {
namespace nn {

// d += a * b with bf16 operands and an fp32 accumulator; a bf16 is the upper half of an fp32, so widening is
// exact and the single-rounding fp32 FMA gives the same bits as a mixed-precision bf16 FMA
__device__ __forceinline__ void fhfma(float& d, uint16_t a, uint16_t b) {
  d = fmaf(__uint_as_float((uint32_t)a << 16), __uint_as_float((uint32_t)b << 16), d);
}
__device__ __forceinline__ void split16(uint32_t v, uint16_t& lo, uint16_t& hi) {
  asm("mov.b32 {%0, %1}, %2;" : "=h"(lo), "=h"(hi) : "r"(v));
}

constexpr int kGatherWarps = 16;      // 2 CTAs x 16 warps per SM at <= 64 registers: latency hiding for LDS / LDG
constexpr int kGatherThreads = kGatherWarps * 32;
constexpr int kGatherPre = 2;         // staged pixels per thread and strip: 4 rows * W <= 2 * 512
constexpr int kGatherNJ = 8;          // windows per warp and strip: Wp <= 16 * 8

__global__ void __launch_bounds__(kGatherThreads, 2)
wgrad0_gather_kernel(const __nv_bfloat16* __restrict__ X, const __nv_bfloat16* __restrict__ g,
                     const uint8_t* __restrict__ amax, float* __restrict__ ws, int B, int H, int W, int Hp, int Wp) {
  extern __shared__ __align__(16) uint8_t sm[];
  const int rowb = W * 8 + 16;
  const int bufb = 4 * rowb;
  float* red = reinterpret_cast<float*>(sm + 2 * bufb);   // [28][32]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 28 * 32; i += kGatherThreads) red[i] = 0.f;
  pdl_prologue();

  float acc[9][3];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t][0] = acc[t][1] = acc[t][2] = 0.f;
  float accb = 0.f;

  const int nstrips = B * Hp;
  const int npx = 4 * W;
  uint2 pre[kGatherPre];

  // strip-invariant staging coordinates of this thread's pixels (4 rows x W pixels, 8 B each)
  int src_off[kGatherPre], dst_off[kGatherPre];
#pragma unroll
  for (int k = 0; k < kGatherPre; ++k) {
    const int p = threadIdx.x + k * kGatherThreads;
    const int r = p / W, c = p - r * W;
    src_off[k] = p * 16;
    dst_off[k] = p < npx ? r * rowb + c * 8 : -1;
  }
  auto fetch = [&](int s) {
    const int b = s / Hp, i = s - b * Hp;
    const __nv_bfloat16* src = X + ((size_t)(b * H + 2 * i) * W) * 16;     // 4 consecutive image rows
#pragma unroll
    for (int k = 0; k < kGatherPre; ++k)
      if (dst_off[k] >= 0) pre[k] = __ldg(reinterpret_cast<const uint2*>(src + src_off[k]));
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int k = 0; k < kGatherPre; ++k)
      if (dst_off[k] >= 0) *reinterpret_cast<uint2*>(sm + buf * bufb + dst_off[k]) = pre[k];
  };

  int s = blockIdx.x;
  int buf = 0;
  if (s < nstrips) { fetch(s); stash(0); }
  __syncthreads();
  for (; s < nstrips; s += gridDim.x) {
    const int nxt = s + gridDim.x;
    // this warp's windows of the strip: all loads in flight before the first use
    // (prefetching them one strip ahead was measured slower: 103 vs 69 us)
    const size_t rowbase = (size_t)s * Wp * 32 + lane;
    uint32_t ga[kGatherNJ];                                              // g bits | argmax byte << 16
#pragma unroll
    for (int k = 0; k < kGatherNJ; ++k) {
      const int j = warp + k * kGatherWarps;
      ga[k] = 0;
      if (j < Wp)
        ga[k] = (uint32_t)__ldg(reinterpret_cast<const uint16_t*>(g) + rowbase + (size_t)j * 32) |
                ((uint32_t)__ldg(amax + rowbase + (size_t)j * 32) << 16);
    }
    if (nxt < nstrips) fetch(nxt);
    const uint8_t* xb = sm + buf * bufb;
#pragma unroll
    for (int k = 0; k < kGatherNJ; ++k) {
      const int j = warp + k * kGatherWarps;
      if (j < Wp) {                                                      // warp-uniform
        const uint32_t am = ga[k] >> 16;
        const uint16_t gv = (am & 4u) ? (uint16_t)(ga[k] & 0xFFFFu) : (uint16_t)0;   // ReLU mask (bf16 bits)
        const uint8_t* p0 = xb + ((am >> 1) & 1u) * rowb + (2 * j + (am & 1u)) * 8;
        fhfma(accb, gv, (uint16_t)0x3F80);
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            const uint2 v = *reinterpret_cast<const uint2*>(p0 + r * rowb + q * 8);
            uint16_t c0, c1, c2, c3;
            split16(v.x, c0, c1);
            split16(v.y, c2, c3);
            fhfma(acc[r * 3 + q][0], c0, gv);
            fhfma(acc[r * 3 + q][1], c1, gv);
            fhfma(acc[r * 3 + q][2], c2, gv);
          }
      }
    }
    if (nxt < nstrips) stash(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }

  // cross-warp reduction in warp order (a fixed summation order: the same bits on every run), then this CTA's
  // partial; wgrad0_reduce adds the partials of all CTAs in CTA order
#pragma unroll 1
  for (int w = 0; w < kGatherWarps; ++w) {
    if (warp == w) {
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        red[(t * 3 + 0) * 32 + lane] += acc[t][0];
        red[(t * 3 + 1) * 32 + lane] += acc[t][1];
        red[(t * 3 + 2) * 32 + lane] += acc[t][2];
      }
      red[27 * 32 + lane] += accb;
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < kWgrad0Part; i += kGatherThreads) ws[(size_t)blockIdx.x * kWgrad0Part + i] = red[i];
}

bool wgrad0_gather_supported(int W, int Wp, int CK, int Ci, int Co) {
  return CK == 16 && Ci <= 3 && Co == 32 && 4 * W <= kGatherPre * kGatherThreads && Wp <= kGatherWarps * kGatherNJ;
}

void wgrad0_gather(const void* X, const void* g, const uint8_t* amax, float* dW, float* ws, int B, int H, int W, int Hp,
                   int Wp, cudaStream_t st) {
  const int smem = 2 * 4 * (W * 8 + 16) + 28 * 32 * 4;
  const int grid = wgrad0_parts(B, Hp);
  cudaFuncSetAttribute(wgrad0_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  launch_pdl(wgrad0_gather_kernel, dim3(grid), dim3(kGatherThreads), smem, st, reinterpret_cast<const __nv_bfloat16*>(X),
             reinterpret_cast<const __nv_bfloat16*>(g), amax, ws, B, H, W, Hp, Wp);
  hefl::cuda::note_launch();
  wgrad0_reduce(ws, grid, dW, st);
}

}  // namespace nn
}  // namespace hefl
