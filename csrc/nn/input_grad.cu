// Layer-1 input gradient of the medical CNN (DESIGN.md §12), straight from the pooled gradient: no conv-grid gradient
// tensor (66 MB at batch 32, 256 x 256), one launch.
//
// After ReLU + 2x2 floor max-pool the conv-grid gradient dY0 has at most one non-zero per window and channel: the
// pooled gradient g at the window's arg-max position, if the unit is active (code bit 2). The input gradient is the
// full correlation of dY0 with the layer's weights,
//     dx[i, j, ci] = sum_{co, r, s} dY0[i - r, j - s, co] * W[co][ci][r][s],
// and the 3 x 3 conv positions reaching pixel (i, j) lie in at most 2 x 2 pooling windows. One thread owns a 2 x 2
// block of pixels, (2a + {0, 1}, 2b + {0, 1}), which is reached by exactly the windows (a - 1 .. a, b - 1 .. b): it
// reads their 4 x 32 gradients and codes once with 16-byte loads and adds, per window and channel, the product with the
// tap (r, s) = pixel - arg-max position into each of the block's pixels it reaches. Every pixel's sum runs over the
// windows in row-major order and the channels in order, an order fixed by (S, Ci): no float atomics, and the same
// bits wherever a scan sits in the batch. The sum is added to the fp32 accumulator once. Pixels no window reaches
// (the dropped floor-pool edge and the 2-pixel border) get a gradient of 0.
#include <cuda_bf16.h>

#include "../he/kernels.h"
#include "launch.cuh"
#include "nn.h"

namespace hefl {
namespace nn {

namespace ig {
constexpr int CO = 32;
constexpr int NT = 128;          // threads per CTA: 128 pixel blocks of one block row
}  // namespace ig

__device__ __forceinline__ float ig_bf16(uint32_t w, int hi) {
  return __uint_as_float(hi ? (w & 0xFFFF0000u) : (w << 16));
}

template <int CI>
__global__ void __launch_bounds__(ig::NT)
input_grad0_kernel(const __nv_bfloat16* __restrict__ g, const uint8_t* __restrict__ amax,
                   const __nv_bfloat16* __restrict__ w, float* __restrict__ acc, int S, int Hp) {
  using namespace ig;
  __shared__ float wsm[CO * 9 * CI];     // [co][r * 3 + s][ci]
  pdl_prologue();                        // the weights may have just been written by Adam
  for (int e = threadIdx.x; e < CO * 9 * CI; e += NT) {
    const int co = e / (9 * CI), rem = e - co * 9 * CI, t = rem / CI, ci = rem - t * CI;
    wsm[e] = __bfloat162float(w[(co * CI + ci) * 9 + t]);
  }
  __syncthreads();
  const int Sb = (S + 1) >> 1;
  const int bc = blockIdx.x * NT + threadIdx.x, a = blockIdx.y, b = blockIdx.z;
  if (bc >= Sb) return;

  float sum[2][2][CI];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int c = 0; c < CI; ++c) sum[i][j][c] = 0.f;

#pragma unroll
  for (int wa = 0; wa < 2; ++wa) {
    const int pa = a - 1 + wa;
    if (pa < 0 || pa >= Hp) continue;
#pragma unroll
    for (int wb = 0; wb < 2; ++wb) {
      const int pb = bc - 1 + wb;
      if (pb < 0 || pb >= Hp) continue;
      const size_t win = ((size_t)b * Hp + pa) * Hp + pb;
      const uint4* gp = reinterpret_cast<const uint4*>(g + win * CO);
      const uint4* cp = reinterpret_cast<const uint4*>(amax + win * CO);
      uint32_t gw[16], cw[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 v = __ldg(gp + q);
        gw[4 * q] = v.x; gw[4 * q + 1] = v.y; gw[4 * q + 2] = v.z; gw[4 * q + 3] = v.w;
      }
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const uint4 v = __ldg(cp + q);
        cw[4 * q] = v.x; cw[4 * q + 1] = v.y; cw[4 * q + 2] = v.z; cw[4 * q + 3] = v.w;
      }
#pragma unroll
      for (int co = 0; co < CO; ++co) {
        const uint32_t code = (cw[co >> 2] >> (8 * (co & 3))) & 0xFFu;
        if (!(code & 4u)) continue;
        const float gv = ig_bf16(gw[co >> 1], co & 1);
        // arg-max position relative to the block's top-left pixel: rows / columns -2 .. 1
        const int y = 2 * (wa - 1) + (int)((code >> 1) & 1u), x = 2 * (wb - 1) + (int)(code & 1u);
        const float* wc = wsm + co * 9 * CI;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = i - y;
          if (r < 0 || r > 2) continue;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int s = j - x;
            if (s < 0 || s > 2) continue;
            const float* wt = wc + (r * 3 + s) * CI;
#pragma unroll
            for (int c = 0; c < CI; ++c) sum[i][j][c] = fmaf(gv, wt[c], sum[i][j][c]);
          }
        }
      }
    }
  }

#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int y = 2 * a + i;
    if (y >= S) continue;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int x = 2 * bc + j;
      if (x >= S) continue;
      float* o = acc + (((size_t)b * S + y) * S + x) * CI;
#pragma unroll
      for (int c = 0; c < CI; ++c) o[c] += sum[i][j][c];
    }
  }
}

void input_grad0(const void* g, const uint8_t* amax, const void* w, float* acc, int S, int Hp, int in_channels,
                 int nvalid, cudaStream_t st) {
  const int Sb = (S + 1) / 2;
  const dim3 grid((Sb + ig::NT - 1) / ig::NT, Sb, nvalid);
  const auto* gb = reinterpret_cast<const __nv_bfloat16*>(g);
  const auto* wb = reinterpret_cast<const __nv_bfloat16*>(w);
  if (in_channels == 3)
    launch_pdl(input_grad0_kernel<3>, grid, dim3(ig::NT), 0, st, gb, amax, wb, acc, S, Hp);
  else
    launch_pdl(input_grad0_kernel<1>, grid, dim3(ig::NT), 0, st, gb, amax, wb, acc, S, Hp);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl
