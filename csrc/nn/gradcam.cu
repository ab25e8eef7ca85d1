// Grad-CAM maps of the sequential CNNs (DESIGN.md §11), one launch, one cluster of 8 CTAs per scan.
//
// Inputs are a conv stage's output X and the class score's gradient G at it, both bf16 [B*Hp*Hp][C] (NHWC). Per scan:
//   alpha[c] = (1 / Hp^2) sum_hw G[hw][c]
//   cam[hw]  = max(0, sum_c alpha[c] X[hw][c])
//   out      = bilinear(cam, S x S, half-pixel centres, edge clamp) / max_hw cam   (0 where that maximum is 0)
// The 8 CTAs of a cluster split the Hp rows of the map: each sums G over its rows, the partial alphas are added in
// rank order through distributed shared memory, each CTA maps its rows and writes them into all 8 CTAs' copy of the
// Hp x Hp map, and each then upsamples one eighth of the S x S output from its own copy. G and X are read once each
// with 16-byte loads, the output is written once with 16-byte stores (S even), and nothing else touches global
// memory. Every sum runs in an order fixed by (Hp, C) alone: no float atomics, no dependence on the batch row.
#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include "../he/kernels.h"
#include "launch.cuh"
#include "nn.h"

namespace cg = cooperative_groups;

namespace hefl {
namespace nn {

namespace gc {
constexpr int R = 8;                     // cluster size: CTAs per scan
constexpr int NT = 256;
constexpr int CMAX = 128;
// shared-memory layout (floats)
constexpr int O_PART = 0;                // [NT][8]   per-thread channel sums of G
constexpr int O_APART = O_PART + NT * 8; // [CMAX]    this CTA's sum of G over its rows
constexpr int O_ALPHA = O_APART + CMAX;  // [CMAX]
constexpr int O_MAX = O_ALPHA + CMAX;    // [R]       every CTA's maximum of its rows of the map
constexpr int O_RED = O_MAX + R;         // [NT / 32] warp maxima
constexpr int O_CAM = O_RED + NT / 32;   // [Hp*Hp]   the whole low-resolution map
constexpr int kMaxSmem = 227 * 1024;
}  // namespace gc

__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }

// the upsampled map at output pixel (y, x), before normalisation (F.interpolate, bilinear, align_corners=False)
__device__ __forceinline__ float gradcam_sample(const float* cam, int Hp, float scale, int y, int x) {
  const float sy = fmaxf((y + 0.5f) * scale - 0.5f, 0.f), sx = fmaxf((x + 0.5f) * scale - 0.5f, 0.f);
  const int y0 = min((int)sy, Hp - 1), x0 = min((int)sx, Hp - 1);
  const int y1 = y0 + (y0 < Hp - 1 ? 1 : 0), x1 = x0 + (x0 < Hp - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  return hy * (hx * cam[y0 * Hp + x0] + lx * cam[y0 * Hp + x1]) + ly * (hx * cam[y1 * Hp + x0] + lx * cam[y1 * Hp + x1]);
}

__global__ void __cluster_dims__(gc::R, 1, 1) __launch_bounds__(gc::NT)
gradcam_kernel(const __nv_bfloat16* __restrict__ X, const __nv_bfloat16* __restrict__ G, float* __restrict__ out,
               int Hp, int C, int S, int nvalid) {
  using namespace gc;
  extern __shared__ __align__(16) float sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int r = (int)cluster.block_rank();
  const int b = blockIdx.x / R;
  const int t = threadIdx.x;
  // the same b for all 8 CTAs of a cluster: a cluster leaves as a whole, before its first barrier
  if (b >= nvalid) return;
  pdl_prologue();
  float* part = sm + O_PART;
  float* apart = sm + O_APART;
  float* alpha = sm + O_ALPHA;
  float* maxS = sm + O_MAX;
  float* red = sm + O_RED;
  float* cam = sm + O_CAM;
  const int P = Hp * Hp, G8 = C >> 3;
  const int p0 = (Hp * r / R) * Hp, p1 = (Hp * (r + 1) / R) * Hp;    // this CTA's rows of the map
  const size_t base = (size_t)b * P;

  // ---- alpha: thread t sums channels [8 cg, 8 cg + 8) over pixels p0 + pl, p0 + pl + lanes, ...
  {
    const int lanes = NT / G8, cg8 = t % G8, pl = t / G8;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    if (pl < lanes) {
      const uint4* src = reinterpret_cast<const uint4*>(G + base * C) + cg8;
#pragma unroll 4
      for (int p = p0 + pl; p < p1; p += lanes) {
        const uint4 v = __ldg(src + (size_t)p * G8);
        acc[0] += bf16_lo(v.x); acc[1] += bf16_hi(v.x); acc[2] += bf16_lo(v.y); acc[3] += bf16_hi(v.y);
        acc[4] += bf16_lo(v.z); acc[5] += bf16_hi(v.z); acc[6] += bf16_lo(v.w); acc[7] += bf16_hi(v.w);
      }
    }
    *reinterpret_cast<float4*>(part + t * 8) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(part + t * 8 + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    __syncthreads();
    if (t < C) {
      float s = 0.f;
      for (int j = 0; j < lanes; ++j) s += part[(j * G8 + (t >> 3)) * 8 + (t & 7)];
      apart[t] = s;
    }
  }
  cluster.sync();                        // every CTA's partial alpha is complete (and every CTA has started)
  if (t < C) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < R; ++q) s += cluster.map_shared_rank(apart, q)[t];
    alpha[t] = s / (float)P;
  }
  __syncthreads();

  // ---- the map on this CTA's rows, written into every CTA's copy
  float mx = 0.f;
  for (int p = p0 + t; p < p1; p += NT) {
    const uint4* src = reinterpret_cast<const uint4*>(X + (base + p) * C);
    float a = 0.f;
    for (int k = 0; k < G8; ++k) {
      const uint4 v = __ldg(src + k);
      const float* al = alpha + k * 8;
      a = fmaf(al[0], bf16_lo(v.x), a); a = fmaf(al[1], bf16_hi(v.x), a);
      a = fmaf(al[2], bf16_lo(v.y), a); a = fmaf(al[3], bf16_hi(v.y), a);
      a = fmaf(al[4], bf16_lo(v.z), a); a = fmaf(al[5], bf16_hi(v.z), a);
      a = fmaf(al[6], bf16_lo(v.w), a); a = fmaf(al[7], bf16_hi(v.w), a);
    }
    const float v = a > 0.f ? a : 0.f;
    mx = fmaxf(mx, v);
#pragma unroll
    for (int q = 0; q < R; ++q) cluster.map_shared_rank(cam, q)[p] = v;
  }
  // the maximum is exact in any order
  for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if ((t & 31) == 0) red[t >> 5] = mx;
  __syncthreads();
  if (t == 0) {
    float m = 0.f;
    for (int w = 0; w < NT / 32; ++w) m = fmaxf(m, red[w]);
#pragma unroll
    for (int q = 0; q < R; ++q) cluster.map_shared_rank(maxS, q)[r] = m;
  }
  cluster.sync();                        // the whole map and all 8 maxima are here; no remote access after this
  float m = 0.f;
#pragma unroll
  for (int q = 0; q < R; ++q) m = fmaxf(m, maxS[q]);

  // ---- upsample and normalise this CTA's eighth of the S x S output
  const float scale = (float)Hp / (float)S;
  const bool zero = !(m > 0.f);
  float* o = out + (size_t)b * S * S;
  if ((S & 1) == 0) {                    // S * S is a multiple of 4: 16-byte stores of 4 consecutive pixels
    const int nq = S * S / 4, q0 = (int)((int64_t)nq * r / R), q1 = (int)((int64_t)nq * (r + 1) / R);
    for (int q = q0 + t; q < q1; q += NT) {
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int e = 4 * q + i, y = e / S, x = e - y * S;
        v[i] = zero ? 0.f : gradcam_sample(cam, Hp, scale, y, x) / m;
      }
      reinterpret_cast<float4*>(o)[q] = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
    const int n = S * S, e0 = (int)((int64_t)n * r / R), e1 = (int)((int64_t)n * (r + 1) / R);
    for (int e = e0 + t; e < e1; e += NT) {
      const int y = e / S, x = e - y * S;
      o[e] = zero ? 0.f : gradcam_sample(cam, Hp, scale, y, x) / m;
    }
  }
}

static int gradcam_smem(int Hp) { return (gc::O_CAM + Hp * Hp) * 4; }

bool gradcam_supported(int Hp, int C, int S) {
  return C >= 8 && C <= gc::CMAX && C % 8 == 0 && Hp >= 1 && S >= 1 && gradcam_smem(Hp) <= gc::kMaxSmem;
}

void gradcam(const void* X, const void* G, float* out, int Hp, int C, int S, int nvalid, cudaStream_t st) {
  const int smem = gradcam_smem(Hp);
  cudaFuncSetAttribute(gradcam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  launch_pdl(gradcam_kernel, dim3(nvalid * gc::R), dim3(gc::NT), smem, st, reinterpret_cast<const __nv_bfloat16*>(X),
             reinterpret_cast<const __nv_bfloat16*>(G), out, Hp, C, S, nvalid);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl
