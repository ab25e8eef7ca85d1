// TMA-fed tensor-core GEMM kernels for the ResNet convolutions (SURVEY.md K13-K15; BASELINE.json configs[2], [4]).
// On NHWC activations
//
//   * a 1x1 convolution is the GEMM  Y[pixels, Co] = X[pixels, Ci] . W[Co, Ci]^T,
//   * a 3x3 / pad-1 / stride-1 convolution is NINE such GEMMs accumulated in one tile: tap (r, s) multiplies the same
//     activation matrix shifted by (r-1)*Wp + (s-1) rows, when the activations live on a zero-padded
//     (H+2) x (W+2) grid -- the shift is just the row coordinate of the TMA copy (no im2col),
//   * dgrad is the same kernel with the transposed / flipped filter,
//   * wgrad is  dW[tap][Co, Ci] = sum_pixels dY[p, Co] . X[p + shift(tap), Ci]: both operands are consumed as
//     stored (ldmatrix.trans, the pixel axis is K), split over pixel ranges, fp32 vector RED.
//
// kmajor_gemm_kernel : C[M, N] = sum_taps A[M + shift_t, K] . B_t[N, K]^T, bf16 or e4m3 (per-tensor scales folded
//                      into the epilogue), fp32 accumulation in registers (asynchronous wgmma), bf16 out. Warp-specialised
//                      and persistent: 1 TMA producer warp, 2 consumer warpgroups; 6/7-stage smem ring (128 B swizzle).
// wgrad_mn_kernel    : one tap per unit, split over pixel ranges.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <stdexcept>

#include "../he/kernels.h"
#include "nn.h"
#include "tc_common.cuh"

namespace hefl {
namespace nn {

using namespace hefl::sm90;
using namespace hefl::tc;

namespace {

// 2-D tensor [rows][cols] of `esize`-byte elements, row pitch in bytes; box = box_cols x box_rows, 128 B swizzle.
CUtensorMap map2d(const void* ptr, int esize, uint64_t cols, uint64_t rows, uint64_t pitch_bytes, uint32_t box_cols,
                  uint32_t box_rows) {
  return tensor_map(ptr, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, {cols, rows},
                    {pitch_bytes}, {box_cols, box_rows}, CU_TENSOR_MAP_SWIZZLE_128B);
}

// ------------------------------------------------------------------------------------------------------------
// K-major GEMM with row-shifted taps
// ------------------------------------------------------------------------------------------------------------
struct GemmArgs {
  int m_tiles, n_tiles;   // 128-row tiles of the A grid, BN-column tiles
  int kblocks;            // K / (128 bytes of K)
  int taps;
  int shift[9];           // row shift of A for tap t
  int n_total;            // N (rows of B per tap, row pitch of C in elements)
  int64_t m_rows;         // rows of the A grid (dense: valid output rows)
  // padded-grid mode (3x3 convolutions): A rows index a zero-padded [B][Hp][Wp] grid, only interior pixels are
  // written, to row (b*H + hp-1)*W + wp-1 of C
  int padded, Bn, H, W, Hp, Wp;
  __nv_bfloat16* C;
  const float* scale_a;   // fp8: de-quantisation factors (device scalars) or null
  const float* scale_b;
};

// ---- warpgroup MMA (sm_90a wgmma) ---------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major tile written by TMA with 128-byte swizzle: 8-row core-matrix groups
// 1024 bytes apart (SBO), LBO unused (1), layout type 1 = 128B swizzle. Advancing K by 32 bytes inside the swizzle
// atom is +2 on the start-address field.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x N] (fp32, registers of the warpgroup) += A[64 x K] . B[N x K]^T, both K-major in shared memory
__device__ __forceinline__ void wgmma_n128_bf16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_n64_bf16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_n128_e4m3(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_n64_e4m3(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db));
}

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = 128 * 128;          // 128 rows x 128 bytes of K
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int NSTAGE = BN == 128 ? 6 : 7;
  static constexpr int SMEM = NSTAGE * STAGE + 256 + 1024;
  static_assert(SMEM <= kSmemMax, "shared memory");
};

// Warpgroups 0 and 1 (warps 0..7) each own 64 rows x BN columns of the 128-row output tile, fp32 accumulators in
// registers fed by asynchronous wgmma (m64nBNk16 bf16 / m64nBNk32 e4m3) straight from the TMA-written stages; the
// wgmma group of one stage stays in flight while the next is issued. Warp 8 is the TMA producer; persistent.
template <int BN, bool FP8>
__global__ void __launch_bounds__(288, 1)
kmajor_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmArgs a) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::NSTAGE * Cfg::STAGE);
  uint64_t* full = bars;                          // [NSTAGE]
  uint64_t* empty = bars + Cfg::NSTAGE;           // [NSTAGE]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int KE = FP8 ? 128 : 64;              // K elements per 128-byte k-block

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int num_tiles = a.m_tiles * a.n_tiles;
  const int ksteps = a.taps * a.kblocks;

  if (warp == 8) {
    // ===== TMA producer =====
    if (elect_one()) {
      int st = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int mb = t / a.n_tiles, nb = t - mb * a.n_tiles;
        for (int tap = 0; tap < a.taps; ++tap) {
          const int arow = mb * 128 + a.shift[tap];
          const int brow = tap * a.n_total + nb * BN;
          for (int kb = 0; kb < a.kblocks; ++kb) {
            mbar_wait(&empty[st], phase ^ 1u);
            uint8_t* sA = smem + st * Cfg::STAGE;
            mbar_expect_tx(&full[st], Cfg::STAGE);
            tma_load_2d(sA, &tmA, kb * KE, arow, &full[st]);
            tma_load_2d(sA + Cfg::A_BYTES, &tmB, kb * KE, brow, &full[st]);
            if (++st == Cfg::NSTAGE) { st = 0; phase ^= 1u; }
          }
        }
      }
    }
    return;
  }
  // ===== consumer warpgroups
  const int wg = warp >> 2, wq = warp & 3;
  float alpha = 1.0f;
  if (FP8 && a.scale_a) alpha = (*a.scale_a) * (*a.scale_b);
  int st = 0;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int mb = t / a.n_tiles, nb = t - mb * a.n_tiles;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int ks = 0; ks < ksteps; ++ks) {
      mbar_wait(&full[st], phase);
      const uint32_t sa = smem_u32(smem + st * Cfg::STAGE) + wg * 64 * 128;
      const uint32_t sb = smem_u32(smem + st * Cfg::STAGE + Cfg::A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {                // 4 x 32 bytes of K per stage
        const uint64_t da = gmma_desc_sw128(sa + k * 32), db = gmma_desc_sw128(sb + k * 32);
        if constexpr (FP8) {
          if constexpr (BN == 128) wgmma_n128_e4m3(acc, da, db); else wgmma_n64_e4m3(acc, da, db);
        } else {
          if constexpr (BN == 128) wgmma_n128_bf16(acc, da, db); else wgmma_n64_bf16(acc, da, db);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                             // the previous stage's MMAs are done: release its buffer
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = st;
      if (++st == Cfg::NSTAGE) { st = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
    }
    // accumulator layout: element 4j + q is row 16*wq + lane/4 (+8 for q >= 2), column 8j + 2*(lane%4) + (q & 1)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = (int64_t)mb * 128 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      bool valid;
      int64_t orow;
      if (a.padded) {
        const int per = a.Hp * a.Wp;
        const int b = (int)(m / per);
        const int rem = (int)(m - (int64_t)b * per);
        const int hp = rem / a.Wp, wp = rem - hp * a.Wp;
        valid = b < a.Bn && hp >= 1 && hp <= a.H && wp >= 1 && wp <= a.W;
        orow = ((int64_t)b * a.H + (hp - 1)) * a.W + (wp - 1);
      } else {
        valid = m < a.m_rows;
        orow = m;
      }
      if (!valid) continue;
      __nv_bfloat16* dst = a.C + orow * a.n_total + nb * BN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(acc[4 * j + 2 * h] * alpha, acc[4 * j + 2 * h + 1] * alpha);
    }
  }
}

template <int BN, bool FP8>
void launch_kmajor(const void* A, const void* Bm, const GemmArgs& a, int64_t a_rows, int K, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  const int es = FP8 ? 1 : 2;
  const int ke = FP8 ? 128 : 64;
  const CUtensorMap tmA = map2d(A, es, (uint64_t)K, (uint64_t)a_rows, (uint64_t)K * es, ke, 128);
  const CUtensorMap tmB = map2d(Bm, es, (uint64_t)K, (uint64_t)a.taps * a.n_total, (uint64_t)K * es, ke, BN);
  auto kern = kmajor_gemm_kernel<BN, FP8>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
  const int tiles = a.m_tiles * a.n_tiles;
  const int grid = std::min(tiles, hefl::cuda::device_sm_count());
  kern<<<grid, 288, Cfg::SMEM, st>>>(tmA, tmB, a);
  hefl::cuda::note_launch();
}

// ------------------------------------------------------------------------------------------------------------
// Block-scaled e4m3 GEMM: one UE8M0 scale per row and per 32 elements of K
// ------------------------------------------------------------------------------------------------------------
// C[M, N] = sum_k (A[m, k] 2^(sa[m, k/32] - 127)) (B[n, k] 2^(sb[n, k/32] - 127)). A, B: e4m3 bytes, K-major.
// Scale factors travel in tiles: for every (128-row block, group of four 32-element k-blocks) one 512-byte tile
// [lane l = 0..31][row quarter i = 0..3][k-block kb = 0..3] holding the scale of row 32*i + l; a stage brings its
// two tiles in with a bulk copy.
struct MxArgs {
  int m_tiles, n_tiles, kgroups;   // 128-row tiles, BN-column tiles, K / 128
  int n_total;
  int64_t m_rows;
  __nv_bfloat16* C;
  const uint8_t* sfa;              // [m_tiles][kgroups][512]
  const uint8_t* sfb;              // [N / 128][kgroups][512]
};

constexpr int kMxStage = 128 * 128 + 128 * 128 + 1024;    // A tile, B tile, two scale tiles
constexpr int kMxStages = 5;
constexpr int kMxSmem = kMxStages * kMxStage + 256 + 1024;

// Warps 0..7 compute (warp w: rows 32*(w%4) .. +31, columns (w/4)*64 .. +63), warp 8 is the TMA producer. Each
// 32-element k-block is one m16n8k32 e4m3 MMA into a zeroed fragment, which is then added to the fp32 accumulator
// scaled by 2^(sa - 127) * 2^(sb - 127) of its row and column (powers of two: the scaling is exact).
__global__ void __launch_bounds__(288, 1)
mx_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const MxArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kMxStages * kMxStage);
  uint64_t* full = bars;
  uint64_t* empty = bars + kMxStages;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int BN = 128;
  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < kMxStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int num_tiles = a.m_tiles * a.n_tiles;

  if (warp == 8) {
    if (elect_one()) {
      int st = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int mb = t / a.n_tiles, nb = t - mb * a.n_tiles;
        for (int kg = 0; kg < a.kgroups; ++kg) {
          mbar_wait(&empty[st], phase ^ 1u);
          uint8_t* s = smem + st * kMxStage;
          mbar_expect_tx(&full[st], kMxStage);
          tma_load_2d(s, &tmA, kg * 128, mb * 128, &full[st]);
          tma_load_2d(s + 16384, &tmB, kg * 128, nb * BN, &full[st]);
          bulk_load_1d(s + 32768, a.sfa + ((size_t)mb * a.kgroups + kg) * 512, 512, &full[st]);
          bulk_load_1d(s + 32768 + 512, a.sfb + ((size_t)nb * a.kgroups + kg) * 512, 512, &full[st]);
          if (++st == kMxStages) { st = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }
  const int qd = warp & 3, half = warp >> 2;
  const int g8 = lane >> 2, c2 = (lane & 3) * 2;
  int st = 0;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int mb = t / a.n_tiles, nb = t - mb * a.n_tiles;
    float acc[8][2][4];
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[n][mt][q] = 0.f;
    for (int kg = 0; kg < a.kgroups; ++kg) {
      mbar_wait(&full[st], phase);
      uint8_t* s = smem + st * kMxStage;
      const uint32_t sa = smem_u32(s), sb = sa + 16384;
      // scale tile layout: byte l*16 + i*4 + kb holds the scale of row (or column) 32*i + l, k-block kb
      const uint8_t* sfa = s + 32768;
      const uint8_t* sfb = s + 32768 + 512;
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        uint32_t af[2][4];
        float fa[2][2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          ld_a_kmajor<128>(sa, qd * 32 + mt * 16, kb * 32, lane, af[mt]);
#pragma unroll
          for (int h = 0; h < 2; ++h) fa[mt][h] = ldexpf(1.0f, (int)sfa[(mt * 16 + g8 + 8 * h) * 16 + qd * 4 + kb] - 127);
        }
#pragma unroll
        for (int n = 0; n < 8; n += 2) {
          uint32_t bf[4];
          const int n0 = half * 64 + n * 8;
          ld_b_kmajor<128>(sb, n0, n0 + 8, kb * 32, lane, bf);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = n0 + e * 8 + c2;
            const float fb0 = ldexpf(1.0f, (int)sfb[(col & 31) * 16 + (col >> 5) * 4 + kb] - 127);
            const float fb1 = ldexpf(1.0f, (int)sfb[((col + 1) & 31) * 16 + ((col + 1) >> 5) * 4 + kb] - 127);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              float p[4] = {0.f, 0.f, 0.f, 0.f};
              mma_e4m3(p, af[mt], bf[2 * e], bf[2 * e + 1]);
              acc[n + e][mt][0] += p[0] * fa[mt][0] * fb0;
              acc[n + e][mt][1] += p[1] * fa[mt][0] * fb1;
              acc[n + e][mt][2] += p[2] * fa[mt][1] * fb0;
              acc[n + e][mt][3] += p[3] * fa[mt][1] * fb1;
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
      if (++st == kMxStages) { st = 0; phase ^= 1u; }
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = (int64_t)mb * 128 + qd * 32 + mt * 16 + g8 + 8 * h;
        if (m >= a.m_rows) continue;
        __nv_bfloat16* dst = a.C + m * a.n_total + nb * BN + half * 64 + c2;
#pragma unroll
        for (int n = 0; n < 8; ++n)
          *reinterpret_cast<uint32_t*>(dst + n * 8) = pack_bf16x2(acc[n][mt][2 * h], acc[n][mt][2 * h + 1]);
      }
  }
}

// ------------------------------------------------------------------------------------------------------------
// wgrad: MN-major operands (pixel axis = K), up to 3 taps per CTA, split over pixel ranges
// ------------------------------------------------------------------------------------------------------------
struct WgArgs {
  int co_tiles, ci_tiles;     // 128-wide tiles (64-wide when CT = 64)
  int groups;                 // tap groups (1 for a 1x1 convolution, 3 filter rows for 3x3)
  int taps_per;               // taps in a group (1 or 3)
  int gshift[3];              // row shift of X for the FIRST tap of group g (the others follow at +1, +2)
  int ksplit, kchunks;        // pixel-range splits, 64-row chunks in total
  int Co, Ci;
  float* dW;                  // [taps][Co][Ci] fp32, accumulated with RED
};

// The dY operand (MMA "A", M = output channels) is always 128 channels = two 64-channel atoms; when Co = 64 the
// second atom lies outside the tensor and TMA fills it with zeros. CT = input-channel tile (MMA N): 64 or 128.
template <int CT>
struct WgCfg {
  static constexpr int ATOMS = CT / 64;                       // 64-channel (128-byte) atoms of the X operand
  static constexpr int A_ATOM = 64 * 128;                     // dY: 64 k-rows x 128 B
  static constexpr int B_ROWS = 72;                           // X: 64 rows, rounded up with slack
  static constexpr int B_ATOM = B_ROWS * 128;
  static constexpr int A_BYTES = 2 * A_ATOM;
  static constexpr int B_BYTES = ATOMS * B_ATOM;
  static constexpr int STAGE = ((A_BYTES + B_BYTES + 1023) / 1024) * 1024;
  static constexpr int NSTAGE = CT == 128 ? 5 : 7;
  static constexpr int SMEM = NSTAGE * STAGE + 256 + 1024;
  static constexpr int NT = CT / 16;                          // n8 tiles per compute warp (half of CT)
};

// Warps 0..7 compute (warp w: output channels 32*(w%4) .. +31, input channels (w/4)*CT/2 .. +CT/2; both operands
// read from their [pixel][channel] tiles with ldmatrix.trans, pixels = K), warp 8 is the TMA producer. A unit is
// one (Co tile, Ci tile, tap, pixel range): its accumulators are flushed with fp32 RED.
template <int CT>
__global__ void __launch_bounds__(288, 1)
wgrad_mn_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WgArgs a) {
  using Cfg = WgCfg<CT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::NSTAGE * Cfg::STAGE);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::NSTAGE;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmDY);
    prefetch_tmap(&tmX);
    for (int s = 0; s < Cfg::NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int units = a.co_tiles * a.ci_tiles * a.groups * a.taps_per * a.ksplit;
  const int per_split = (a.kchunks + a.ksplit - 1) / a.ksplit;

  auto decode = [&](int u, int& co0, int& ci0, int& g, int& j, int& c0, int& c1) {
    const int ks = u % a.ksplit;
    int r = u / a.ksplit;
    j = r % a.taps_per;
    r /= a.taps_per;
    g = r % a.groups;
    r /= a.groups;
    ci0 = (r % a.ci_tiles) * CT;
    co0 = (r / a.ci_tiles) * 128;
    c0 = ks * per_split;
    c1 = min(a.kchunks, c0 + per_split);
  };

  if (warp == 8) {
    if (elect_one()) {
      int st = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int co0, ci0, g, j, c0, c1;
        decode(u, co0, ci0, g, j, c0, c1);
        for (int c = c0; c < c1; ++c) {
          mbar_wait(&empty[st], phase ^ 1u);
          uint8_t* s = smem + st * Cfg::STAGE;
          mbar_expect_tx(&full[st], Cfg::A_BYTES + Cfg::B_BYTES);
          for (int at = 0; at < 2; ++at) tma_load_2d(s + at * Cfg::A_ATOM, &tmDY, co0 + at * 64, c * 64, &full[st]);
          for (int at = 0; at < Cfg::ATOMS; ++at)
            tma_load_2d(s + Cfg::A_BYTES + at * Cfg::B_ATOM, &tmX, ci0 + at * 64, c * 64 + a.gshift[g] + j, &full[st]);
          if (++st == Cfg::NSTAGE) { st = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }
  const int qd = warp & 3, half = warp >> 2;
  const int lrow = lane & 7, ia = lane >> 3;
  int st = 0;
  uint32_t phase = 0;
  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    int co0, ci0, g, j, c0, c1;
    decode(u, co0, ci0, g, j, c0, c1);
    if (c1 <= c0) continue;
    float acc[Cfg::NT][2][4];
#pragma unroll
    for (int n = 0; n < Cfg::NT; ++n)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[n][mt][q] = 0.f;
    for (int c = c0; c < c1; ++c) {
      mbar_wait(&full[st], phase);
      const uint32_t sa = smem_u32(smem + st * Cfg::STAGE);
      const uint32_t sb = sa + Cfg::A_BYTES;
#pragma unroll
      for (int k = 0; k < 4; ++k) {                       // 4 x 16 pixel rows per chunk
        uint32_t af[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const int m = qd * 32 + mt * 16 + (ia & 1) * 8;   // output channel of this lane's 8x8 matrix
          ldsm_x4_t(swz<128>(sa + (m >> 6) * Cfg::A_ATOM + (k * 16 + (ia >> 1) * 8 + lrow) * 128 + (m & 63) * 2), af[mt]);
        }
#pragma unroll
        for (int n = 0; n < Cfg::NT; n += 2) {
          uint32_t bf[4];
          const int nn = half * (CT / 2) + (n + (ia >> 1)) * 8;   // input channel of this lane's 8x8 matrix
          ldsm_x4_t(swz<128>(sb + (nn >> 6) * Cfg::B_ATOM + (k * 16 + (ia & 1) * 8 + lrow) * 128 + (nn & 63) * 2), bf);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma_bf16(acc[n][mt], af[mt], bf[0], bf[1]);
            mma_bf16(acc[n + 1][mt], af[mt], bf[2], bf[3]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
      if (++st == Cfg::NSTAGE) { st = 0; phase ^= 1u; }
    }
    const int tap = g * a.taps_per + j;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int co = co0 + qd * 32 + mt * 16 + (lane >> 2) + 8 * h;
        if (co >= a.Co) continue;
        float* dst = a.dW + ((size_t)tap * a.Co + co) * a.Ci + ci0 + half * (CT / 2) + 2 * (lane & 3);
#pragma unroll
        for (int n = 0; n < Cfg::NT; ++n)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + n * 8), "f"(acc[n][mt][2 * h]),
                       "f"(acc[n][mt][2 * h + 1])
                       : "memory");
      }
  }
}

template <int CT>
void launch_wgrad_mn(const void* DY, const void* X, const WgArgs& a, int64_t rows, cudaStream_t st) {
  using Cfg = WgCfg<CT>;
  const CUtensorMap tmDY = map2d(DY, 2, (uint64_t)a.Co, (uint64_t)rows, (uint64_t)a.Co * 2, 64, 64);
  const CUtensorMap tmX = map2d(X, 2, (uint64_t)a.Ci, (uint64_t)rows, (uint64_t)a.Ci * 2, 64, Cfg::B_ROWS);
  auto kern = wgrad_mn_kernel<CT>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
  const int units = a.co_tiles * a.ci_tiles * a.groups * a.taps_per * a.ksplit;
  const int grid = std::min(units, hefl::cuda::device_sm_count());
  kern<<<grid, 288, Cfg::SMEM, st>>>(tmDY, tmX, a);
  hefl::cuda::note_launch();
}

// ------------------------------------------------------------------------------------------------------------
// data movement around the GEMMs: one pass each (ATen needs a fill + a strided copy, resp. cast + permute + flip)
// ------------------------------------------------------------------------------------------------------------
// x [B][H][W][C] -> xp [B][H+2][W+2][C] with a zero border; 16-byte vectors, C % 8 == 0
__global__ void pad_nhwc_kernel(const uint4* __restrict__ x, uint4* __restrict__ xp, int B, int H, int W, int C8) {
  const int Hp = H + 2, Wp = W + 2;
  const int64_t total = (int64_t)B * Hp * Wp * C8;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8);
    int64_t p = i / C8;
    const int wp = (int)(p % Wp);
    p /= Wp;
    const int hp = (int)(p % Hp);
    const int b = (int)(p / Hp);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (hp >= 1 && hp <= H && wp >= 1 && wp <= W) v = x[(((int64_t)b * H + hp - 1) * W + wp - 1) * C8 + c];
    xp[i] = v;
  }
}

// w fp32 [Co][Ci][3][3] -> wt bf16 [tap][Co][Ci] (forward) and wd bf16 [tap][Ci][Co] with the filter rotated by 180
// degrees (dgrad); for k = 1: wt [Co][Ci] and wd = its transpose [Ci][Co]. One 32 x 32 (co, ci) tile per block and
// tap, transposed through shared memory so that both outputs are written with unit stride.
__global__ void __launch_bounds__(256)
conv_weight_prep_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ wt, __nv_bfloat16* __restrict__ wd,
                        int Co, int Ci, int kk) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int tap = blockIdx.z;
  const int ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;            // 32 x 8
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int co = co0 + ty + 8 * r, ci = ci0 + tx;
    if (co < Co && ci < Ci) {
      const __nv_bfloat16 v = __float2bfloat16(w[((int64_t)co * Ci + ci) * kk + tap]);
      tile[ty + 8 * r][tx] = v;
      wt[((int64_t)tap * Co + co) * Ci + ci] = v;
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int ci = ci0 + ty + 8 * r, co = co0 + tx;
    if (co < Co && ci < Ci) wd[((int64_t)(kk - 1 - tap) * Ci + ci) * Co + co] = tile[tx][ty + 8 * r];
  }
}

// dW fp32 [tap][Co][Ci] -> grad fp32 [Co][Ci][kh][kw]
__global__ void conv_wgrad_unpack_kernel(const float* __restrict__ dw, float* __restrict__ g, int Co, int Ci, int kk) {
  const int64_t total = (int64_t)kk * Co * Ci;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int tap = (int)(i % kk);
    const int64_t cc = i / kk;                     // co * Ci + ci
    g[i] = dw[(int64_t)tap * Co * Ci + cc];
  }
}

}  // namespace

void pad_nhwc(const void* x, void* xp, int B, int H, int W, int C, cudaStream_t st) {
  if (C % 8) throw std::runtime_error("pad_nhwc: C must be a multiple of 8");
  const int64_t total = (int64_t)B * (H + 2) * (W + 2) * (C / 8);
  int blocks = (int)((total + 255) / 256);
  blocks = std::min(blocks, hefl::cuda::device_sm_count() * 16);
  pad_nhwc_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(xp), B, H, W, C / 8);
  hefl::cuda::note_launch();
}

void conv_weight_prep(const float* w, void* wt, void* wd, int Co, int Ci, int kk, cudaStream_t st) {
  dim3 grid((Ci + 31) / 32, (Co + 31) / 32, kk);
  conv_weight_prep_kernel<<<grid, 256, 0, st>>>(w, reinterpret_cast<__nv_bfloat16*>(wt), reinterpret_cast<__nv_bfloat16*>(wd), Co, Ci, kk);
  hefl::cuda::note_launch();
}

void conv_wgrad_unpack(const float* dw, float* g, int Co, int Ci, int kk, cudaStream_t st) {
  const int64_t total = (int64_t)kk * Co * Ci;
  int blocks = (int)((total + 255) / 256);
  blocks = std::min(blocks, hefl::cuda::device_sm_count() * 8);
  conv_wgrad_unpack_kernel<<<blocks, 256, 0, st>>>(dw, g, Co, Ci, kk);
  hefl::cuda::note_launch();
}

// Block-scaled e4m3 GEMM; sfa / sfb in the tiled layout described at MxArgs.
void gemm_mxfp8(const void* A, const void* Bm, const void* sfa, const void* sfb, void* C, int64_t M, int N, int K,
                cudaStream_t st) {
  if (K % 128 != 0 || N % 128 != 0) throw std::runtime_error("gemm_mxfp8: K and N must be multiples of 128");
  MxArgs a{};
  a.m_tiles = (int)((M + 127) / 128);
  a.n_tiles = N / 128;
  a.kgroups = K / 128;
  a.n_total = N;
  a.m_rows = M;
  a.C = reinterpret_cast<__nv_bfloat16*>(C);
  a.sfa = reinterpret_cast<const uint8_t*>(sfa);
  a.sfb = reinterpret_cast<const uint8_t*>(sfb);
  const CUtensorMap tmA = map2d(A, 1, (uint64_t)K, (uint64_t)M, (uint64_t)K, 128, 128);
  const CUtensorMap tmB = map2d(Bm, 1, (uint64_t)K, (uint64_t)N, (uint64_t)K, 128, 128);
  cudaFuncSetAttribute(mx_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMxSmem);
  const int tiles = a.m_tiles * a.n_tiles;
  const int grid = std::min(tiles, hefl::cuda::device_sm_count());
  mx_gemm_kernel<<<grid, 288, kMxSmem, st>>>(tmA, tmB, a);
  hefl::cuda::note_launch();
}

// C[rows_out, N] (bf16) = sum_taps A[m + shift_t, K] . B[t*N + n, K]; see GemmArgs. fp8: A, B are e4m3 bytes.
void gemm_taps(const void* A, const void* Bm, void* C, int64_t a_rows, int N, int K, int taps, const int* shifts, int padded,
               int Bn, int H, int W, bool fp8, const float* scale_a, const float* scale_b, cudaStream_t st) {
  const int kbytes = fp8 ? K : 2 * K;
  if (kbytes % 128 != 0) throw std::runtime_error("gemm_taps: K must cover whole 128-byte blocks");
  if (N % 64 != 0) throw std::runtime_error("gemm_taps: N must be a multiple of 64");
  if (taps < 1 || taps > 9) throw std::runtime_error("gemm_taps: 1..9 taps");
  GemmArgs a{};
  a.m_tiles = (int)((a_rows + 127) / 128);
  a.kblocks = kbytes / 128;
  a.taps = taps;
  for (int t = 0; t < taps; ++t) a.shift[t] = shifts ? shifts[t] : 0;
  a.n_total = N;
  a.m_rows = a_rows;
  a.padded = padded;
  a.Bn = Bn; a.H = H; a.W = W; a.Hp = H + 2; a.Wp = W + 2;
  a.C = reinterpret_cast<__nv_bfloat16*>(C);
  a.scale_a = scale_a;
  a.scale_b = scale_b;
  const bool wide = N % 128 == 0;
  a.n_tiles = wide ? N / 128 : N / 64;
  if (wide) {
    if (fp8) launch_kmajor<128, true>(A, Bm, a, a_rows, K, st);
    else launch_kmajor<128, false>(A, Bm, a, a_rows, K, st);
  } else {
    if (fp8) launch_kmajor<64, true>(A, Bm, a, a_rows, K, st);
    else launch_kmajor<64, false>(A, Bm, a, a_rows, K, st);
  }
}

// dW[taps][Co][Ci] (fp32, must be zeroed by the caller) += dY[rows, Co]^T . X[rows + shift, Ci]; taps = 1 or 9
// (3x3 on a padded grid of row length Wp).
void wgrad_taps(const void* DY, const void* X, float* dW, int64_t rows, int Co, int Ci, int taps, int Wp, cudaStream_t st) {
  if (Co % 64 != 0 || Ci % 64 != 0) throw std::runtime_error("wgrad_taps: channel counts must be multiples of 64");
  if (taps != 1 && taps != 9) throw std::runtime_error("wgrad_taps: 1 or 9 taps");
  WgArgs a{};
  const bool wide = Ci % 128 == 0;
  const int ct = wide ? 128 : 64;
  a.co_tiles = (Co + 127) / 128;
  a.ci_tiles = Ci / ct;
  a.groups = taps == 9 ? 3 : 1;
  a.taps_per = taps == 9 ? 3 : 1;
  for (int g = 0; g < a.groups; ++g) a.gshift[g] = taps == 9 ? (g - 1) * Wp - 1 : 0;
  a.kchunks = (int)((rows + 63) / 64);
  const int base_units = a.co_tiles * a.ci_tiles * a.groups * a.taps_per;
  // about one wave of CTAs: longer K runs per unit, fewer REDs onto the same dW words
  int ks = (hefl::cuda::device_sm_count() + base_units - 1) / base_units;
  if (ks < 1) ks = 1;
  if (ks > a.kchunks) ks = a.kchunks;
  a.ksplit = ks;
  a.Co = Co; a.Ci = Ci;
  a.dW = dW;
  if (wide) launch_wgrad_mn<128>(DY, X, a, rows, st);
  else launch_wgrad_mn<64>(DY, X, a, rows, st);
}

}  // namespace nn
}  // namespace hefl
