// Layer-1 weight gradient from the POOLED gradient on the tensor cores (warp-level mma.sync): the gather of
// wgrad_gather.cu rewritten as four masked GEMMs.
//
// After ReLU + 2x2 max-pool the conv-grid gradient has one non-zero per window and channel, at the arg-max
// position code c = (dy, dx). Splitting the pooled gradient by code,
//     G_c[px, co] = g[px, co]  if unit (px, co) is active and its arg-max code is c,  else 0,
// turns the data-dependent gather into
//     dW[(r, q, ci), co] = sum_c sum_px  X[(2i + dy + r, 2j + dx + q), ci] * G_c[px, co],        px = (b, i, j)
// i.e. for each code a GEMM over the pooled pixels with an A operand that is a plain strided view of the input.
// With the s-packed layer-1 input (channels = pixels (x, x+1, x+2) x 3, nn_kernels.cu) the 16 channels of pixel
// (2j + dx) ARE the (q, ci) rows of filter row r, so M = 3 x 16, N = 32, K = 4 x pooled pixels: 0.125 warp
// instructions per (window, channel) against 2.6 for the FP32-pipe gather (profiles/ncu_summary.md prof_gather:
// 43 M warp instructions, issue-bound at 66 us). The masks are built once per strip with byte-wise SIMD compares
// (4 codes x 16 B per 8 channels) and never leave shared memory.
//
//   * one CTA walks a contiguous run of pooled rows ("strips"): consecutive strips of an image share two of
//     their four input rows, kept in a six-slot ring. One thread issues the copies of the next strip while the
//     current one is multiplied: each input row is one TMA tensor copy ([pixel pairs][2 x 16 ch], SWIZZLE_64B),
//     gradient and codes are plain bulk copies; all of them complete on one mbarrier per strip parity;
//   * both operands are read with ldmatrix.trans from "K rows, M/N contiguous" tiles whose 16-byte chunks are
//     XOR-swizzled so that every phase touches 8 distinct bank groups (A: the TMA swizzle, rows 64 B apart;
//     B: [pixel][32 co] rows at 64 B, written by the mask pass with the same pattern);
//   * the mask pass uses PRMT as an 8-entry table: the code bytes, nibble-duplicated by one multiply, are the
//     selector, the table is 0xFF at entry 4 + c, so one instruction yields the 16-bit masks of two channels;
//   * 8 warps = 8 x 16 pooled pixels of a strip; each keeps the full 48 x 32 fp32 tile (48 registers). At the end
//     every warp parks its tile in shared memory (no atomics: fp32 shared atomics are CAS loops on this part and
//     cost 29 % of the first version), the tiles are summed, and one fp32 RED per CTA and useful element goes to
//     the split-K buffer the other weight-gradient kernels use. The bias gradient is the sum of the active g,
//     taken in the mask pass.
//
// With the rs-packed one-channel input (channel 3r + s = pixel (h + r, w + s), nn_kernels.cu) the 16 channels of pixel
// (2i + dy, 2j + dx) already are all nine taps, so each code's GEMM has M = 16 (9 rows used) and a pooled row needs
// input rows 2i and 2i+1 only (wgrad0_mma_rs_kernel); the partial rows tap * 3 + 0 carry the result.
//
// With the compact RGB input ([P, 4] = R, G, B, 0; wgrad0_mma_compact_kernel) an input row is one plain 1-D bulk copy
// of W x 8 bytes into a 2 KB ring slot, and the 32 bytes at 16j (pixels 2j .. 2j+3 x 4 channels) are the A rows of
// window j: M = 16 = 4 pixel slots x 4 channels, read with ldmatrix.trans at a 16-byte row stride (8 rows = 128
// contiguous bytes, conflict-free without a swizzle). Slot s + dx holds tap s, so the two column parities keep separate
// accumulators (96 registers) and are folded when the warp tiles are parked: tile row 4s + ci of dx = 1 is added to row
// 4(s - 1) + ci of dx = 0.
//
// (Why mma.sync and not tcgen05 here: the B operand is produced by the CUDA cores, M x N is 48 x 32 and the
// kernel is bound by the 116 MB it reads; the legacy tensor path needs no TMEM / descriptor round trip for that.)
// Reference semantics: Keras Conv2D/MaxPooling2D backward of the first block (FLPyfhelin.py:120-121).
#include <cuda_bf16.h>

#include <cstdlib>

#include "../he/kernels.h"
#include "launch.cuh"
#include "nn.h"
#include "tc_common.cuh"

namespace hefl {
namespace nn {

namespace {

using namespace hefl::sm90;
using namespace hefl::tc;

constexpr int kT = 256;                 // 8 warps
constexpr int kPx = 128;                // pooled pixels per strip tile (Wp <= 128)
constexpr int kSlot = 8192;             // one input row: W <= 256 pixels x 32 B
constexpr int kSlotC = 2048 + 128;      // compact: W <= 256 pixels x 8 B + zeroed slack (window 127 reads 16 B past)
constexpr int kRing = 6;
constexpr int kGst = kPx * 64;          // staged g of a strip      [px][32] bf16
constexpr int kCst = kPx * 32;          // staged codes of a strip  [px][32] u8
constexpr int kGs = kPx * 64;           // one masked tile
constexpr int bar_off(int slot) { return kRing * slot + 2 * kGst + 2 * kCst + 4 * kGs; }
constexpr int kBarOff = bar_off(kSlot);
constexpr int kSmem = kBarOff + 64;     // 104 KB -> 2 CTAs / SM
constexpr int kSmemC = bar_off(kSlotC) + 64 + 8 * kT * 4;   // 77 KB (+ bias sums); registers keep it at 2 CTAs / SM
constexpr int kPartStride = 40;         // floats per row of a parked accumulator tile (bank spread)
constexpr int kPart = 48 * kPartStride + 32;   // one warp's tile + its bias sums
static_assert(8 * kPart * 4 <= bar_off(kSlotC), "parked tiles must fit in the operand buffers");

// FR = filter rows that are separate GEMMs: 3 on the s-packed input (M = 3 x 16, a strip reads input rows 2i .. 2i+3),
// 1 on the rs-packed one-channel input (channel 3r + s = pixel (h + r, w + s): M = 16 with 9 rows used, a strip reads
// rows 2i and 2i+1 only, so consecutive strips share none). CPT: the compact RGB input (FR = 3; A = overlapping
// 32-byte rows of plain [pixel][4] rows, dx in separate accumulators).
template <int FR, bool CPT = false>
__device__ __forceinline__ void wgrad0_mma_body(const CUtensorMap* tmX, const __nv_bfloat16* __restrict__ xc,
                                                const __nv_bfloat16* __restrict__ g,
                                                const uint8_t* __restrict__ amax, float* __restrict__ ws, int B, int H,
                                                int W, int Hp, int Wp) {
  constexpr int NR = FR + 1;            // input rows under one pooled row
  constexpr int SLOT = CPT ? kSlotC : kSlot;
  constexpr int NDX = CPT ? 2 : 1;      // accumulator sets: column parities kept apart on the compact input
  extern __shared__ __align__(1024) uint8_t sm[];
  uint8_t* ring = sm;
  uint8_t* gst = ring + kRing * SLOT;
  uint8_t* cst = gst + 2 * kGst;
  uint8_t* Gs = cst + 2 * kCst;
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + bar_off(SLOT));   // [2]: everything strip s needs, by strip parity
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // stale / never-written shared memory is multiplied by zero masks: it has to be finite
  for (int i = tid; i < (kRing * SLOT) / 16; i += kT) reinterpret_cast<uint4*>(ring)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (tid == 0) {
    if constexpr (!CPT) prefetch_tmap(tmX);
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_barrier_init();
  }
  fence_proxy_async();                 // the zeros (generic proxy) before the TMA writes (async proxy)
  __syncthreads();
  pdl_prologue();

  const long long S = (long long)B * Hp;
  const int s0 = (int)(S * blockIdx.x / gridDim.x), s1 = (int)(S * (blockIdx.x + 1) / gridDim.x);
  const uint32_t row_bytes = (uint32_t)W * (CPT ? 8u : 32u), g_bytes = (uint32_t)Wp * 64u, c_bytes = (uint32_t)Wp * 32u;
  const int pairs = W >> 1;
  // input row `row` (of the B*H rows) into ring slot `sl`
  auto load_row = [&](int sl, int row, uint64_t* bar) {
    if constexpr (CPT) bulk_load_1d(ring + sl * SLOT, xc + (size_t)row * W * 4, row_bytes, bar);
    else tma_load_2d(ring + sl * SLOT, tmX, 0, row * pairs, bar);
  };

  float acc[FR][NDX][4][4];
#pragma unroll
  for (int r = 0; r < FR; ++r)
#pragma unroll
    for (int d = 0; d < NDX; ++d)
#pragma unroll
      for (int n = 0; n < 4; ++n) acc[r][d][n][0] = acc[r][d][n][1] = acc[r][d][n][2] = acc[r][d][n][3] = 0.f;
  float bsum[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
  // compact: the bias sums wait in shared memory ([e][thread]) between mask passes, so that the 96 accumulators fit
  // in 128 registers without spills (the same additions in the same order)
  float* bs = reinterpret_cast<float*>(sm + bar_off(SLOT) + 64) + tid;
  if constexpr (CPT) {
#pragma unroll
    for (int e = 0; e < 8; ++e) bs[e * kT] = 0.f;
  }

  // lane-constant pieces of the ldmatrix addresses
  const int mq = lane >> 3, li = lane & 7;
  const int j0 = warp * 16;
  // A (slot = [pixel pair j][dx][16 ch], 16-byte chunk index XOR (j >> 1) & 3): matrices (k-half 0, m-half 0),
  // (0, 1), (1, 0), (1, 1) = a0..a3 of m16n8k16
  const int ja = j0 + (mq >> 1) * 8 + li;
  // compact: window ja's 32-byte row at 16 ja, the same for both dx
  const uint32_t a_off0 = CPT ? ja * 16 + ((mq & 1) << 4) : ja * 64 + (((0 + (mq & 1)) ^ ((ja >> 1) & 3)) << 4);
  const uint32_t a_off1 = CPT ? a_off0 : ja * 64 + (((2 + (mq & 1)) ^ ((ja >> 1) & 3)) << 4);
  // B: matrices (k-half 0, n-tile nb), (1, nb), (0, nb + 1), (1, nb + 1)
  const int pb = j0 + (mq & 1) * 8 + li;
  const uint32_t b_off0 = pb * 64 + ((((mq >> 1) + 0) ^ ((pb >> 1) & 3)) << 4);
  const uint32_t b_off2 = pb * 64 + ((((mq >> 1) + 2) ^ ((pb >> 1) & 3)) << 4);
  const uint32_t ring_u = smem_u32(ring), Gs_u = smem_u32(Gs);

  int head = 0;
  bool pref = false;                                         // strip s was requested during strip s - 1
  for (int s = s0; s < s1; ++s) {
    const int b = s / Hp, i = s - b * Hp;
    const int par = (s - s0) & 1;
    if (!pref) head = 0;
    const bool pref_next = (s + 1 < s1) && (i + 1 < Hp);
    if (tid == 0) {
      if (!pref) {                                           // first strip of the CTA or of an image: all of it, now
        mbar_expect_tx(&full[par], NR * row_bytes + g_bytes + c_bytes);
#pragma unroll
        for (int r = 0; r < NR; ++r) load_row(r, b * H + 2 * i + r, &full[par]);
        bulk_load_1d(gst + par * kGst, g + (size_t)s * Wp * 32, g_bytes, &full[par]);
        bulk_load_1d(cst + par * kCst, amax + (size_t)s * Wp * 32, c_bytes, &full[par]);
      }
      if (pref_next) {                                       // the next strip: two new rows, its gradient and codes
        const int q = par ^ 1;
        int sl4 = head + NR, sl5 = head + NR + 1;
        sl4 = sl4 >= kRing ? sl4 - kRing : sl4;
        sl5 = sl5 >= kRing ? sl5 - kRing : sl5;
        mbar_expect_tx(&full[q], 2 * row_bytes + g_bytes + c_bytes);
        load_row(sl4, b * H + 2 * i + NR, &full[q]);
        load_row(sl5, b * H + 2 * i + NR + 1, &full[q]);
        bulk_load_1d(gst + q * kGst, g + (size_t)(s + 1) * Wp * 32, g_bytes, &full[q]);
        bulk_load_1d(cst + q * kCst, amax + (size_t)(s + 1) * Wp * 32, c_bytes, &full[q]);
      }
    }
    mbar_wait(&full[par], ((s - s0) >> 1) & 1);

    if constexpr (CPT) {
#pragma unroll
      for (int e = 0; e < 8; ++e) bsum[e] = bs[e * kT];
    }
    // masks: item = (pooled pixel, 8 channels)
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int item = tid + it * kT;
      const int px = item >> 2, ch = item & 3;
      uint4 gv = make_uint4(0u, 0u, 0u, 0u);
      uint2 cv = make_uint2(0u, 0u);
      if (px < Wp) {
        gv = *reinterpret_cast<const uint4*>(gst + par * kGst + px * 64 + ch * 16);
        cv = *reinterpret_cast<const uint2*>(cst + par * kCst + px * 32 + ch * 8);
      }
      const uint32_t dsto = px * 64 + ((ch ^ ((px >> 1) & 3)) << 4);
      // selector nibbles (code, code) per channel: PRMT looks the mask byte up in {0,0,0,0, table}
      const uint32_t u0 = (cv.x & 0x07070707u) * 0x11u, u1 = (cv.y & 0x07070707u) * 0x11u;
      const uint32_t u0h = u0 >> 16, u1h = u1 >> 16;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint32_t tbl = 0xFFu << (8 * c);               // entry 4 + c: active and arg-max at position c
        uint4 o;
        o.x = gv.x & __byte_perm(0u, tbl, u0);
        o.y = gv.y & __byte_perm(0u, tbl, u0h);
        o.z = gv.z & __byte_perm(0u, tbl, u1);
        o.w = gv.w & __byte_perm(0u, tbl, u1h);
        *reinterpret_cast<uint4*>(Gs + c * kGs + dsto) = o;
      }
      {   // bias gradient: every active unit, whatever its position (entries 4..7)
        const uint32_t w0 = gv.x & __byte_perm(0u, 0xFFFFFFFFu, u0), w1 = gv.y & __byte_perm(0u, 0xFFFFFFFFu, u0h);
        const uint32_t w2 = gv.z & __byte_perm(0u, 0xFFFFFFFFu, u1), w3 = gv.w & __byte_perm(0u, 0xFFFFFFFFu, u1h);
        bsum[0] += __uint_as_float(w0 << 16); bsum[1] += __uint_as_float(w0 & 0xFFFF0000u);
        bsum[2] += __uint_as_float(w1 << 16); bsum[3] += __uint_as_float(w1 & 0xFFFF0000u);
        bsum[4] += __uint_as_float(w2 << 16); bsum[5] += __uint_as_float(w2 & 0xFFFF0000u);
        bsum[6] += __uint_as_float(w3 << 16); bsum[7] += __uint_as_float(w3 & 0xFFFF0000u);
      }
    }
    if constexpr (CPT) {
#pragma unroll
      for (int e = 0; e < 8; ++e) bs[e * kT] = bsum[e];
    }
    __syncthreads();

    if (j0 < Wp) {                                           // warp-uniform
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int dy = c >> 1;
        uint32_t bq[2][4];
        ldsm_x4_t(Gs_u + c * kGs + b_off0, bq[0]);
        ldsm_x4_t(Gs_u + c * kGs + b_off2, bq[1]);
#pragma unroll
        for (int r = 0; r < FR; ++r) {
          int slot = head + dy + r;
          slot = slot >= kRing ? slot - kRing : slot;
          const int d = CPT ? (c & 1) : 0;
          uint32_t a[4];
          ldsm_x4_t(ring_u + slot * SLOT + ((c & 1) ? a_off1 : a_off0), a);
          mma_bf16(acc[r][d][0], a, bq[0][0], bq[0][1]);
          mma_bf16(acc[r][d][1], a, bq[0][2], bq[0][3]);
          mma_bf16(acc[r][d][2], a, bq[1][0], bq[1][1]);
          mma_bf16(acc[r][d][3], a, bq[1][2], bq[1][3]);
        }
      }
    }
    __syncthreads();                                         // ring slots / masked tiles / staging are free again
    head = head + 2 >= kRing ? head + 2 - kRing : head + 2;
    pref = pref_next;
  }

  // every warp parks its tile (all copies have landed: the last strip requests nothing), then a plain sum
  float* part = reinterpret_cast<float*>(sm);
  {
    float* mine = part + warp * kPart;
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int r = 0; r < FR; ++r)
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int col = n * 8 + 2 * tq;
        *reinterpret_cast<float2*>(mine + (r * 16 + gq) * kPartStride + col) = make_float2(acc[r][0][n][0], acc[r][0][n][1]);
        *reinterpret_cast<float2*>(mine + (r * 16 + gq + 8) * kPartStride + col) =
            make_float2(acc[r][0][n][2], acc[r][0][n][3]);
      }
    if constexpr (CPT) {
      // dx = 1: tile row 4 (s + 1) + ci is tap s; each lane adds to rows only it owns in the dx = 1 tile (rows 0..3,
      // slot 0, are no tap of dx = 1)
      __syncwarp();
#pragma unroll
      for (int r = 0; r < FR; ++r)
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          const int col = n * 8 + 2 * tq;
          if (gq >= 4) {
            float2* p = reinterpret_cast<float2*>(mine + (r * 16 + gq - 4) * kPartStride + col);
            *p = make_float2(p->x + acc[r][1][n][0], p->y + acc[r][1][n][1]);
          }
          float2* p = reinterpret_cast<float2*>(mine + (r * 16 + gq + 4) * kPartStride + col);
          *p = make_float2(p->x + acc[r][1][n][2], p->y + acc[r][1][n][3]);
        }
    }
    if constexpr (CPT) {
#pragma unroll
      for (int e = 0; e < 8; ++e) bsum[e] = bs[e * kT];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {                            // lanes with the same (lane & 3) hold the same 8 channels
      float v = bsum[e];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane < 4) mine[48 * kPartStride + lane * 8 + e] = v;
    }
  }
  __syncthreads();
  for (int idx = tid; idx < 28 * 32; idx += kT) {
    const int row = idx >> 5, co = idx & 31;
    // partial row = tap * 3 + ci (as in wgrad0_reduce_kernel), 27 = bias
    float v = 0.f;
    if (FR == 3) {
      // tile row of (r, s, ci): r * 16 + s * 3 + ci on the s-packed input, r * 16 + 4 s + ci on the compact one
      int src;
      if constexpr (CPT) src = row < 27 ? ((row / 9) * 16 + ((row / 3) % 3) * 4 + row % 3) * kPartStride + co
                                        : 48 * kPartStride + co;
      else src = row < 27 ? ((row / 9) * 16 + row % 9) * kPartStride + co : 48 * kPartStride + co;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += part[w * kPart + src];
    } else if (row >= 27 || row % 3 == 0) {               // rs: tile row 3r + s holds tap 3r + s of channel 0
      const int src = row < 27 ? (row / 3) * kPartStride + co : 48 * kPartStride + co;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += part[w * kPart + src];
    }
    ws[(size_t)blockIdx.x * kWgrad0Part + idx] = v;
  }
}

__global__ void __launch_bounds__(kT, 2)
wgrad0_mma_kernel(const __grid_constant__ CUtensorMap tmX, const __nv_bfloat16* __restrict__ g,
                  const uint8_t* __restrict__ amax, float* __restrict__ ws, int B, int H, int W, int Hp, int Wp) {
  wgrad0_mma_body<3>(&tmX, nullptr, g, amax, ws, B, H, W, Hp, Wp);
}

__global__ void __launch_bounds__(kT, 2)
wgrad0_mma_rs_kernel(const __grid_constant__ CUtensorMap tmX, const __nv_bfloat16* __restrict__ g,
                     const uint8_t* __restrict__ amax, float* __restrict__ ws, int B, int H, int W, int Hp, int Wp) {
  wgrad0_mma_body<1>(&tmX, nullptr, g, amax, ws, B, H, W, Hp, Wp);
}

__global__ void __launch_bounds__(kT, 2)
wgrad0_mma_compact_kernel(const __nv_bfloat16* __restrict__ X, const __nv_bfloat16* __restrict__ g,
                          const uint8_t* __restrict__ amax, float* __restrict__ ws, int B, int H, int W, int Hp, int Wp) {
  wgrad0_mma_body<3, true>(nullptr, X, g, amax, ws, B, H, W, Hp, Wp);
}

}  // namespace

bool wgrad0_mma_supported(int W, int Wp, int CK, int Ci, int Co) {
  static const bool on = []() { const char* e = std::getenv("HEFL_WGRAD0_MMA"); return !(e && e[0] == '0'); }();
  return on && CK == 16 && Ci <= 3 && Co == 32 && W <= 256 && (W & 1) == 0 && Wp <= kPx && Wp >= 1;
}

// dW[out_row(i) * 32 + co] += sum over CTAs p (in order) of ws[p][i]: the same bits on every run, unlike fp32 atomics
__global__ void __launch_bounds__(256) wgrad0_reduce_kernel(const float* __restrict__ ws, int parts, float* __restrict__ dW) {
  __shared__ float red[256];
  const float s = sum_partials(ws, parts, kWgrad0Part, red);
  const int i = blockIdx.x * 32 + threadIdx.x;
  if (threadIdx.x >= 32 || i >= kWgrad0Part) return;
  const int row = i >> 5, co = i & 31;
  const int out_row = row < 27 ? (row / 3) * 16 + (row % 3) : 9 * 16;     // dW32 rows: tap*CK + ci, bias at 9*CK
  dW[out_row * 32 + co] += s;
}

int wgrad0_parts(int B, int Hp) {
  const int sms = hefl::cuda::device_sm_count();
  return sms * 2 < B * Hp ? sms * 2 : B * Hp;
}

void wgrad0_reduce(const float* ws, int parts, float* dW, cudaStream_t st) {
  wgrad0_reduce_kernel<<<(kWgrad0Part + 31) / 32, 256, 0, st>>>(ws, parts, dW);
  hefl::cuda::note_launch();
}

void wgrad0_mma(const void* X, const void* g, const uint8_t* amax, float* dW, float* ws, int B, int H, int W, int Hp,
                int Wp, int in_channels, cudaStream_t st) {
  static bool attrs_set = false;
  if (!attrs_set) {
    for (auto* k : {wgrad0_mma_kernel, wgrad0_mma_rs_kernel}) {
      cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
      cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    }
    attrs_set = true;
  }
  // X viewed as [pixel pairs][2 x 16 channels]: one box = one image row, 64-byte swizzle
  const CUtensorMap tmX = tensor_map(X, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, {32, (uint64_t)B * H * (W / 2)}, {64},
                                     {32, (uint32_t)(W / 2)}, CU_TENSOR_MAP_SWIZZLE_64B);
  const int grid = wgrad0_parts(B, Hp);
  launch_pdl(in_channels == 1 ? wgrad0_mma_rs_kernel : wgrad0_mma_kernel, dim3(grid), dim3(kT), kSmem, st, tmX,
             reinterpret_cast<const __nv_bfloat16*>(g), amax, ws, B, H, W, Hp, Wp);
  hefl::cuda::note_launch();
  wgrad0_reduce(ws, grid, dW, st);
}

void wgrad0_mma_compact(const void* X, const void* g, const uint8_t* amax, float* dW, float* ws, int B, int H, int W,
                        int Hp, int Wp, cudaStream_t st) {
  static bool attrs_set = false;
  if (!attrs_set) {
    cudaFuncSetAttribute(wgrad0_mma_compact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemC);
    cudaFuncSetAttribute(wgrad0_mma_compact_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    attrs_set = true;
  }
  const int grid = wgrad0_parts(B, Hp);
  launch_pdl(wgrad0_mma_compact_kernel, dim3(grid), dim3(kT), kSmemC, st, reinterpret_cast<const __nv_bfloat16*>(X),
             reinterpret_cast<const __nv_bfloat16*>(g), amax, ws, B, H, W, Hp, Wp);
  hefl::cuda::note_launch();
  wgrad0_reduce(ws, grid, dW, st);
}

}  // namespace nn
}  // namespace hefl
