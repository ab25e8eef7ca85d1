// TMA-fed implicit-GEMM 3x3 convolution on the tensor cores for sm_90a (SURVEY.md K13-K15).
//
// Activations are NHWC bf16 viewed as a 2-D matrix [P = B*H*W pixels, C channels]. A 3x3 valid
// convolution is then 9 "tap" GEMMs whose A operand is the SAME matrix shifted by
// r*W + s rows:   Y[m, :] = sum_{r,s} X[m + r*W + s, :] * W[r,s]^T   (m on the input grid; rows
// with h >= H-2 or w >= W-2 are garbage and masked). Each tap's A tile is therefore one plain
// 2-D TMA box — no im2col buffer, no gather.
//
//   conv_fwd_pool : per CTA tile = 2 image rows x 128 columns (two accumulators) so that the
//                   epilogue does bias + ReLU + 2x2 max-pool + argmax straight from the accumulators (vertical
//                   max in-thread across the two accumulators, horizontal max by one shuffle) and
//                   writes only the pooled tensor (4x less HBM traffic than the conv output). Maps of even
//                   height and width <= 64 pack 128 / W row pairs into one tile instead (G1).
//   conv_dgrad    : dX[m,:] = sum_taps dY[m - off, :] * W[r,s]   (same kernel, negative offsets,
//                   plain bf16 store).
//   conv_wgrad    : dW[r,s] = sum_m X[m+off,:]^T dY[m,:]. Both operands are consumed in their
//                   native [P, C] layout (ldmatrix.trans, pixels = K), so no transposed copies exist;
//                   split-K over pixels and over filter rows, fp32 vector-RED into a [9*C+1, Co] buffer whose
//                   extra row is the bias gradient.
//
// Warp roles: eight compute warps (mma.sync with fp32 accumulators in registers, then the epilogue), one TMA
// producer warp; a smem ring of halo tiles with full/empty mbarriers lets TMA fill tile i+1 while tile i is
// multiplied (the tap-GEMM's compute warps are two groups of four that take alternate tiles, so one group's epilogue
// runs under the other's MMAs). Weights for all 9 taps stay resident in shared memory for the CTA's lifetime.
#include <cuda_bf16.h>

#include <stdexcept>

#include "../he/kernels.h"
#include "nn.h"
#include "tc_common.cuh"
#include "launch.cuh"

namespace hefl {
namespace nn {

using namespace hefl::sm90;
using namespace hefl::tc;

// ------------------------------------------------------------------------------------------
// host: tensor maps
// ------------------------------------------------------------------------------------------
// 2-D bf16 tensor [outer rows][inner cols], row pitch in bytes; box = box_inner x box_outer.
static CUtensorMap make_map(const void* ptr, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
                            uint32_t box_inner, uint32_t box_outer) {
  return tensor_map(ptr, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, {inner, outer}, {pitch_bytes}, {box_inner, box_outer},
                    swizzle_for(box_inner * 2));
}

// ------------------------------------------------------------------------------------------
// G1: halo-tile tap-GEMM kernel (forward + pool epilogue, or dgrad with plain store)
//
// A K-major swizzled tile written by TMA can be read starting at ANY row: the swizzle is a function of
// absolute shared-memory address bits (tc_common.cuh swz<>; umma_shift_probe checks it on the device). So each input row segment
// is loaded ONCE per tile and all 9 taps address shifted windows of it:
//   forward : tile = 2 image rows x 128 columns; 4 halo segments (rows h..h+3) of 130 pixels;
//             accumulator j (row h+j), tap (r,s) reads segment j+r at row offset s.
//   forward, row-packed (even H and W <= 64): a 2 x 128 tile of a narrow map would be mostly pixels of the
//             following rows whose results are discarded, so a tile is instead R = 128 / W image-row PAIRS
//             (pairs q0 .. q0+R-1, pair q = rows 2q, 2q+1 of the [B*H] row axis). Segment j holds R*W rows:
//             GEMM row m = k*W + w is column w of row 2(q0+k) + j (4-D tensor map, one TMA box per segment).
//             The accumulators, taps and row offsets are the ones above, so every output gets the same MMAs
//             in the same order (bit-identical results) on a fraction of the tiles.
//   forward, rs-packed input (one-channel layer 1, TS = kTapsRS): the input already carries the 3x3 neighbourhood
//             in its channels, so a tile is one tap on 2 halo segments (rows h, h+1), column or row-packed alike.
//   dgrad   :tile = 128 consecutive pixels; 3 segments starting at m0 - r*W - 2; tap (r,s)
//             reads segment r at row offset 2 - s.
// L2->SM traffic drops from 9 tap tiles to ~2 (fwd) / ~3 (dgrad) tiles per output tile.
// ------------------------------------------------------------------------------------------
struct TapGemmArgs {
  int B, H, W;          // input grid of the A matrix
  int Hp, Wp;           // pooled output grid (POOL)
  int tiles_w;          // column tiles per row pair (POOL, column tiling)
  int pairs_per_tile;   // POOL: R image-row pairs per tile when row-packed, 0 = 2 rows x 128 columns
  int num_tiles;
  int P;                // B*H*W
  int co_total;         // output channels of the layer (CO per CTA column block = blockIdx.y)
#ifdef HEFL_CONV_DEBUG
  int dbg;              // bottleneck isolation, ONLY in -DHEFL_CONV_DEBUG builds: 1 = skip TMA data, 2 = skip MMAs, 4 = skip epilogue
#endif
  const float* bias;    // [CO] (POOL)
  __nv_bfloat16* out;   // POOL: [B,Hp,Wp,CO]; else [P,CO]
  uint8_t* argmax;      // POOL, may be null
  // tile -> (image, row pair, column tile) without integer division: q = umulhi(n, magic) is exact for
  // n, d < 2^16 with magic = ceil(2^32 / d) (the epilogue warps spent ~40 of their ~100 per-tile set-up
  // instructions in two software divisions)
  uint32_t magic_per_img, magic_tiles_w;
  uint32_t magic_w, magic_half_h;     // row-packed: GEMM row -> (pair, column), pair -> (image, pooled row)
};

// magic for fast_div(n, d) when every n is below n_max; 0 = divide at run time
static uint32_t div_magic(int n_max, int d) {
  return (n_max < 65536 && d > 1 && d < 65536) ? (uint32_t)((0x100000000ull + d - 1) / d) : 0u;
}

__device__ __forceinline__ int fast_div(int n, int d, uint32_t magic) {
  if (d == 1) return n;
  return magic ? (int)__umulhi((uint32_t)n, magic) : n / d;
}

// TS = filter taps along the image row that are separate GEMMs: 3 normally; 1 when the three horizontal taps
// are packed into the channel dimension by the producer of the input (layer 1: 3 channels x 3 taps = 9 of the
// 16 padded channels, written by preprocess_u8) — a third of the MMAs for the same bytes.
// TS = kTapsRS (0): the whole 3x3 neighbourhood is packed (rs layout of a one-channel layer 1: channel 3r + s =
// pixel (h + r, w + s)), so one GEMM per accumulator remains and a pooled tile needs only its own 2 image rows.
constexpr int kTapsRS = 0;

template <int CK, int CO, bool POOL, int TS = 3>
struct TapGemmCfg {
  static constexpr int NTAP = TS ? 3 * TS : 1;
  static constexpr int KB = CK < 64 ? CK : 64;            // channels per k-block (one swizzle atom)
  static constexpr int NKB = CK / KB;
  static constexpr int ROW_BYTES = KB * 2;
  static constexpr int NSEG = POOL ? (TS ? 4 : 2) : 3;
  static constexpr int NACC = POOL ? 2 : 1;
  static constexpr int SEG_ROWS = 136;                    // 130 used, multiple of 8
  static constexpr int SEG_BYTES = SEG_ROWS * ROW_BYTES;
  static constexpr int HALO = NKB * NSEG * SEG_BYTES;     // one tile's input
  static constexpr int W_SUB = CO * ROW_BYTES;
  static constexpr int W_TAP = W_SUB * NKB;
  static constexpr int W_BYTES = NTAP * W_TAP;
  static constexpr int BAR_BYTES = 384;
  static constexpr int SCR_BYTES = 8 * 1024;              // 1 KB accumulator staging per compute warp
  static constexpr int FIXED = W_BYTES + BAR_BYTES + SCR_BYTES + 1024;
  // 8-channel chunks per warp and pass: accumulators = NACC x NCH x 2 m16 tiles x 4 floats = 64 registers or fewer
  static constexpr int NCH = (CO / 8) < (8 / NACC) ? (CO / 8) : (8 / NACC);
  static constexpr int NPASS = CO / 8 / NCH;
  static constexpr int ACC_REGS = NACC * NCH * 8;
  // Two CTAs per SM when a two-tile ring fits twice and the accumulators leave room in the 96 registers a thread
  // then gets (64 accumulators spill there); otherwise one CTA per SM. The ring takes what the CTA's share of shared
  // memory holds, up to 4 tiles. Two consumer groups need a ring of at least 2 (one tile per group in flight); a ring
  // of 1 leaves one group.
  static constexpr int OCC = blocks_fit(FIXED + 2 * HALO, 2) && ACC_REGS <= 32 ? 2 : 1;
  static constexpr int SMEM_CAP = OCC == 2 ? 228 * 1024 / 2 - 1024 : kSmemMax;
  static constexpr int NBUF_FIT = (SMEM_CAP - FIXED) / HALO;
  static constexpr int NBUF = NBUF_FIT > 4 ? 4 : NBUF_FIT;
  static constexpr int SMEM = FIXED + NBUF * HALO;
  static constexpr int NGRP = NBUF >= 2 ? 2 : 1;
  static_assert(NBUF >= 1, "halo tile does not fit in shared memory");
  static_assert(blocks_fit(SMEM, OCC), "occupancy");
  static_assert(NCH % 2 == 0 && (CO / 8) % NCH == 0, "chunk passes");
  static_assert(CO % 32 == 0 && CO <= 128, "CO must be 32, 64, 96 or 128");
};

// Warp roles (DESIGN.md §4): warps 0..7 are two consumer groups of four; group w/4 takes the CTA's tiles k = w/4,
// w/4 + 2, ... and warp w owns GEMM rows 32*(w%4) .. +31 and all CO channels of the column block (NPASS passes of NCH
// 8-channel chunks). The groups hand the MMA loop to each other in tile order (named barriers 1 and 2), so one
// group's epilogue runs under the other group's MMAs and the two groups stay within one tile of each other. Warp 8 is
// the TMA producer and fills the ring in tile order. Accumulators live in registers (mma.sync m16n8k16).
template <int CK, int CO, bool POOL, int TS>
__global__ void __launch_bounds__(288, TapGemmCfg<CK, CO, POOL, TS>::OCC)
tap_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                const TapGemmArgs a) {
  using Cfg = TapGemmCfg<CK, CO, POOL, TS>;
  constexpr int RB = Cfg::ROW_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem;
  uint8_t* sA = smem + Cfg::W_BYTES;
  float* scr_all = reinterpret_cast<float*>(sA + Cfg::NBUF * Cfg::HALO);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(scr_all) + Cfg::SCR_BYTES);
  uint64_t* full = bars;                       // [NBUF]
  uint64_t* empty = bars + Cfg::NBUF;          // [NBUF]
  uint64_t* wfull = bars + 2 * Cfg::NBUF;      // [1]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmW);
    for (int s = 0; s < Cfg::NBUF; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: the set-up above and the weight tile (written only by the re-layout kernel, which never triggers its
  // dependents early — launch.cuh) overlap the previous kernel's tail; activations only after the wait.
  pdl_trigger();
  if (warp == 8 && elect_one()) {
    mbar_expect_tx(wfull, Cfg::W_BYTES);
    for (int tap = 0; tap < Cfg::NTAP; ++tap)
      for (int kb = 0; kb < Cfg::NKB; ++kb)
        tma_load_2d(sW + tap * Cfg::W_TAP + kb * Cfg::W_SUB, &tmW, kb * Cfg::KB,
                    tap * a.co_total + blockIdx.y * CO, wfull);
  }
  pdl_wait();

  if (warp == 8) {
    // ===== TMA producer =====
    if (elect_one()) {
      int buf = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < a.num_tiles; t += gridDim.x) {
        mbar_wait(&empty[buf], phase ^ 1);
        uint8_t* dst = sA + buf * Cfg::HALO;
#ifdef HEFL_CONV_DEBUG
        if (a.dbg & 1) {
          mbar_arrive(&full[buf]);
        } else
#endif
        if (POOL && a.pairs_per_tile) {
          // segment sg = row parity sg & 1 of pairs q0 + (sg >> 1) ..: rows 2(q0+k) + sg; bytes actually boxed
          const int q0 = t * a.pairs_per_tile;
          mbar_expect_tx(&full[buf], Cfg::NKB * Cfg::NSEG * a.pairs_per_tile * a.W * RB);
          for (int kb = 0; kb < Cfg::NKB; ++kb)
            for (int sg = 0; sg < Cfg::NSEG; ++sg)
              tma_load_4d(dst + (kb * Cfg::NSEG + sg) * Cfg::SEG_BYTES, &tmA, kb * Cfg::KB, 0, sg & 1, q0 + (sg >> 1),
                          &full[buf]);
        } else {
          int base, seg_stride;
          if (POOL) {
            const int per_img = a.Hp * a.tiles_w;
            const int b = fast_div(t, per_img, a.magic_per_img);
            const int rem = t - b * per_img;
            const int hp = fast_div(rem, a.tiles_w, a.magic_tiles_w);
            const int tw = rem - hp * a.tiles_w;
            base = (b * a.H + 2 * hp) * a.W + tw * 128;
            seg_stride = a.W;                      // segment j = image row h + j
          } else {
            base = t * 128 - 2;
            seg_stride = -a.W;                     // segment r starts at m0 - r*W - 2
          }
          mbar_expect_tx(&full[buf], Cfg::HALO);
          for (int kb = 0; kb < Cfg::NKB; ++kb)
            for (int sg = 0; sg < Cfg::NSEG; ++sg)
              tma_load_2d(dst + (kb * Cfg::NSEG + sg) * Cfg::SEG_BYTES, &tmA, kb * Cfg::KB, base + sg * seg_stride,
                          &full[buf]);
        }
        if (++buf == Cfg::NBUF) { buf = 0; phase ^= 1; }
      }
    }
  } else {
    // ===== consumer group grp (warps 4*grp .. +3): tiles kt = grp, grp + NGRP, ...; rows qd*32 .. +31, all channels
    const int qd = warp & 3;
    const int grp = warp >> 2;
    if (grp >= Cfg::NGRP) return;
    float* scr = scr_all + warp * 256;
    const uint32_t w_base = smem_u32(sW);
    mbar_wait(wfull, 0);
    for (int kt = grp, t = blockIdx.x + grp * gridDim.x; t < a.num_tiles; kt += Cfg::NGRP, t += Cfg::NGRP * gridDim.x) {
      const int buf = kt % Cfg::NBUF;
      mbar_wait(&full[buf], (kt / Cfg::NBUF) & 1);
      const uint32_t a_base = smem_u32(sA + buf * Cfg::HALO);
      // MMA turn: the CTA's tile kt starts its MMAs once tile kt-1 (the other group's) has finished its own
      if (Cfg::NGRP == 2 && kt > 0) named_barrier_sync(1 + grp, 256);
#pragma unroll 1
      for (int g = 0; g < Cfg::NPASS; ++g) {
        float acc[Cfg::NACC][Cfg::NCH][2][4];
#pragma unroll
        for (int j = 0; j < Cfg::NACC; ++j)
#pragma unroll
          for (int i = 0; i < Cfg::NCH; ++i)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int q = 0; q < 4; ++q) acc[j][i][mt][q] = 0.f;
        // three taps per iteration (one filter row): their row shifts are constants, and the next tap's fragment loads
        // are issued under the current tap's MMAs instead of after a loop back-edge
#ifdef HEFL_CONV_DEBUG
        if (!(a.dbg & 2))
#endif
#pragma unroll 3
        for (int tap = 0; tap < Cfg::NTAP; ++tap) {
          const int r = TS ? tap / (TS ? TS : 1) : 0, s = TS ? tap % (TS ? TS : 1) : 0;
          const int shift = POOL ? s : (2 - s);
#pragma unroll
          for (int kb = 0; kb < Cfg::NKB; ++kb) {
#pragma unroll
            for (int ks = 0; ks < Cfg::KB / 16; ++ks) {
              uint32_t bf[Cfg::NCH / 2][4];
#pragma unroll
              for (int i = 0; i < Cfg::NCH; i += 2) {
                const int c0 = g * Cfg::NCH + i;
                ld_b_kmajor<RB>(w_base + tap * Cfg::W_TAP + kb * Cfg::W_SUB, c0 * 8, (c0 + 1) * 8, ks * 32, lane,
                                bf[i / 2]);
              }
#pragma unroll
              for (int j = 0; j < Cfg::NACC; ++j) {
                const int seg = POOL ? (j + r) : r;
                const uint32_t seg_base = a_base + (kb * Cfg::NSEG + seg) * Cfg::SEG_BYTES;
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                  uint32_t af[4];
                  ld_a_kmajor<RB>(seg_base, shift + qd * 32 + mt * 16, ks * 32, lane, af);
#pragma unroll
                  for (int i = 0; i < Cfg::NCH; ++i)
                    mma_bf16(acc[j][i][mt], af, bf[i / 2][(i & 1) * 2], bf[i / 2][(i & 1) * 2 + 1]);
                }
              }
            }
          }
        }
        if (g == Cfg::NPASS - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[buf]);     // this warp's last read of the halo tile is done
          if (Cfg::NGRP == 2 && t + (int)gridDim.x < a.num_tiles) named_barrier_arrive(2 - grp, 256);
        }
        // POOL: pooled pixel of this lane's conv column (window = this lane and lane ^ 1) and whether it is stored
        int pix = 0;
        bool writer = false;
        if (POOL) {
          if (a.pairs_per_tile) {
            // W even: m and w have the same parity, so lane ^ 1 is the other column of the same window
            const int m = qd * 32 + lane;
            const int k = fast_div(m, a.W, a.magic_w);
            const int w = m - k * a.W;
            const int half_h = a.H >> 1;
            const int q = t * a.pairs_per_tile + k;
            const int b = fast_div(q, half_h, a.magic_half_h);
            const int hp = q - b * half_h;                      // the last pair of an image is never a pooled row
            writer = k < a.pairs_per_tile && b < a.B && hp < a.Hp && (w >> 1) < a.Wp;
            pix = (b * a.Hp + hp) * a.Wp + (w >> 1);
          } else {
            const int per_img = a.Hp * a.tiles_w;
            const int b = fast_div(t, per_img, a.magic_per_img);
            const int rem = t - b * per_img;
            const int hp = fast_div(rem, a.tiles_w, a.magic_tiles_w);
            const int tw = rem - hp * a.tiles_w;
            const int wp = (tw * 128 + qd * 32 + lane) >> 1;   // conv-output column of this thread, halved
            writer = wp < a.Wp;
            pix = (b * a.Hp + hp) * a.Wp + wp;
          }
        }
#pragma unroll
        for (int i = 0; i < Cfg::NCH; ++i) {
          const int ch = g * Cfg::NCH + i;
#ifdef HEFL_CONV_DEBUG
          if (a.dbg & 4) continue;
#endif
          if (POOL) {
            const bool odd = (lane & 1) != 0;
            const int c0 = blockIdx.y * CO + ch * 8 + (odd ? 4 : 0);   // channel of the layer's co_total
            float v0[8], v1[8];
            frag_rows(scr, acc[0][i][0], acc[0][i][1], lane, v0);
            frag_rows(scr, acc[Cfg::NACC - 1][i][0], acc[Cfg::NACC - 1][i][1], lane, v1);
            // the two lanes of a window split the 8 channels: even lane -> 0..3, odd lane -> 4..7
            const float4 bq = __ldg(reinterpret_cast<const float4*>(a.bias + c0));
            const float bias4[4] = {bq.x, bq.y, bq.z, bq.w};
            // max over the two image rows on the raw accumulators (bias + ReLU commute with max)
            uint32_t vbits = 0;                                 // 1 = lower image row wins
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              const bool lw = v1[c] > v0[c];
              v0[c] = lw ? v1[c] : v0[c];
              vbits |= lw ? (1u << c) : 0u;
            }
            const uint32_t pvbits = __shfl_xor_sync(0xffffffffu, vbits, 1);
            const uint32_t mb = (vbits >> (odd ? 4 : 0)) & 15u;   // row bits of my column, my 4 channels
            const uint32_t pb = (pvbits >> (odd ? 4 : 0)) & 15u;  // ... of the partner's column
            float x[4];
            uint32_t idx = 0u;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float keep = odd ? v0[4 + q] : v0[q];
              const float send = odd ? v0[q] : v0[4 + q];
              const float recv = __shfl_xor_sync(0xffffffffu, send, 1);
              const float left = odd ? recv : keep, right = odd ? keep : recv;
              const bool rw = right > left;                       // right column wins only if strictly greater
              const uint32_t rowbit = ((rw != odd) ? (pb >> q) : (mb >> q)) & 1u;
              const float y = (rw ? right : left) + bias4[q];
              // bits 0-1: arg-max position (row*2 + col) in the window, bit 2: unit active (ReLU mask)
              idx |= ((rowbit << 1) | (rw ? 1u : 0u) | (y > 0.f ? 4u : 0u)) << (q * 8);
              x[q] = y > 0.f ? y : 0.f;
            }
            if (writer) {
              const size_t o = (size_t)pix * a.co_total + c0;
              *reinterpret_cast<uint2*>(a.out + o) = make_uint2(pack_bf16x2(x[0], x[1]), pack_bf16x2(x[2], x[3]));
              if (a.argmax) *reinterpret_cast<uint32_t*>(a.argmax + o) = idx;
            }
          } else {
            const int m = t * 128 + qd * 32 + lane;
            float v[8];
            frag_rows(scr, acc[0][i][0], acc[0][i][1], lane, v);
            if (m < a.P) {
              const int c0 = blockIdx.y * CO + ch * 8;
              *reinterpret_cast<uint4*>(a.out + (size_t)m * a.co_total + c0) =
                  make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                             pack_bf16x2(v[6], v[7]));
            }
          }
        }
      }
    }
  }
}

template <int CK, int CO, bool POOL, int TS = 3>
static void launch_tap_gemm(const __nv_bfloat16* A, const __nv_bfloat16* Wt, TapGemmArgs a, cudaStream_t st) {
  using Cfg = TapGemmCfg<CK, CO, POOL, TS>;
  CUtensorMap tmA;
  if (POOL && a.pairs_per_tile) {
    // [B*H rows][W][CK] viewed as image-row pairs, 4-D {CK, W, row parity, B*H/2 pairs}: one box is pairs_per_tile * W
    // consecutive smem rows of one parity (pairs past the end zero-fill)
    const uint64_t W = (uint64_t)a.W, pairs = (uint64_t)a.B * a.H / 2;
    tmA = tensor_map(A, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, {CK, W, 2, pairs}, {CK * 2, W * CK * 2, 2 * W * CK * 2},
                     {Cfg::KB, (uint32_t)a.W, 1, (uint32_t)a.pairs_per_tile}, swizzle_for(Cfg::KB * 2));
  } else {
    tmA = make_map(A, CK, (uint64_t)a.P, (uint64_t)CK * 2, Cfg::KB, Cfg::SEG_ROWS);
  }
  const CUtensorMap tmW = make_map(Wt, CK, (uint64_t)Cfg::NTAP * a.co_total, (uint64_t)CK * 2, Cfg::KB, CO);
  auto kern = tap_gemm_kernel<CK, CO, POOL, TS>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
  const int ny = a.co_total / CO;
  const int slots = hefl::cuda::device_sm_count() * Cfg::OCC / ny;
  int gx = a.num_tiles < slots ? a.num_tiles : slots;
  if (gx < 1) gx = 1;
  dim3 grid(gx, ny);
  launch_pdl(kern, grid, dim3(288), Cfg::SMEM, st, tmA, tmW, a);
  hefl::cuda::note_launch();
}

// The work-skipping switch exists only in -DHEFL_CONV_DEBUG builds (HEFL_NVCC_EXTRA); release kernels carry
// no such code and conv_set_debug refuses to arm it.
#ifdef HEFL_CONV_DEBUG
static int g_dbg = 0;
void conv_set_debug(int mask) { g_dbg = mask; }
#else
void conv_set_debug(int mask) {
  if (mask != 0) throw std::runtime_error("conv_set_debug: this build has no debug switch (rebuild with -DHEFL_CONV_DEBUG)");
}
#endif

void conv_fwd_pool(const void* X, const void* Wf, const float* bias, void* out, uint8_t* argmax, int B, int H,
                   int W, int CK, int CO, int spack, int in_channels, cudaStream_t st) {
  TapGemmArgs a{};
#ifdef HEFL_CONV_DEBUG
  a.dbg = g_dbg;
#endif
  if (!((CK == 16 && CO == 32) || (CK == 32 && (CO == 32 || CO == 64)) || (CK == 64 && (CO == 64 || CO == 128))))
    throw std::runtime_error("conv_fwd_pool: unsupported (CK, CO)");
  a.B = B; a.H = H; a.W = W;
  a.Hp = (H - 2) / 2; a.Wp = (W - 2) / 2;
  if (W % 2 == 0 && H % 2 == 0 && W <= 64) {
    // row-packed tiles (G1 above): R = 128 / W pairs of image rows per tile instead of 2 rows x 128 columns;
    // even H keeps every pair inside one image, even W keeps both columns of a pooling window in one lane pair
    a.pairs_per_tile = 128 / W;
    const int pairs = B * H / 2;
    a.num_tiles = (pairs + a.pairs_per_tile - 1) / a.pairs_per_tile;
    a.magic_w = div_magic(128, W);
    a.magic_half_h = div_magic(a.num_tiles * a.pairs_per_tile, H / 2);
  } else {
    a.tiles_w = (2 * a.Wp + 127) / 128;
    a.num_tiles = B * a.Hp * a.tiles_w;
    a.magic_per_img = div_magic(a.num_tiles, a.Hp * a.tiles_w);
    a.magic_tiles_w = div_magic(a.num_tiles, a.tiles_w);
  }
  a.P = B * H * W;
  a.co_total = CO;
  a.bias = bias;
  a.out = reinterpret_cast<__nv_bfloat16*>(out);
  a.argmax = argmax;
  // Output-channel blocks (blockIdx.y) while the tiles alone would leave SMs idle (the late, small layers): a CTA
  // then holds and multiplies 1/ny of the weights, and the input tile is read once per block (from L2).
  int co_blk = CO;
  while (co_blk % 64 == 0 && a.num_tiles * (CO / co_blk) < hefl::cuda::device_sm_count()) co_blk /= 2;
  const auto* x = reinterpret_cast<const __nv_bfloat16*>(X);
  const auto* w = reinterpret_cast<const __nv_bfloat16*>(Wf);
  if (spack && !(CK == 16 && CO == 32 && (in_channels == 1 || in_channels == 3)))
    throw std::runtime_error("conv_fwd_pool: packed input is the 1- or 3-channel first layer (CK=16, CO=32) only");
  if (CK == 16 && spack && in_channels == 1) launch_tap_gemm<16, 32, true, kTapsRS>(x, w, a, st);
  else if (CK == 16 && spack) launch_tap_gemm<16, 32, true, 1>(x, w, a, st);
  else if (CK == 16) launch_tap_gemm<16, 32, true>(x, w, a, st);
  else if (CK == 32 && co_blk == 32) launch_tap_gemm<32, 32, true>(x, w, a, st);
  else if (CK == 32) launch_tap_gemm<32, 64, true>(x, w, a, st);
  else if (co_blk == 32) launch_tap_gemm<64, 32, true>(x, w, a, st);
  else if (co_blk == 64) launch_tap_gemm<64, 64, true>(x, w, a, st);
  else launch_tap_gemm<64, 128, true>(x, w, a, st);
}

void conv_dgrad(const void* dY, const void* Wd, void* dX, int B, int H, int W, int CK, int CO, cudaStream_t st) {
  TapGemmArgs a{};
#ifdef HEFL_CONV_DEBUG
  a.dbg = g_dbg;
#endif
  a.B = B; a.H = H; a.W = W;
  a.P = B * H * W;
  a.num_tiles = (a.P + 127) / 128;
  a.co_total = CO;
  a.out = reinterpret_cast<__nv_bfloat16*>(dX);
  const auto* x = reinterpret_cast<const __nv_bfloat16*>(dY);
  const auto* w = reinterpret_cast<const __nv_bfloat16*>(Wd);
  if (CK == 32 && CO == 32) launch_tap_gemm<32, 32, false>(x, w, a, st);
  else if (CK == 64 && CO == 32) launch_tap_gemm<64, 32, false>(x, w, a, st);
  else if (CK == 64 && CO == 64) launch_tap_gemm<64, 64, false>(x, w, a, st);
  else if (CK == 128 && CO == 64) launch_tap_gemm<128, 32, false>(x, w, a, st);   // two column blocks
  else throw std::runtime_error("conv_dgrad: unsupported (CK, CO)");
}

// ------------------------------------------------------------------------------------------
// G1b (layer 1 by default, HEFL_FWD_PAIR=0 / all to change): forward + pool with both columns of a pooling window in
// the SAME thread.
// Validated against G1 on hardware (tests/test_gpu_conv.py::test_conv_fwd_pool_pair_matches_plain_kernel: same
// pooled values and arg-max codes); 33.7 vs 40.4 us on layer 1 (B=32, 256x256), slower on the small layers.
//
// ncu on G1 (prof_fwd0_v4): the pool epilogue is the limiter of the forward kernels — 62 % issue-active,
// 6 % tensor pipe, ~33 instructions per pooled output — because a lane owns one conv COLUMN, so the 2x2 window
// needs a lane exchange (5 shuffles, 16 parity selects) per 8-channel chunk.
//
// Here the activation matrix [pixels, CK] is viewed as [pixel PAIRS, 2*CK] (same memory; needs an even image
// width so pairs never straddle rows). GEMM row j of accumulator (dy, dx) is window j of the pooled row:
//     acc(dy,dx)[j] = sum_{r,s} X[row 2hp+dy+r, column 2j+dx+s] . W[r,s]
// With e = dx + s, column 2j+e is pair-row j + (e >> 1), half e & 1: a row shift of the A descriptor plus a
// K byte offset of (e & 1) * CK * 2 inside the pair-row — both are things G1 already does (row-shifted starts,
// 32-byte K steps inside a swizzle atom). Four accumulators (2 rows x 2 column parities), M = 128 windows.
// The four accumulators share one fragment layout, so max/arg-max are element-wise on the fragments (no shuffles, no
// transpose); the pooled row is staged in shared memory and leaves the CTA as two TMA stores (values, codes).
// Restricted to CK <= 32 (one swizzle atom per pair-row) and CO <= 64 (4 accumulators in registers).
// ------------------------------------------------------------------------------------------
template <int CK, int CO, int NSEG_ = 4, int SEG_BYTES_ = 136 * 2 * CK * 2, int NBUF_ = 2>
struct PairFwdCfg {
  static constexpr int ROW_BYTES = 2 * CK * 2;            // one pair-row: 2 pixels x CK channels, 64 or 128 B
  static constexpr int NSEG = NSEG_;                      // image rows 2hp .. 2hp+3 (2hp, 2hp+1 on the rs layout)
  static constexpr int SEG_ROWS = 136;                    // 130 pair-rows used (128 windows + shift 1 + slack)
  static constexpr int SEG_BYTES = SEG_BYTES_;
  static constexpr int HALO = NSEG * SEG_BYTES;
  static constexpr int W_ROW = CK * 2;                    // weight rows: [tap][CO][CK], 32 or 64 B (as G1)
  static constexpr int W_TAP = CO * W_ROW;
  static constexpr int W_BYTES = 9 * W_TAP;
  static constexpr int BAR_BYTES = 384;
  // pooled output tile of one pooled row, staged for the TMA store: [128 windows][CO] bf16, then [128][CO] codes,
  // each laid out as its tensor map's swizzle (span = one row) so the fragment writes are free of bank conflicts;
  // two of them, so one is filled while the store of the other still reads it
  static constexpr int OUT_V = 128 * CO * 2;
  static constexpr int OUT_BYTES = OUT_V + 128 * CO;
  static constexpr int NBUF = NBUF_;
  static constexpr int SMEM = W_BYTES + NBUF * HALO + 2 * OUT_BYTES + BAR_BYTES + 1024;
  static constexpr int NACC = 4;
  static constexpr int NG = 2;                            // 8-channel chunks per warp and pass
  static constexpr int OCC = blocks_fit(SMEM, 2) ? 2 : 1;
  static_assert(CK == 16 || CK == 32, "pair-row forward: one swizzle atom per pair-row");
  static_assert(CO == 32 || CO == 64, "pair-row forward: CO is 32 or 64");
  static_assert(SMEM <= kSmemMax, "shared memory");
  static_assert((W_BYTES + NBUF * HALO) % 1024 == 0 && OUT_V % 1024 == 0 && OUT_BYTES % 1024 == 0,
                "output tiles start on the 1024-byte swizzle repeat");
};

struct PairFwdArgs {
  int B, H, W;          // input grid (W even)
  int Hp, Wp;           // pooled grid
  int num_tiles;        // B * Hp (one pooled row per tile; Wp <= 128)
#ifdef HEFL_CONV_DEBUG
  int dbg;              // as TapGemmArgs::dbg: 1 = skip TMA data, 2 = skip MMAs, 4 = skip epilogue
#endif
  const float* bias;
  __nv_bfloat16* out;   // [B,Hp,Wp,CO]
  uint8_t* argmax;      // may be null
};

// Input layouts (PK):
//   kPairPlain : CK channels per pixel, 9 tap GEMMs;
//   kPairS     : s-packed layer-1 input (channels = pixels x, x+1, x+2): the three horizontal taps are already inside
//                the 16 channels, so only the three filter rows remain — 3 MMAs per accumulator, column parity = K
//                byte offset;
//   kPairRS    : rs-packed one-channel layer-1 input (channel 3r + s = pixel (y + r, x + s)): one filter row,
//                acc(dy,dx)[j] = X[row 2hp+dy, pair-row j, half dx] . W — one MMA k-step per accumulator on a
//                2-row halo.
//   kPairC     : compact RGB layer-1 input, 8 bytes per pixel (R, G, B, 0). Each of the 4 halo rows lands as one plain
//                row segment (a 1-D bulk copy, pixel p at byte 8p), and the 32 bytes at 16j are pixels 2j .. 2j+3: one
//                K = 16 row of window j holding the taps of both its columns. A fragments are those overlapping rows
//                (16-byte row stride, so an 8-row ldmatrix phase reads 128 contiguous bytes: no bank conflicts, no
//                swizzle); the column parity dx is in the weights ([3 r][2 dx][CO][16], slot s + dx = tap s), so one
//                A fragment feeds both dx accumulators. Same MMAs as kPairS, a third of its A loads, a quarter of its
//                halo bytes.
// Warp roles as in G1: warps 0..7 compute + epilogue (windows 32 * (warp % 4) .., chunks by warp / 4),
// warp 8 is the TMA producer.
constexpr int kPairPlain = 0, kPairS = 1, kPairRS = 2, kPairC = 3;
// compact segment: one image row of <= 256 pixels x 8 B, plus zeroed slack for the 16 bytes window 127 reads past it
constexpr int kPairCSeg = 2048 + 128;
constexpr int kPairCBuf = 4;

template <int CK, int CO, int PK>
using PairCfgOf = PairFwdCfg<CK, CO, PK == kPairRS ? 2 : 4, PK == kPairC ? kPairCSeg : 136 * 2 * CK * 2,
                             PK == kPairC ? kPairCBuf : 2>;

template <int CK, int CO, int PK>
__device__ __forceinline__ void pair_fwd_body(const CUtensorMap* tmA, const CUtensorMap& tmW, const CUtensorMap& tmO,
                                              const CUtensorMap& tmC, const PairFwdArgs& a,
                                              const __nv_bfloat16* __restrict__ xc = nullptr) {
  using Cfg = PairCfgOf<CK, CO, PK>;
  constexpr bool SP = PK == kPairS;
  constexpr int RB = Cfg::ROW_BYTES;
  constexpr int WB = Cfg::W_ROW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem;
  uint8_t* sA = smem + Cfg::W_BYTES;
  uint8_t* sOut = sA + Cfg::NBUF * Cfg::HALO;           // [2][OUT_BYTES]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sOut + 2 * Cfg::OUT_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::NBUF;
  uint64_t* wfull = bars + 2 * Cfg::NBUF;
  float* sBias = reinterpret_cast<float*>(bars + 16);      // [CO], in the barrier block
  static_assert(16 * 8 + CO * 4 <= Cfg::BAR_BYTES, "bias slot");
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if constexpr (PK == kPairC) {
    // the slack past a row segment is never written by a copy but read by the windows past the pooled row's end
    for (int i = threadIdx.x; i < Cfg::NBUF * Cfg::HALO / 16; i += blockDim.x)
      reinterpret_cast<uint4*>(sA)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async();
  }
  if (warp == 8 && lane == 0) {
    if constexpr (PK != kPairC) prefetch_tmap(tmA);
    prefetch_tmap(&tmW);
    prefetch_tmap(&tmO);
    if (a.argmax) prefetch_tmap(&tmC);
    for (int s = 0; s < Cfg::NBUF; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  if (warp == 8 && elect_one()) {
    constexpr int NTAPW = PK == kPairRS ? 1 : (PK == kPairC ? 6 : (SP ? 3 : 9));
    mbar_expect_tx(wfull, NTAPW * Cfg::W_TAP);
    for (int tap = 0; tap < NTAPW; ++tap) tma_load_2d(sW + tap * Cfg::W_TAP, &tmW, 0, tap * CO, wfull);
  }
  pdl_wait();
  const int half_w = a.W >> 1;

  if (warp == 8) {
    // ===== TMA producer: 4 image rows of pair-rows per tile =====
    if (elect_one()) {
      int buf = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < a.num_tiles; t += gridDim.x) {
        const int b = t / a.Hp, hp = t - b * a.Hp;
        const int q0 = (b * a.H + 2 * hp) * half_w;          // first pair-row of image row 2hp
        mbar_wait(&empty[buf], phase ^ 1);
        uint8_t* dst = sA + buf * Cfg::HALO;
#ifdef HEFL_CONV_DEBUG
        if (a.dbg & 1) {
          mbar_arrive(&full[buf]);
        } else
#endif
        if constexpr (PK == kPairC) {
          const uint32_t row_bytes = (uint32_t)a.W * 8u;
          mbar_expect_tx(&full[buf], Cfg::NSEG * row_bytes);
          for (int sg = 0; sg < Cfg::NSEG; ++sg)
            bulk_load_1d(dst + sg * Cfg::SEG_BYTES, xc + (size_t)(q0 + sg * half_w) * 8, row_bytes, &full[buf]);
        } else {
          mbar_expect_tx(&full[buf], Cfg::HALO);
          for (int sg = 0; sg < Cfg::NSEG; ++sg) tma_load_2d(dst + sg * Cfg::SEG_BYTES, tmA, 0, q0 + sg * half_w, &full[buf]);
        }
        if (++buf == Cfg::NBUF) { buf = 0; phase ^= 1; }
      }
    }
  } else {
    // ===== compute + epilogue warps 0..7; accumulator (dy, dx) = acc[dy * 2 + dx] =====
    const int qd = warp & 3;
    const int grp = warp >> 2;
    const uint32_t w_base = smem_u32(sW);
    // the bias (written by the previous kernel, so read after pdl_wait) from shared memory: a per-chunk global
    // address would stay live across the MMAs
    if (threadIdx.x < CO) sBias[threadIdx.x] = a.bias[threadIdx.x];
    named_barrier_sync(1, 256);
    mbar_wait(wfull, 0);
    int buf = 0, ob = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < a.num_tiles; t += gridDim.x) {
      mbar_wait(&full[buf], phase);
      const uint32_t a_base = smem_u32(sA + buf * Cfg::HALO);
      const uint32_t sv = smem_u32(sOut + ob * Cfg::OUT_BYTES);   // [128 windows][CO] bf16, swizzle span CO * 2 B
      const uint32_t sc = sv + Cfg::OUT_V;                         // [128 windows][CO] codes, swizzle span CO B
#pragma unroll 1
      for (int g = 0; g < CO / 16 / Cfg::NG; ++g) {
        const int c0 = grp + 2 * g * Cfg::NG;              // chunks c0 and c0 + 2
        float acc[4][2][2][4];
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int q = 0; q < 4; ++q) acc[x][i][mt][q] = 0.f;
#ifdef HEFL_CONV_DEBUG
        if (!(a.dbg & 2))
#endif
        if constexpr (PK == kPairRS) {
          uint32_t bf[4];
          ld_b_kmajor<WB>(w_base, c0 * 8, (c0 + 2) * 8, 0, lane, bf);
#pragma unroll
          for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx)
#pragma unroll
              for (int mt = 0; mt < 2; ++mt) {
                uint32_t af[4];
                ld_a_kmajor<RB>(a_base + dy * Cfg::SEG_BYTES, qd * 32 + mt * 16, dx * CK * 2, lane, af);
                mma_bf16(acc[dy * 2 + dx][0][mt], af, bf[0], bf[1]);
                mma_bf16(acc[dy * 2 + dx][1][mt], af, bf[2], bf[3]);
              }
        } else if constexpr (PK == kPairC) {
          uint32_t bf[3][2][4];
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx)
              ld_b_kmajor<WB>(w_base + (r * 2 + dx) * Cfg::W_TAP, c0 * 8, (c0 + 2) * 8, 0, lane, bf[r][dx]);
          // halo row R = dy + r serves (dy, r) = (0, R) and (1, R - 1); every accumulator still sums r = 0, 1, 2 in order
#pragma unroll
          for (int R = 0; R < 4; ++R)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              uint32_t af[4];
              ldsm_x4(a_base + R * Cfg::SEG_BYTES + (uint32_t)((qd * 32 + mt * 16 + (lane & 15)) * 16 + ((lane >> 4) << 4)),
                      af);
#pragma unroll
              for (int dy = 0; dy < 2; ++dy) {
                const int r = R - dy;
                if (r < 0 || r > 2) continue;
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                  mma_bf16(acc[dy * 2 + dx][0][mt], af, bf[r][dx][0], bf[r][dx][1]);
                  mma_bf16(acc[dy * 2 + dx][1][mt], af, bf[r][dx][2], bf[r][dx][3]);
                }
              }
            }
        } else if constexpr (SP) {
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            uint32_t bf[4];
            ld_b_kmajor<WB>(w_base + r * Cfg::W_TAP, c0 * 8, (c0 + 2) * 8, 0, lane, bf);
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
              for (int dx = 0; dx < 2; ++dx)
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                  uint32_t af[4];
                  ld_a_kmajor<RB>(a_base + (dy + r) * Cfg::SEG_BYTES, qd * 32 + mt * 16, dx * CK * 2, lane, af);
                  mma_bf16(acc[dy * 2 + dx][0][mt], af, bf[0], bf[1]);
                  mma_bf16(acc[dy * 2 + dx][1][mt], af, bf[2], bf[3]);
                }
          }
        } else {
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap) {
            const int r = tap / 3, s = tap % 3;
#pragma unroll
            for (int k = 0; k < CK / 16; ++k) {
              uint32_t bf[4];
              ld_b_kmajor<WB>(w_base + tap * Cfg::W_TAP, c0 * 8, (c0 + 2) * 8, k * 32, lane, bf);
#pragma unroll
              for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                  const int e = dx + s;
#pragma unroll
                  for (int mt = 0; mt < 2; ++mt) {
                    uint32_t af[4];
                    ld_a_kmajor<RB>(a_base + (dy + r) * Cfg::SEG_BYTES, (e >> 1) + qd * 32 + mt * 16,
                                    (e & 1) * CK * 2 + k * 32, lane, af);
                    mma_bf16(acc[dy * 2 + dx][0][mt], af, bf[0], bf[1]);
                    mma_bf16(acc[dy * 2 + dx][1][mt], af, bf[2], bf[3]);
                  }
                }
            }
          }
        }
        if (g == CO / 16 / Cfg::NG - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[buf]);
        }
        // Pool on the fragments: the four accumulators of a window share one fragment layout (element q of m16 tile
        // mt is window qd*32 + mt*16 + (q >> 1)*8 + lane/4, channel ch*8 + (lane%4)*2 + (q & 1)), so the 2x2 max
        // and its arg-max are element-wise; only the pooled value (bf16 pair) and code (byte pair) reach the
        // staged output tile. The windows of a fragment row are 8k + lane / 4, and 8 rows span one swizzle repeat of
        // either tile, so the swizzle (address bits 7.. XORed into the 16-byte chunk bits 4..6) is a per-lane constant.
        const uint32_t vx = swz<CO * 2>((lane >> 2) * CO * 2) ^ ((lane >> 2) * CO * 2);
        const uint32_t cx = swz<CO>((lane >> 2) * CO) ^ ((lane >> 2) * CO);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int col = (c0 + 2 * i) * 8 + (lane & 3) * 2;   // this lane's first channel
#ifdef HEFL_CONV_DEBUG
          if (a.dbg & 4) continue;
#endif
          const float2 bb = *reinterpret_cast<const float2*>(sBias + col);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int win = qd * 32 + mt * 16 + hh * 8 + (lane >> 2);
              float x[2];
              uint32_t code = 0u;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int q = hh * 2 + e;
                const float a00 = acc[0][i][mt][q], a01 = acc[1][i][mt][q];
                const float a10 = acc[2][i][mt][q], a11 = acc[3][i][mt][q];
                // same tie-breaking as G1: lower row wins only if strictly greater, then right column likewise
                const bool l0 = a10 > a00;
                const bool l1 = a11 > a01;
                const float m0 = l0 ? a10 : a00;
                const float m1 = l1 ? a11 : a01;
                const bool rw = m1 > m0;
                const uint32_t rowbit = (rw ? l1 : l0) ? 1u : 0u;
                const float y = (rw ? m1 : m0) + (e ? bb.y : bb.x);
                // bits 0-1: arg-max position (row*2 + col) in the window, bit 2: unit active (ReLU mask)
                code |= ((rowbit << 1) | (rw ? 1u : 0u) | (y > 0.f ? 4u : 0u)) << (e * 8);
                x[e] = y > 0.f ? y : 0.f;
              }
              const uint32_t o = (uint32_t)(win * CO + col);
              sts_u32(sv + ((o * 2) ^ vx), pack_bf16x2(x[0], x[1]));
              sts_u16(sc + (o ^ cx), (uint16_t)code);        // staged always, stored only with an arg-max buffer
            }
        }
      }
      // The pooled row t = b * Hp + hp is rows t*Wp .. t*Wp + Wp-1 of the [B*Hp*Wp, CO] outputs: one TMA store
      // each, whose box of Wp rows leaves the staged windows past the row's end behind. Thread 0 issues the stores
      // after the eight warps' writes are visible to the async proxy; it first waits until the previous tile's
      // stores have read the other buffer, which the next tile fills, so one barrier per tile suffices.
      fence_proxy_async();
      if (threadIdx.x == 0) tma_wait_read<0>();
      named_barrier_sync(1, 256);
      if (threadIdx.x == 0
#ifdef HEFL_CONV_DEBUG
          && !(a.dbg & 4)
#endif
      ) {
        const uint8_t* tile = sOut + ob * Cfg::OUT_BYTES;
        tma_store_2d(&tmO, 0, t * a.Wp, tile);
        if (a.argmax) tma_store_2d(&tmC, 0, t * a.Wp, tile + Cfg::OUT_V);
        tma_commit();
      }
      ob ^= 1;
      if (++buf == Cfg::NBUF) { buf = 0; phase ^= 1; }
    }
    if (threadIdx.x == 0) tma_wait_all<0>();
  }
}

template <int CK, int CO, bool SP>
__global__ void __launch_bounds__(288, PairFwdCfg<CK, CO>::OCC)
pair_fwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmC, const PairFwdArgs a) {
  pair_fwd_body<CK, CO, SP ? kPairS : kPairPlain>(&tmA, tmW, tmO, tmC, a);
}

// the one-channel layer 1 on the rs-packed input (CK = 16, CO = 32)
__global__ void __launch_bounds__(288, PairCfgOf<16, 32, kPairRS>::OCC)
pair_fwd_rs_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                   const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmC,
                   const PairFwdArgs a) {
  pair_fwd_body<16, 32, kPairRS>(&tmA, tmW, tmO, tmC, a);
}

// the RGB layer 1 on the compact input (CK = 16, CO = 32): rows are bulk-copied from X, no input tensor map
__global__ void __launch_bounds__(288, PairCfgOf<16, 32, kPairC>::OCC)
pair_fwd_compact_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmO,
                        const __grid_constant__ CUtensorMap tmC, const PairFwdArgs a,
                        const __nv_bfloat16* __restrict__ X) {
  pair_fwd_body<16, 32, kPairC>(nullptr, tmW, tmO, tmC, a, X);
}

// Store maps of the pooled outputs, both viewed as [B*Hp*Wp rows][CO]: one box is one pooled row (Wp rows), with the
// swizzle the epilogue stages it in. Without arg-max codes the code map is left empty and never used.
static void make_pair_out_maps(const PairFwdArgs& a, int CO, CUtensorMap& tmO, CUtensorMap& tmC) {
  const uint64_t rows = (uint64_t)a.B * a.Hp * a.Wp;
  tmO = make_map(a.out, CO, rows, (uint64_t)CO * 2, CO, a.Wp);
  tmC = CUtensorMap{};
  if (a.argmax)
    tmC = tensor_map(a.argmax, CU_TENSOR_MAP_DATA_TYPE_UINT8, {(uint64_t)CO, rows}, {(uint64_t)CO},
                     {(uint32_t)CO, (uint32_t)a.Wp}, swizzle_for(CO));
}

template <int CK, int CO, int PK = kPairPlain>
static void launch_pair_fwd(const __nv_bfloat16* X, const __nv_bfloat16* Wt, PairFwdArgs a, cudaStream_t st) {
  using Cfg = PairCfgOf<CK, CO, PK>;
  const uint64_t pair_rows = ((uint64_t)a.B * a.H * a.W) / 2;
  const CUtensorMap tmA = make_map(X, 2 * CK, pair_rows, (uint64_t)Cfg::ROW_BYTES, 2 * CK, Cfg::SEG_ROWS);
  const int ntap = PK == kPairRS ? 1 : (PK == kPairS ? 3 : 9);
  const CUtensorMap tmW = make_map(Wt, CK, (uint64_t)ntap * CO, (uint64_t)CK * 2, CK, CO);
  CUtensorMap tmO, tmC;
  make_pair_out_maps(a, CO, tmO, tmC);
  void (*kern)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const PairFwdArgs);
  if constexpr (PK == kPairRS) kern = pair_fwd_rs_kernel;
  else kern = pair_fwd_kernel<CK, CO, PK == kPairS>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
  int gx = hefl::cuda::device_sm_count() * Cfg::OCC;
  if (gx > a.num_tiles) gx = a.num_tiles;
  launch_pdl(kern, dim3(gx), dim3(288), Cfg::SMEM, st, tmA, tmW, tmO, tmC, a);
  hefl::cuda::note_launch();
}

static void launch_pair_fwd_compact(const __nv_bfloat16* X, const __nv_bfloat16* Wt, PairFwdArgs a, cudaStream_t st) {
  using Cfg = PairCfgOf<16, 32, kPairC>;
  const CUtensorMap tmW = make_map(Wt, 16, 6 * 32, 32, 16, 32);
  CUtensorMap tmO, tmC;
  make_pair_out_maps(a, 32, tmO, tmC);
  cudaFuncSetAttribute(pair_fwd_compact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
  int gx = hefl::cuda::device_sm_count() * Cfg::OCC;
  if (gx > a.num_tiles) gx = a.num_tiles;
  launch_pdl(pair_fwd_compact_kernel, dim3(gx), dim3(288), Cfg::SMEM, st, tmW, tmO, tmC, a, X);
  hefl::cuda::note_launch();
}

bool conv_fwd_pool_pair_supported(int H, int W, int CK, int CO) {
  return H == W && (W % 2) == 0 && (W - 2) / 2 <= 128 && (CK == 16 || CK == 32) && (CO == 32 || CO == 64);
}

// Same contract as conv_fwd_pool (plain 9-tap weight layout [9][CO][CK], [3][CO][16] with the s-packed input,
// [1][CO][16] with the rs-packed one-channel input); see G1b above.
void conv_fwd_pool_pair(const void* X, const void* Wf, const float* bias, void* out, uint8_t* argmax, int B, int H,
                        int W, int CK, int CO, int spack, int in_channels, int compact, cudaStream_t st) {
  if (!conv_fwd_pool_pair_supported(H, W, CK, CO)) throw std::runtime_error("conv_fwd_pool_pair: unsupported shape");
  if (compact && !(CK == 16 && CO == 32 && in_channels == 3 && W <= 256))
    throw std::runtime_error("conv_fwd_pool_pair: the compact input is the RGB first layer (CK=16, CO=32, W <= 256)");
  PairFwdArgs a{};
#ifdef HEFL_CONV_DEBUG
  a.dbg = g_dbg;
#endif
  a.B = B; a.H = H; a.W = W;
  a.Hp = (H - 2) / 2; a.Wp = (W - 2) / 2;
  a.num_tiles = B * a.Hp;
  a.bias = bias;
  a.out = reinterpret_cast<__nv_bfloat16*>(out);
  a.argmax = argmax;
  const auto* x = reinterpret_cast<const __nv_bfloat16*>(X);
  const auto* w = reinterpret_cast<const __nv_bfloat16*>(Wf);
  if (spack && !(CK == 16 && CO == 32)) throw std::runtime_error("conv_fwd_pool_pair: s-packed input is CK=16, CO=32 only");
  if (spack && in_channels != 1 && in_channels != 3)
    throw std::runtime_error("conv_fwd_pool_pair: packed input has 1 or 3 channels");
  if (compact) launch_pair_fwd_compact(x, w, a, st);
  else if (CK == 16 && CO == 32 && spack && in_channels == 1) launch_pair_fwd<16, 32, kPairRS>(x, w, a, st);
  else if (CK == 16 && CO == 32 && spack) launch_pair_fwd<16, 32, kPairS>(x, w, a, st);
  else if (CK == 16 && CO == 32) launch_pair_fwd<16, 32>(x, w, a, st);
  else if (CK == 32 && CO == 32) launch_pair_fwd<32, 32>(x, w, a, st);
  else if (CK == 32 && CO == 64) launch_pair_fwd<32, 64>(x, w, a, st);
  else throw std::runtime_error("conv_fwd_pool_pair: unsupported (CK, CO)");
}

// ------------------------------------------------------------------------------------------
// G2: weight-gradient kernel.
//
// dW[r,s][ci][co] = sum_m X[m + r*W + s][ci] * dY[m][co]. Both operands are consumed in their
// native NHWC layout (ldmatrix.trans, pixels = K), so no transposed copies exist.
// Work is organised by image rows: a CTA walks down a 64-column strip; at row h it needs the X
// row segments h, h+1, h+2 (72 pixels each) and the dY chunk of row h. Segments live in a ring
// of stages, so each X segment is fetched ONCE and serves filter rows r = 2, 1, 0 on three
// consecutive steps; the tap column s is a row offset of the MMA descriptor (LBO = one pixel).
// 3-D tensor maps (C, W, B*H) keep chunks inside an image row (out-of-range columns zero-fill).
// Split over (image, strip, row range); fp32 vector-RED of the partial sums into a [9*C+1, Co]
// buffer whose last row is the bias gradient (an all-ones A tile).
// ------------------------------------------------------------------------------------------
struct WgradArgs {
  int H, W, Ho;     // input grid height/width, valid output rows
  int strips;       // ceil((W-2) / 64)
  int rsplit;       // row ranges per (image, strip)
  int rows_per;     // rows per range
  int units;        // B * strips * rsplit
  int nchunks;      // FLAT: ceil(B*H*W / 64)
  int Co;           // total output channels (row pitch of a partial)
  float* ws;        // [gridDim.x][9*CK + 1][Co] fp32: the partial sums of CTA column x (plain stores)
};

// FLAT = small feature maps (W <= 32): a 64-pixel chunk of one image row would be mostly padding, so
// chunks are 64 consecutive pixels of the flattened [B*H*W] axis and each stage carries its own
// three X segments (rows offset by W); no ring reuse, L2 traffic is irrelevant at these sizes.
template <int CK, int COT, bool FLAT = false>
struct WgradCfg {
  // CK = 16 (layer 1): the X tensor map uses OVERLAPPING rows: row m is the 128 bytes starting at pixel m
  // (4 pixels x 16 channels, row stride 32 B), so one 128-byte row already holds the tap columns s = 0..3 and
  // no pixel shift is needed.
  static constexpr bool PACK4 = CK == 16;
  static constexpr int ATOM_A = PACK4 ? 128 : CK * 2;          // bytes of one pixel row of the X tile
  static constexpr int ATOM_B = COT * 2;
  static constexpr int XROWS = PACK4 ? 64 : 72;                // 64 + pixel shifts (none when packed)
  static constexpr int X_BYTES = XROWS * ATOM_A;
  static constexpr int X_SEG = ((X_BYTES + 1023) / 1024) * 1024;
  static constexpr int DY_BYTES = 64 * ATOM_B;
  static constexpr int DY_OFF = FLAT ? 3 * X_SEG : X_SEG;
  static constexpr int TX = (FLAT ? 3 : 1) * X_BYTES + DY_BYTES;
  static constexpr int STAGE_FULL = DY_OFF + ((DY_BYTES + 1023) / 1024) * 1024;
  static_assert(!(FLAT && PACK4), "layer 1 always uses the rolling-window path");
  // deep ring: stages are small (one X row segment + one dY chunk), so the number of bytes in
  // flight, not the MMA rate, bounds throughput
  static constexpr int NSTAGE_RAW = (200 * 1024) / STAGE_FULL;
  static constexpr int NSTAGE = NSTAGE_RAW > 6 ? 6 : NSTAGE_RAW;
  static constexpr int SMEM = NSTAGE * STAGE_FULL + 512 + 1024;
  static_assert(NSTAGE >= 4, "ring needs 3 live stages + 1 in flight");
  // m16 tiles of one filter row: (tap column s, 16 input channels); warp w owns tiles w and w + 8
  static constexpr int MT = 3 * CK / 16;
  static constexpr int NT = COT / 8;
  static constexpr int OCC = blocks_fit(SMEM, 2) ? 2 : 1;
  static_assert(CK == 16 || CK == 32 || CK == 64, "CK must be one swizzle atom");
  static_assert(COT == 32 || COT == 64, "COT must be one swizzle atom");
};

// dW[r,s][ci][co] = sum_p X[p + s][ci] dY[p][co] for the filter row r = blockIdx.z over the pixels of CTA column
// blockIdx.x, stored into that column's partial (reduce_partials adds the columns in a fixed order, so the gradient
// is the same bits on every run): a CTA holds 3*CK x COT fp32 accumulators in the registers of its 8 compute warps (mma.sync m16n8k16, both operands read from their native
// [pixel][channel] tiles with ldmatrix.trans: pixels are the K axis), warp 8 is the TMA producer. The bias
// gradient (column sums of dY) is one more MMA per k-step with an all-ones A fragment, in the r = 0 CTAs.
template <int CK, int COT, bool FLAT>
__global__ void __launch_bounds__(288, WgradCfg<CK, COT, FLAT>::OCC)
wgrad_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmDY,
             const WgradArgs a) {
  using Cfg = WgradCfg<CK, COT, FLAT>;
  constexpr int SA = Cfg::ATOM_A, SB = Cfg::ATOM_B;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::NSTAGE * Cfg::STAGE_FULL);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::NSTAGE;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int co0 = blockIdx.y * COT;
  const int fr = blockIdx.z;                                    // filter row r

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmDY);
    for (int s = 0; s < Cfg::NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_prologue();
  const int per_img = a.strips * a.rsplit;

  if (warp == 8) {
    if (FLAT) {
      if (elect_one()) {
        int slot = 0;
        uint32_t phase = 0;
        for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
          mbar_wait(&empty[slot], phase ^ 1u);
          uint8_t* st = smem + slot * Cfg::STAGE_FULL;
          mbar_expect_tx(&full[slot], Cfg::TX);
          for (int r = 0; r < 3; ++r) tma_load_2d(st + r * Cfg::X_SEG, &tmX, 0, c * 64 + r * a.W, &full[slot]);
          tma_load_2d(st + Cfg::DY_OFF, &tmDY, co0, c * 64, &full[slot]);
          if (++slot == Cfg::NSTAGE) { slot = 0; phase ^= 1; }
        }
      }
    } else if (elect_one()) {
      int slot = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
        const int b = u / per_img;
        const int rem = u - b * per_img;
        const int strip = rem / a.rsplit;
        const int h0 = (rem - strip * a.rsplit) * a.rows_per;
        const int h1 = min(a.Ho, h0 + a.rows_per);
        if (h0 >= h1) continue;
        for (int i = h0 - 2; i < h1; ++i) {
          mbar_wait(&empty[slot], phase ^ 1u);
          uint8_t* st = smem + slot * Cfg::STAGE_FULL;
          mbar_expect_tx(&full[slot], Cfg::X_BYTES + (i >= h0 ? Cfg::DY_BYTES : 0));
          tma_load_3d(st, &tmX, 0, strip * 64, b * a.H + i + 2, &full[slot]);   // PACK4: 128-byte windows
          if (i >= h0) tma_load_3d(st + Cfg::DY_OFF, &tmDY, co0, strip * 64, b * a.H + i, &full[slot]);
          if (++slot == Cfg::NSTAGE) { slot = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== compute warps 0..7
  float acc[2][Cfg::NT][4];
  float bacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int n = 0; n < Cfg::NT; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[u][n][q] = 0.f;
  constexpr uint32_t kOnes = 0x3F803F80u;                       // bf16 1.0 x2
  const uint32_t ones[4] = {kOnes, kOnes, kOnes, kOnes};
  const int bias_nt = warp % Cfg::NT;
  // per-lane parts of the ldmatrix.trans addresses: matrix i = lane / 8 covers (M or N block i & 1 or i >> 1)
  const int lrow = lane & 7;
  const int ia = lane >> 3;
  uint32_t a_off[2];                                            // byte offset of my A rows for tiles w, w + 8
  int a_shift[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int tile = warp + 8 * u;
    const int s = tile / (CK / 16), ci0 = (tile % (CK / 16)) * 16;
    a_shift[u] = Cfg::PACK4 ? 0 : s;
    a_off[u] = (uint32_t)((Cfg::PACK4 ? s * CK + ci0 : ci0) * 2 + (ia & 1) * 16);
  }
  const uint32_t smem0 = smem_u32(smem);

  auto step = [&](uint32_t x_tile, uint32_t dy_tile) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {                            // 4 x 16 pixels per 64-pixel chunk
      uint32_t bf[Cfg::NT / 2][4];
#pragma unroll
      for (int n = 0; n < Cfg::NT; n += 2)
        ldsm_x4_t(swz<SB>(dy_tile + (uint32_t)((kk * 16 + (ia & 1) * 8 + lrow) * SB + (n + (ia >> 1)) * 16)), bf[n / 2]);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (warp + 8 * u >= Cfg::MT) break;
        uint32_t af[4];
        ldsm_x4_t(swz<SA>(x_tile + (uint32_t)((kk * 16 + (ia >> 1) * 8 + lrow + a_shift[u]) * SA) + a_off[u]), af);
#pragma unroll
        for (int n = 0; n < Cfg::NT; ++n) mma_bf16(acc[u][n], af, bf[n / 2][(n & 1) * 2], bf[n / 2][(n & 1) * 2 + 1]);
      }
      if (fr == 0) {
#pragma unroll
        for (int n = 0; n < Cfg::NT; ++n)
          if (n == bias_nt) mma_bf16(bacc, ones, bf[n / 2][(n & 1) * 2], bf[n / 2][(n & 1) * 2 + 1]);
      }
    }
  };

  int slot = 0;
  uint32_t phase = 0;
  if (FLAT) {
    for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
      mbar_wait(&full[slot], phase);
      const uint32_t st = smem0 + slot * Cfg::STAGE_FULL;
      step(st + fr * Cfg::X_SEG, st + Cfg::DY_OFF);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);
      if (++slot == Cfg::NSTAGE) { slot = 0; phase ^= 1; }
    }
  } else {
    for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
      const int rem = u % per_img;
      const int strip = rem / a.rsplit;
      const int h0 = (rem - strip * a.rsplit) * a.rows_per;
      const int h1 = min(a.Ho, h0 + a.rows_per);
      if (h0 >= h1) continue;
      for (int i = h0 - 2; i < h1; ++i) {
        mbar_wait(&full[slot], phase);
        const int s1 = slot == 0 ? Cfg::NSTAGE - 1 : slot - 1;       // stage of X row h+1
        const int s0 = s1 == 0 ? Cfg::NSTAGE - 1 : s1 - 1;           // stage of X row h
        if (i >= h0) {
          const int sx = fr == 0 ? s0 : (fr == 1 ? s1 : slot);
          step(smem0 + sx * Cfg::STAGE_FULL, smem0 + slot * Cfg::STAGE_FULL + Cfg::DY_OFF);
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[s0]);                    // stage of X row h is done
        }
        if (++slot == Cfg::NSTAGE) { slot = 0; phase ^= 1; }
      }
      __syncwarp();
      if (lane == 0) {                                               // release the last two stages of the unit
        const int l1 = slot == 0 ? Cfg::NSTAGE - 1 : slot - 1;
        const int l0 = l1 == 0 ? Cfg::NSTAGE - 1 : l1 - 1;
        mbar_arrive(&empty[l0]);
        mbar_arrive(&empty[l1]);
      }
    }
  }
  // every CTA writes its whole share of the partial (zeros when it had no work), so the partial is fully defined
  float* part = a.ws + (size_t)blockIdx.x * (9 * CK + 1) * a.Co;
  // fragment element q of (m16 tile, n8 tile): row ci0 + lane/4 (+8 for q >= 2), column 2*(lane%4) + (q & 1)
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int tile = warp + 8 * u;
    if (tile >= Cfg::MT) break;
    const int s = tile / (CK / 16), ci0 = (tile % (CK / 16)) * 16;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int R = (fr * 3 + s) * CK + ci0 + (lane >> 2) + 8 * h;   // dW32 row: (r*3+s)*CK + ci
      float* dst = part + (size_t)R * a.Co + co0 + 2 * (lane & 3);
#pragma unroll
      for (int n = 0; n < Cfg::NT; ++n)
        *reinterpret_cast<float2*>(dst + n * 8) = make_float2(acc[u][n][2 * h], acc[u][n][2 * h + 1]);
    }
  }
  if (fr == 0 && warp < Cfg::NT && lane < 4)                        // bias: row 0 of the all-ones product
    *reinterpret_cast<float2*>(part + (size_t)(9 * CK) * a.Co + co0 + bias_nt * 8 + 2 * lane) =
        make_float2(bacc[0], bacc[1]);
}

// 3-D bf16 tensor [rows][W][C] (C contiguous) with pixels `pixel_bytes` apart (below C * 2 they overlap, which TMA
// allows); box = {box_c, box_w, 1}.
static CUtensorMap make_map_3d(const void* ptr, uint64_t C, uint64_t W, uint64_t rows, uint64_t pixel_bytes,
                               uint32_t box_c, uint32_t box_w) {
  return tensor_map(ptr, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, {C, W, rows}, {pixel_bytes, W * pixel_bytes},
                    {box_c, box_w, 1}, swizzle_for(box_c * 2));
}

template <int CK, int COT, bool FLAT>
struct WgradKind {
  static constexpr int kCK = CK, kCOT = COT;
  static constexpr bool kFLAT = FLAT;
};

// Calls f(WgradKind<...>{}) for the kernel configuration that serves (W, CK, Co).
template <class F>
static auto wgrad_dispatch(int W, int CK, int Co, F&& f) {
  const bool flat = W <= 32 && CK != 16;
  if (CK == 16 && Co == 32) return f(WgradKind<16, 32, false>{});
  if (CK == 32 && Co == 32) return flat ? f(WgradKind<32, 32, true>{}) : f(WgradKind<32, 32, false>{});
  if (CK == 32 && Co == 64) return flat ? f(WgradKind<32, 64, true>{}) : f(WgradKind<32, 64, false>{});
  if (CK == 64 && (Co == 64 || Co == 128)) return flat ? f(WgradKind<64, 64, true>{}) : f(WgradKind<64, 64, false>{});
  throw std::runtime_error("conv_wgrad: unsupported (CK, Co)");
}

// Work split of one weight-gradient launch; returns the number of CTA columns (= partials).
template <int CK, int COT, bool FLAT>
static int wgrad_plan(int B, int H, int W, int Co, WgradArgs& a) {
  using Cfg = WgradCfg<CK, COT, FLAT>;
  a = WgradArgs{};
  a.H = H; a.W = W; a.Ho = H - 2;
  a.strips = (W - 2 + 63) / 64;
  const int cot = Co / COT;
  // units of <= 16 image rows, dealt round-robin: load imbalance <= one unit, ring warm-up 2/16
  a.rows_per = a.Ho < 16 ? a.Ho : 16;
  a.rsplit = (a.Ho + a.rows_per - 1) / a.rows_per;
  a.units = B * a.strips * a.rsplit;
  a.nchunks = (B * H * W + 63) / 64;
  a.Co = Co;
  const int total_steps = FLAT ? a.nchunks : a.units * (a.rows_per + 2);
  // every CTA pays a fixed epilogue (a store of all accumulators): give each at least a few steps
  int gx = total_steps / (FLAT ? 6 : 24);
  const int slots = hefl::cuda::device_sm_count() * Cfg::OCC / (3 * cot);
  if (gx > slots) gx = slots;
  if (gx > (FLAT ? a.nchunks : a.units)) gx = FLAT ? a.nchunks : a.units;
  if (gx < 1) gx = 1;
  return gx;
}

// dst[i] += the sum of the partials ws[p * n + i] over p, in a fixed order (sum_partials).
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ ws, int parts, int64_t n,
                                                              float* __restrict__ dst) {
  __shared__ float red[256];
  const float s = sum_partials(ws, parts, n, red);
  const int64_t i = (int64_t)blockIdx.x * 32 + threadIdx.x;
  if (threadIdx.x < 32 && i < n) dst[i] += s;
}

void reduce_partials(const float* ws, int parts, int64_t n, float* dst, cudaStream_t st) {
  reduce_partials_kernel<<<(unsigned)((n + 31) / 32), 256, 0, st>>>(ws, parts, n, dst);
  hefl::cuda::note_launch();
}

int64_t conv_wgrad_ws_floats(int B, int H, int W, int CK, int Co) {
  return wgrad_dispatch(W, CK, Co, [&](auto k) -> int64_t {
    using K = decltype(k);
    WgradArgs a;
    return (int64_t)wgrad_plan<K::kCK, K::kCOT, K::kFLAT>(B, H, W, Co, a) * (9 * CK + 1) * Co;
  });
}

void conv_wgrad(const void* X, const void* DY, float* dW32, float* ws, int B, int H, int W, int CK, int Co,
                cudaStream_t st) {
  wgrad_dispatch(W, CK, Co, [&](auto k) {
    using K = decltype(k);
    constexpr int CKc = K::kCK, COT = K::kCOT;
    constexpr bool FLAT = K::kFLAT;
    using Cfg = WgradCfg<CKc, COT, FLAT>;
    const auto* x = reinterpret_cast<const __nv_bfloat16*>(X);
    const auto* d = reinterpret_cast<const __nv_bfloat16*>(DY);
    WgradArgs a;
    const int gx = wgrad_plan<CKc, COT, FLAT>(B, H, W, Co, a);
    a.ws = ws;
    const int P = B * H * W;
    CUtensorMap tmX, tmD;
    if (FLAT) {
      tmX = make_map(x, CKc, (uint64_t)P, (uint64_t)CKc * 2, CKc, Cfg::XROWS);
      tmD = make_map(d, Co, (uint64_t)P, (uint64_t)Co * 2, COT, 64);
    } else {
      tmX = Cfg::PACK4 ? make_map_3d(x, 64, W, (uint64_t)B * H, 32, 64, Cfg::XROWS)
                       : make_map_3d(x, CKc, W, (uint64_t)B * H, CKc * 2, CKc, Cfg::XROWS);
      tmD = make_map_3d(d, Co, W, (uint64_t)B * H, (uint64_t)Co * 2, COT, 64);
    }
    auto kern = wgrad_kernel<CKc, COT, FLAT>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    dim3 grid(gx, Co / COT, 3);                              // z = filter row
    launch_pdl(kern, grid, dim3(288), Cfg::SMEM, st, tmX, tmD, a);
    hefl::cuda::note_launch();
    // a plain launch: starts only when every partial is written
    reduce_partials(ws, gx, (int64_t)(9 * CKc + 1) * Co, dW32, st);
  });
}

// ------------------------------------------------------------------------------------------
// G3: fused data + weight gradient of a CK = Co = 32 layer on a wide map (layer 2 of the medical CNN).
//
// The weight gradient keeps wgrad_kernel<32, 32, false>'s work exactly: the same CTA columns (wgrad_plan), units,
// filter row per blockIdx.z, ring of (X row i + 2, dY row i) stages and MMA sequence per accumulator, on the same
// operand values. Every CTA partial, and so dW32 after reduce_partials, is the same bits as conv_wgrad's.
// The data gradient rides on that ring. The dY box is 72 columns starting 2 before the strip (the weight gradient reads
// its columns 2 .. 65) and dY is loaded for every step of a unit, also for its two leading steps, so at step i the
// ring holds dY rows i, i - 1, i - 2: all that image row i of the strip needs for
//   dX[m, :] = sum_{r,s} dY[m - r*W - s, :] * Wd[r,s]      (conv_dgrad's flat formula)
// Columns and rows that flat indexing would take from a neighbouring row or image are the zero border of dY, which the
// 3-D boxes read as zeros, so every MMA operand is the value tap_gemm_kernel<32, 32, false, 3> reads, in its tap,
// k-step order: gX is the same bits as conv_dgrad's. Row i of the strip is computed by the CTA with z = i % 3 (one third
// of the rows each), and the unit that ends at the last valid row also steps over the two border rows below it for
// their data gradient only. The map needs strips * 64 >= W (conv_dgrad_wgrad_supported).
//
// Warps as wgrad_kernel: 0..7 compute, 8 the TMA producer. For a data-gradient row, warp w owns pixels 16 * (w % 4) ..
// +15 of the strip and output channels 16 * (w / 4) .. +15. The 18 fragment loads and MMA pairs of a row are software-
// pipelined (step j + 1's fragments are loaded before step j's MMAs).
// ------------------------------------------------------------------------------------------
struct DgradWgradCfg {
  using WG = WgradCfg<32, 32, false>;
  static constexpr int C = 32;
  static constexpr int RB = C * 2;                        // bytes per pixel (64-byte swizzle)
  static constexpr int X_SEG = WG::X_SEG;                 // X row segment: 72 pixels from the strip start
  static constexpr int DY_COLS = 72;                      // dY row segment: 72 pixels from 2 before the strip start
  static constexpr int DY_BYTES = DY_COLS * RB;
  static constexpr int STAGE = X_SEG + ((DY_BYTES + 1023) / 1024) * 1024;
  static constexpr int TX = WG::X_BYTES + DY_BYTES;
  static constexpr int NSTAGE = WG::NSTAGE;
  static constexpr int W_TAP = C * RB;
  static constexpr int W_BYTES = 9 * W_TAP;
  static constexpr int SCR_BYTES = 8 * 1024;              // 1 KB accumulator staging per compute warp
  static constexpr int SMEM = NSTAGE * STAGE + W_BYTES + SCR_BYTES + 512 + 1024;
  static constexpr int PART = (9 * C + 1) * C;            // floats of one CTA column's partial
  static_assert(blocks_fit(SMEM, 2), "two CTAs per SM, as wgrad_kernel");
  static_assert(NSTAGE >= 4, "ring needs 3 live stages + 1 in flight");
};

struct DgradWgradArgs {
  WgradArgs w;          // wgrad_plan's split; w.ws = [gridDim.x][9*32 + 1][32]
#ifdef HEFL_CONV_DEBUG
  int dbg;              // 1 = skip TMA data, 2 = skip MMAs, 4 = skip the gX store, 8 = skip the weight-gradient MMAs
#endif
  __nv_bfloat16* dx;    // [B*H*W][32]
};

__global__ void __launch_bounds__(288, 2)
dgrad_wgrad_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmDY,
                   const __grid_constant__ CUtensorMap tmW, const DgradWgradArgs args) {
  using Cfg = DgradWgradCfg;
  constexpr int CK = 32, SA = Cfg::RB, SB = Cfg::RB, NT = 4, MT = 6;
  const WgradArgs& a = args.w;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem + Cfg::NSTAGE * Cfg::STAGE;
  float* scr_all = reinterpret_cast<float*>(sW + Cfg::W_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(scr_all) + Cfg::SCR_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::NSTAGE;
  uint64_t* wfull = bars + 2 * Cfg::NSTAGE;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int fr = blockIdx.z;                                    // filter row r of the weight gradient
  bool do_mma = true, do_wgrad = true, do_store = true;
#ifdef HEFL_CONV_DEBUG
  do_mma = !(args.dbg & 2);
  do_store = !(args.dbg & 4);
  do_wgrad = !(args.dbg & 8);
#endif

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmDY);
    prefetch_tmap(&tmW);
    for (int s = 0; s < Cfg::NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // PDL as tap_gemm_kernel: the weight tile before the wait, activations after it
  pdl_trigger();
  if (warp == 8 && elect_one()) {
    mbar_expect_tx(wfull, Cfg::W_BYTES);
    for (int tap = 0; tap < 9; ++tap) tma_load_2d(sW + tap * Cfg::W_TAP, &tmW, 0, tap * CK, wfull);
  }
  pdl_wait();
  const int per_img = a.strips * a.rsplit;

  if (warp == 8) {
    if (elect_one()) {
      int slot = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
        const int b = u / per_img;
        const int rem = u - b * per_img;
        const int strip = rem / a.rsplit;
        const int h0 = (rem - strip * a.rsplit) * a.rows_per;
        const int h1 = min(a.Ho, h0 + a.rows_per);
        if (h0 >= h1) continue;
        const int h_end = h1 == a.Ho ? a.H : h1;               // + the border rows' data gradient
        for (int i = h0 - 2; i < h_end; ++i) {
          mbar_wait(&empty[slot], phase ^ 1u);
          uint8_t* st = smem + slot * Cfg::STAGE;
#ifdef HEFL_CONV_DEBUG
          if (args.dbg & 1) {
            mbar_arrive(&full[slot]);
          } else
#endif
          {
            mbar_expect_tx(&full[slot], Cfg::TX);
            tma_load_3d(st, &tmX, 0, strip * 64, b * a.H + i + 2, &full[slot]);
            tma_load_3d(st + Cfg::X_SEG, &tmDY, 0, strip * 64 - 2, b * a.H + i, &full[slot]);
          }
          if (++slot == Cfg::NSTAGE) { slot = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== compute warps 0..7: the weight gradient exactly as wgrad_kernel<32, 32, false>
  float acc[2][NT][4];
  float bacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[u][n][q] = 0.f;
  constexpr uint32_t kOnes = 0x3F803F80u;                       // bf16 1.0 x2
  const uint32_t ones[4] = {kOnes, kOnes, kOnes, kOnes};
  const int bias_nt = warp % NT;
  const int lrow = lane & 7;
  const int ia = lane >> 3;
  uint32_t a_off[2];
  int a_shift[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int tile = warp + 8 * u;
    const int s = tile / (CK / 16), ci0 = (tile % (CK / 16)) * 16;
    a_shift[u] = s;
    a_off[u] = (uint32_t)(ci0 * 2 + (ia & 1) * 16);
  }
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t w_base = smem_u32(sW);
  float* scr = scr_all + warp * 256;
  const int qd = warp & 3, grp = warp >> 2;                    // data gradient: pixels 16 qd .., channels 16 grp ..

  auto wstep = [&](uint32_t x_tile, uint32_t dy_tile) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t bf[NT / 2][4];
#pragma unroll
      for (int n = 0; n < NT; n += 2)
        ldsm_x4_t(swz<SB>(dy_tile + (uint32_t)((kk * 16 + (ia & 1) * 8 + lrow) * SB + (n + (ia >> 1)) * 16)), bf[n / 2]);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (warp + 8 * u >= MT) break;
        uint32_t af[4];
        ldsm_x4_t(swz<SA>(x_tile + (uint32_t)((kk * 16 + (ia >> 1) * 8 + lrow + a_shift[u]) * SA) + a_off[u]), af);
#pragma unroll
        for (int n = 0; n < NT; ++n) mma_bf16(acc[u][n], af, bf[n / 2][(n & 1) * 2], bf[n / 2][(n & 1) * 2 + 1]);
      }
      if (fr == 0) {
#pragma unroll
        for (int n = 0; n < NT; ++n)
          if (n == bias_nt) mma_bf16(bacc, ones, bf[n / 2][(n & 1) * 2], bf[n / 2][(n & 1) * 2 + 1]);
      }
    }
  };

  // data gradient of image row h (= b*H + h of the [B*H] row axis) of the strip; dyr[r] = dY stage of row h - r
  auto drow = [&](const uint32_t (&dyr)[3], int row, int strip) {
    float d[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int q = 0; q < 4; ++q) d[i][q] = 0.f;
    if (do_mma) {
      // step j = (tap j / 2, k-step j % 2), tap_gemm_kernel's order; dY column c - s is row 2 - s + c of a segment
      auto load = [&](int j, uint32_t(&bf)[4], uint32_t(&af)[4]) {
        const int tap = j >> 1, ks = j & 1, r = tap / 3, s = tap % 3;
        ld_b_kmajor<Cfg::RB>(w_base + tap * Cfg::W_TAP, grp * 16, grp * 16 + 8, ks * 32, lane, bf);
        ld_a_kmajor<Cfg::RB>(dyr[r], (2 - s) + qd * 16, ks * 32, lane, af);
      };
      uint32_t bf[2][4], af[2][4];
      load(0, bf[0], af[0]);
#pragma unroll
      for (int j = 0; j < 18; ++j) {
        const int c = j & 1;
        if (j + 1 < 18) load(j + 1, bf[c ^ 1], af[c ^ 1]);
        mma_bf16(d[0], af[c], bf[c][0], bf[c][1]);
        mma_bf16(d[1], af[c], bf[c][2], bf[c][3]);
      }
    }
    // lane L: pixel 16 qd + L % 16 of the strip, channels 16 grp + 8 (L / 16) .. +7
    float v[8];
    frag_rows(scr, d[0], d[1], lane, v);
    const int w = strip * 64 + qd * 16 + (lane & 15);
    if (do_store && w < a.W)
      *reinterpret_cast<uint4*>(args.dx + ((size_t)row * a.W + w) * CK + grp * 16 + (lane >> 4) * 8) =
          make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                     pack_bf16x2(v[6], v[7]));
  };

  mbar_wait(wfull, 0);
  int slot = 0;
  uint32_t phase = 0;
  for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
    const int b = u / per_img;
    const int rem = u - b * per_img;
    const int strip = rem / a.rsplit;
    const int h0 = (rem - strip * a.rsplit) * a.rows_per;
    const int h1 = min(a.Ho, h0 + a.rows_per);
    if (h0 >= h1) continue;
    const int h_end = h1 == a.Ho ? a.H : h1;
    for (int i = h0 - 2; i < h_end; ++i) {
      mbar_wait(&full[slot], phase);
      const int s1 = slot == 0 ? Cfg::NSTAGE - 1 : slot - 1;       // stage of X row h+1, dY row h-1
      const int s0 = s1 == 0 ? Cfg::NSTAGE - 1 : s1 - 1;           // stage of X row h, dY row h-2
      if (i >= h0) {
        if (i < h1 && do_mma && do_wgrad) {
          const int sx = fr == 0 ? s0 : (fr == 1 ? s1 : slot);
          wstep(smem0 + sx * Cfg::STAGE, smem0 + slot * Cfg::STAGE + Cfg::X_SEG + 2 * SB);
        }
        if (i % 3 == fr) {
          const uint32_t dyr[3] = {smem0 + slot * Cfg::STAGE + Cfg::X_SEG, smem0 + s1 * Cfg::STAGE + Cfg::X_SEG,
                                   smem0 + s0 * Cfg::STAGE + Cfg::X_SEG};
          drow(dyr, b * a.H + i, strip);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s0]);                    // stage of X row h / dY row h-2 is done
      }
      if (++slot == Cfg::NSTAGE) { slot = 0; phase ^= 1; }
    }
    __syncwarp();
    if (lane == 0) {                                               // release the last two stages of the unit
      const int l1 = slot == 0 ? Cfg::NSTAGE - 1 : slot - 1;
      const int l0 = l1 == 0 ? Cfg::NSTAGE - 1 : l1 - 1;
      mbar_arrive(&empty[l0]);
      mbar_arrive(&empty[l1]);
    }
  }
  // wgrad_kernel's partial store: every CTA writes its whole share (zeros when it had no work)
  float* part = a.ws + (size_t)blockIdx.x * (9 * CK + 1) * a.Co;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int tile = warp + 8 * u;
    if (tile >= MT) break;
    const int s = tile / (CK / 16), ci0 = (tile % (CK / 16)) * 16;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int R = (fr * 3 + s) * CK + ci0 + (lane >> 2) + 8 * h;   // dW32 row: (r*3+s)*CK + ci
      float* dst = part + (size_t)R * a.Co + 2 * (lane & 3);
#pragma unroll
      for (int n = 0; n < NT; ++n)
        *reinterpret_cast<float2*>(dst + n * 8) = make_float2(acc[u][n][2 * h], acc[u][n][2 * h + 1]);
    }
  }
  if (fr == 0 && warp < NT && lane < 4)                              // bias: row 0 of the all-ones product
    *reinterpret_cast<float2*>(part + (size_t)(9 * CK) * a.Co + bias_nt * 8 + 2 * lane) = make_float2(bacc[0], bacc[1]);
}

bool conv_dgrad_wgrad_supported(int H, int W, int CK, int Co) {
  return CK == 32 && Co == 32 && H >= 3 && W >= 3 && (W - 2 + 63) / 64 * 64 >= W;
}

int64_t conv_dgrad_wgrad_ws_floats(int B, int H, int W) {
  WgradArgs a;
  return (int64_t)wgrad_plan<32, 32, false>(B, H, W, 32, a) * DgradWgradCfg::PART;
}

void conv_dgrad_wgrad(const void* X, const void* dY, const void* Wd, void* dX, float* dW32, float* ws, int B, int H,
                      int W, int CK, int Co, cudaStream_t st) {
  using Cfg = DgradWgradCfg;
  if (!conv_dgrad_wgrad_supported(H, W, CK, Co))
    throw std::runtime_error("conv_dgrad_wgrad: CK = Co = 32 and a map the 64-column strips cover");
  DgradWgradArgs a{};
#ifdef HEFL_CONV_DEBUG
  a.dbg = g_dbg;
#endif
  const int gx = wgrad_plan<32, 32, false>(B, H, W, Co, a.w);
  a.w.ws = ws;
  a.dx = reinterpret_cast<__nv_bfloat16*>(dX);
  const auto* x = reinterpret_cast<const __nv_bfloat16*>(X);
  const auto* d = reinterpret_cast<const __nv_bfloat16*>(dY);
  const CUtensorMap tmX = make_map_3d(x, Cfg::C, W, (uint64_t)B * H, Cfg::RB, Cfg::C, Cfg::WG::XROWS);
  const CUtensorMap tmD = make_map_3d(d, Cfg::C, W, (uint64_t)B * H, Cfg::RB, Cfg::C, Cfg::DY_COLS);
  const CUtensorMap tmW = make_map(Wd, Cfg::C, 9 * Cfg::C, Cfg::RB, Cfg::C, Cfg::C);
  cudaFuncSetAttribute(dgrad_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
  launch_pdl(dgrad_wgrad_kernel, dim3(gx, 1, 3), dim3(288), Cfg::SMEM, st, tmX, tmD, tmW, a);
  hefl::cuda::note_launch();
  // a plain launch: starts only when every partial is written
  reduce_partials(ws, gx, Cfg::PART, dW32, st);
}

}  // namespace nn
}  // namespace hefl

// ------------------------------------------------------------------------------------------
// Probe: can a K-major swizzled A tile be consumed starting at an arbitrary ROW offset? out[128, 32] =
// A[shift_rows .. shift_rows + 127, :] . B^T, read from one TMA tile. Used to validate halo-tile reuse.
// ------------------------------------------------------------------------------------------
namespace hefl {
namespace nn {
using namespace hefl::sm90;
using namespace hefl::tc;

template <int CK>
__global__ void __launch_bounds__(128, 1)
umma_shift_probe_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        float* out, int shift_rows) {
  constexpr int RB = CK * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                      // 144 rows
  uint8_t* sB = smem + 144 * 128;          // 32 rows
  uint64_t* bar = reinterpret_cast<uint64_t*>(sB + 32 * 128);
  float* scr = reinterpret_cast<float*>(bar + 2);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
    mbar_expect_tx(bar, 144 * RB + 32 * RB);
    tma_load_2d(sA, &tmA, 0, 0, bar);
    tma_load_2d(sB, &tmB, 0, 0, bar);
  }
  __syncthreads();
  mbar_wait(bar, 0);
  float acc[4][2][4] = {};
  for (int k = 0; k < CK / 16; ++k) {
    uint32_t b01[4], b23[4];
    ld_b_kmajor<RB>(smem_u32(sB), 0, 8, k * 32, lane, b01);
    ld_b_kmajor<RB>(smem_u32(sB), 16, 24, k * 32, lane, b23);
    for (int mt = 0; mt < 2; ++mt) {
      uint32_t af[4];
      ld_a_kmajor<RB>(smem_u32(sA), shift_rows + warp * 32 + mt * 16, k * 32, lane, af);
      mma_bf16(acc[0][mt], af, b01[0], b01[1]);
      mma_bf16(acc[1][mt], af, b01[2], b01[3]);
      mma_bf16(acc[2][mt], af, b23[0], b23[1]);
      mma_bf16(acc[3][mt], af, b23[2], b23[3]);
    }
  }
  for (int n = 0; n < 4; ++n) {
    float v[8];
    frag_rows(scr + warp * 256, acc[n][0], acc[n][1], lane, v);
    for (int c = 0; c < 8; ++c) out[(warp * 32 + lane) * 32 + n * 8 + c] = v[c];
  }
}

void umma_shift_probe(const void* A, const void* Bm, float* out, int CK, int shift_rows, cudaStream_t st) {
  const CUtensorMap tmA = make_map(A, CK, 144, (uint64_t)CK * 2, CK, 144);
  const CUtensorMap tmB = make_map(Bm, CK, 32, (uint64_t)CK * 2, CK, 32);
  const int smem = 144 * 128 + 32 * 128 + 16 + 4 * 1024 + 1024;
  if (CK == 64) {
    cudaFuncSetAttribute(umma_shift_probe_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    umma_shift_probe_kernel<64><<<1, 128, smem, st>>>(tmA, tmB, out, shift_rows);
  } else if (CK == 32) {
    cudaFuncSetAttribute(umma_shift_probe_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    umma_shift_probe_kernel<32><<<1, 128, smem, st>>>(tmA, tmB, out, shift_rows);
  } else {
    cudaFuncSetAttribute(umma_shift_probe_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    umma_shift_probe_kernel<16><<<1, 128, smem, st>>>(tmA, tmB, out, shift_rows);
  }
}

}  // namespace nn
}  // namespace hefl
