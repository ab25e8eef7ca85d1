// Persistent, TMA-fed, cluster-shared-twiddle HE kernels for sm_90a (SURVEY.md K3, K4, K6, K7):
//
//   ntt2_kernel      in-place NTT / INTT of rows [rows][N]; coefficients travel by TMA tensor
//                    copies (SWIZZLE_128B) through a double-buffered shared-memory ring fed by a
//                    producer warp, results leave by TMA tensor store
//   encrypt2_kernel  sample -> 3 NTTs -> multiply-add with (pk, pk') -> ciphertext, one unit of
//                    8192/N ciphertexts per iteration; the three NTTs share one twiddle residency
//                    and one Philox call per coefficient
//   decrypt2_kernel  c0 + c1*s -> INTT -> *N^-1, fused
//
// All three are persistent (one CTA per SM), launched as clusters of two CTAs that work on the
// same RNS limb: the limb's (w, w') table is fetched once per cluster, each CTA issuing half of
// it as a multicast tensor copy that lands in both shared memories.
//
// Replaces the per-scalar HE.encryptFrac / decryptFrac loops (FLPyfhelin.py:216-217, :294-295).
#include <cuda.h>

#include <algorithm>

#include "../kernels.h"
#include "../philox.h"
#include "ntt2.cuh"

namespace hefl {
namespace cuda {

using namespace hefl::dev2;
using namespace hefl::sm90;

namespace {

constexpr int kProducerThreads = 32;

// ---- shared-memory carve-up: [twiddles][buf0][buf1?][barriers] ----------------------------
template <int LOGN, int NBUF>
struct Smem {
  static constexpr int kTw = 0;
  static constexpr int kBuf = tw_bytes(LOGN);
  static constexpr int kBars = kBuf + NBUF * unit_bytes(LOGN);
  static constexpr int kTotal = kBars + 64;
};

struct LimbWork {
  int limb;      // RNS limb of this cluster (-1: nothing to do)
  int worker;    // index of this CTA among the CTAs of the limb
  int nworkers;
};

// Clusters are dealt round-robin to limbs; the CTAs of a limb's clusters are its workers.
__device__ __forceinline__ LimbWork limb_work(int nlimbs) {
  const int cid = blockIdx.x >> 1, ncl = gridDim.x >> 1;
  LimbWork w;
  w.limb = cid % nlimbs;
  const int ci = cid / nlimbs;
  const int nci = (ncl - w.limb + nlimbs - 1) / nlimbs;
  w.worker = ci * 2 + (int)cluster_ctarank();
  w.nworkers = nci * 2;
  return w;
}

// Both CTAs of the cluster: arm the local barrier for the whole table, then issue one half of it
// as a multicast copy into both CTAs. Must be preceded by a cluster-wide barrier after mbar_init.
template <int LOGN>
__device__ __forceinline__ void load_twiddles(uint8_t* tw_smem, uint64_t* bar, const CUtensorMap* tmap,
                                              int table_row0) {
  constexpr int ROWS = tw_rows(LOGN);
  constexpr int HALF = ROWS / 2;                 // <= 256 rows per copy
  mbar_expect_tx(bar, ROWS * 128);
  const int r = (int)cluster_ctarank();
  tma_load_2d_mc(tw_smem + r * HALF * 128, tmap, 0, table_row0 + r * HALF, bar, (uint16_t)0x3);
}

__device__ __forceinline__ Limb make_limb(uint32_t tw_smem, const uint64_t* twg, const uint64_t* consts, int limb) {
  const uint64_t* c = consts + (size_t)limb * 8;
  Limb T;
  T.tw = tw_smem;
  T.twg = twg;
  T.q = c[0];
  T.two_q = 2 * c[0];
  T.rhi = c[2];
  T.ninv = c[3];
  T.ninv_p = c[4];
  return T;
}

// ------------------------------------------------------------------------------------------
// Stand-alone NTT / INTT
// ------------------------------------------------------------------------------------------
struct NttArgs {
  const uint64_t* tw2;      // [L][2][N][2]
  const uint64_t* consts;   // [L][8]
  int L;
  int64_t rows;
};

template <int LOGN>
struct Box {
  static constexpr int ROWS128 = (1 << LOGN) / 16;               // 128-byte rows per polynomial
  static constexpr int BOX = ROWS128 < 256 ? ROWS128 : 256;      // rows per tensor copy
  static constexpr int PER_POLY = ROWS128 / BOX;
};

template <int LOGN, bool INV, unsigned CORR>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads + kProducerThreads, 1)
ntt2_kernel(const __grid_constant__ CUtensorMap dmap, const __grid_constant__ CUtensorMap tmap, NttArgs a) {
  constexpr int NBUF = LOGN <= 13 ? 2 : 1;
  constexpr int NP = num_passes(LOGN);
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  constexpr int N = 1 << LOGN;
  using S = Smem<LOGN, NBUF>;
  using B = Box<LOGN>;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBars);   // [0] twiddles, [1..2] full, [3..4] done
  const int tid = threadIdx.x;
  const LimbWork W = limb_work(a.L);

  if (tid == 0) {
    mbar_init(&bars[0], 1);
    for (int b = 0; b < NBUF; ++b) {
      mbar_init(&bars[1 + b], 1);
      mbar_init(&bars[3 + b], kThreads / 32);
    }
    fence_barrier_init();
  }
  cluster_sync_all();

  const int64_t J = a.rows / a.L;                       // polynomials of this limb: rows limb + L*j
  const int64_t units = (J + POLYS - 1) / POLYS;
  const int table = W.limb * 2 + (INV ? 1 : 0);

  if (tid >= kThreads) {
    // ===== producer warp: twiddles, then the load / store ring =====
    if (tid == kThreads) {
      load_twiddles<LOGN>(smem + S::kTw, &bars[0], &tmap, table * (N * 16 / 128));
      auto issue_load = [&](int64_t u, int b) {
        const int64_t j0 = u * POLYS;
        const int np = (int)((J - j0) < POLYS ? (J - j0) : POLYS);
        mbar_expect_tx(&bars[1 + b], (uint32_t)np * N * 8);
        for (int p = 0; p < np; ++p) {
          const int64_t row = W.limb + a.L * (j0 + p);
          for (int x = 0; x < B::PER_POLY; ++x)
            tma_load_2d(smem + S::kBuf + b * unit_bytes(LOGN) + p * N * 8 + x * B::BOX * 128, &dmap, 0,
                        (int)(row * B::ROWS128 + x * B::BOX), &bars[1 + b]);
        }
      };
      int64_t u = W.worker;
      for (int b = 0; b < NBUF && u + (int64_t)b * W.nworkers < units; ++b) issue_load(u + (int64_t)b * W.nworkers, b);
      for (int it = 0; u < units; u += W.nworkers, ++it) {
        const int b = it % NBUF;
        mbar_wait(&bars[3 + b], (it / NBUF) & 1);        // consumers finished (and fenced) buffer b
        const int64_t j0 = u * POLYS;
        const int np = (int)((J - j0) < POLYS ? (J - j0) : POLYS);
        for (int p = 0; p < np; ++p) {
          const int64_t row = W.limb + a.L * (j0 + p);
          for (int x = 0; x < B::PER_POLY; ++x)
            tma_store_2d(&dmap, 0, (int)(row * B::ROWS128 + x * B::BOX),
                         smem + S::kBuf + b * unit_bytes(LOGN) + p * N * 8 + x * B::BOX * 128);
        }
        tma_commit();
        const int64_t un = u + (int64_t)NBUF * W.nworkers;
        if (un < units) {
          tma_wait_read<0>();                             // the store has drained buffer b
          issue_load(un, b);
        }
      }
      tma_wait_all<0>();
    }
  } else {
    // ===== 512 compute threads =====
    mbar_wait(&bars[0], 0);
    const Limb T = make_limb(sbase + S::kTw, a.tw2 + (size_t)table * N * 2, a.consts, W.limb);
    int it = 0;
    for (int64_t u = W.worker; u < units; u += W.nworkers, ++it) {
      const int b = it % NBUF;
      const uint32_t buf = sbase + S::kBuf + b * unit_bytes(LOGN);
      mbar_wait(&bars[1 + b], (it / NBUF) & 1);
      if constexpr (!INV) {
        // passes 0 .. NP-2 in place, the last one reduces to [0, q) on its way out
        if constexpr (NP >= 1) { fwd_pass_smem<LOGN, 0>(buf, T); }
        if constexpr (NP >= 3) { fwd_pass_smem<LOGN, 1>(buf, T); }
        if constexpr (NP >= 4) { fwd_pass_smem<LOGN, 2>(buf, T); }
        {
          using GG = Geo<LOGN, NP - 1>;
#pragma unroll 1
          for (int j = 0; j < GG::PER_THREAD; ++j) {
            const GG G(tid + j * kThreads);
            uint64_t x[GG::E];
            group_load<LOGN, NP - 1>(buf, G, x);
            fwd_butterflies<GG::ST, GG::R>(x, G.high, T);
#pragma unroll
            for (int k = 0; k < GG::E; ++k) x[k] = full_reduce(x[k], T);
            group_store<LOGN, NP - 1>(buf, G, x);
          }
        }
      } else {
        if constexpr (NP >= 4) { inv_pass_smem<LOGN, 3, 4, CORR>(buf, T); }
        if constexpr (NP >= 3) { inv_pass_smem<LOGN, 2, 4, CORR>(buf, T); }
        inv_pass_smem<LOGN, 1, 4, CORR>(buf, T);
        {
          using GG = Geo<LOGN, 0>;
          constexpr int BIN = inv_bound_in<LOGN>(0, 4, CORR);
#pragma unroll 1
          for (int j = 0; j < GG::PER_THREAD; ++j) {
            const GG G(tid + j * kThreads);
            uint64_t x[GG::E];
            group_load<LOGN, 0>(buf, G, x);
            if constexpr (CORR & 1u) {
#pragma unroll
              for (int k = 0; k < GG::E; ++k) x[k] = lazy_reduce(x[k], T);
            }
            inv_butterflies<GG::ST, GG::R, BIN>(x, G.high, T);
#pragma unroll
            for (int k = 0; k < GG::E; ++k) x[k] = mul_shoup(x[k], T.ninv, T.ninv_p, T.q);
            group_store<LOGN, 0>(buf, G, x);
          }
        }
      }
      fence_proxy_async();                 // generic-proxy writes -> visible to the TMA store
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&bars[3 + b]);
    }
  }
  cluster_sync_all();   // nobody leaves while the partner may still be receiving its multicast half
}

// ------------------------------------------------------------------------------------------
// Fused public-key encryption
// ------------------------------------------------------------------------------------------
struct EncArgs {
  const int64_t* msg;       // [C][N] signed, or nullptr (encryption of zero)
  const uint64_t* pkx;      // [2][L][N][2]  (pk, pk')
  uint64_t* ct;             // [C][2][L][N]
  const uint64_t* tw2;
  const uint64_t* consts;
  const uint64_t* msg_scale;
  uint64_t seed;
  uint32_t ct_offset;
  int L;
  int64_t C;
  uint64_t* scratch;        // N = 16384 only: [grid][N] words for u_hat, private to the launch
  bool acc;                 // ct = (ct + Enc(m)) mod q: the epilogue reads the old word where it stores the new one
};

__device__ __forceinline__ uint32_t pack_e(int e0, int e1) { return ((uint32_t)e0 & 0xFFu) | (((uint32_t)e1 & 0xFFu) << 8); }
__device__ __forceinline__ int unpack_e0(uint32_t p) { return (int)(int8_t)(p & 0xFFu); }
__device__ __forceinline__ int unpack_e1(uint32_t p) { return (int)(int8_t)((p >> 8) & 0xFFu); }

// last forward pass of NTT(e + ...) fused with  c = reduce(u_hat * pk + a_hat)  and the store.
// The thread owns E = 8 or 16 contiguous coefficients; the epilogue walks them four at a time so
// that only 4 (pk, pk') pairs and 4 words of u_hat are live next to the E accumulators.
// USCR: u_hat does not fit in shared memory next to the working buffer (N = 16384): it lives in a per-CTA
// global scratch row that the same thread wrote with the same geometry (L2 resident, coherent loads).
template <int LOGN, bool USCR>
__device__ __forceinline__ void enc_epilogue(uint32_t bufA, uint32_t bufU, const uint64_t* uscr, const Limb& T,
                                             const uint64_t* pkx_limb, uint64_t* ct, int64_t c_first, int64_t C,
                                             int which, int L, int limb, bool acc) {
  constexpr int NP = num_passes(LOGN);
  constexpr int N = 1 << LOGN;
  using GG = Geo<LOGN, NP - 1>;
  static_assert(GG::TL == 0, "the last pass must own contiguous coefficients");
#pragma unroll 1
  for (int j = 0; j < GG::PER_THREAD; ++j) {
    const GG G(threadIdx.x + j * kThreads);
    uint64_t x[GG::E];
    group_load<LOGN, NP - 1>(bufA, G, x);
    fwd_butterflies<GG::ST, GG::R>(x, G.high, T);
    const int64_t c = c_first + G.poly;
    const uint64_t* pp = pkx_limb + (size_t)G.coef * 2;
    uint64_t* o = ct + ((size_t)((c < C ? c : C - 1) * 2 + which) * L + limb) * N + G.coef;
    const uint32_t row = (G.base * 8u) & ~127u;
    const uint32_t ch0 = ((G.base * 8u) >> 4) & 7u;
    const uint32_t rs = (row >> 7) & 7u;
#pragma unroll
    for (int v = 0; v < GG::E / 4; ++v) {
      uint64_t pk[2][4], uh[4], r[4];
      ldg256(pp + 8 * v, pk[0]);
      ldg256(pp + 8 * v + 4, pk[1]);
      if constexpr (USCR) {
        asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(uh[0]), "=l"(uh[1]) : "l"(uscr + G.base + 4 * v)
                     : "memory");
        asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(uh[2]), "=l"(uh[3]) : "l"(uscr + G.base + 4 * v + 2)
                     : "memory");
      } else {
        lds128(bufU + row + (((ch0 + 2 * v) ^ rs) << 4), uh[0], uh[1]);
        lds128(bufU + row + (((ch0 + 2 * v + 1) ^ rs) << 4), uh[2], uh[3]);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t t = mul_shoup_lazy(uh[k], pk[k >> 1][(k & 1) * 2], pk[k >> 1][(k & 1) * 2 + 1], T.q);
        uint64_t s = t + lazy_reduce(x[4 * v + k], T);     // < 4q
        s = s >= T.two_q ? s - T.two_q : s;
        r[k] = s >= T.q ? s - T.q : s;
      }
      if (acc && c < C) {
        uint64_t old[4];
        asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(old[0]), "=l"(old[1]) : "l"(o + 4 * v) : "memory");
        asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(old[2]), "=l"(old[3]) : "l"(o + 4 * v + 2) : "memory");
#pragma unroll
        for (int k = 0; k < 4; ++k) r[k] = add_mod(r[k], old[k], T.q);
      }
      if (c < C) stg256(o + 4 * v, r[0], r[1], r[2], r[3]);
    }
  }
  compute_sync();
}

template <int LOGN>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads, 1)
encrypt2_kernel(const __grid_constant__ CUtensorMap tmap, EncArgs a) {
  constexpr int NP = num_passes(LOGN);
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  constexpr int N = 1 << LOGN;
  constexpr bool USCR = LOGN >= 14;                 // one working buffer in shared memory, u_hat in global scratch
  using S = Smem<LOGN, USCR ? 1 : 2>;
  using G0 = Geo<LOGN, 0>;
  constexpr int PT = G0::PER_THREAD;                // radix-16 groups per thread in the first pass (1, or 2 at N = 16384)
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBars);
  const int tid = threadIdx.x;
  const LimbWork W = limb_work(a.L);
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    fence_barrier_init();
  }
  cluster_sync_all();
  if (tid == 0) load_twiddles<LOGN>(smem + S::kTw, &bars[0], &tmap, (W.limb * 2) * (N * 16 / 128));
  const Limb T = make_limb(sbase + S::kTw, a.tw2 + (size_t)(W.limb * 2) * N * 2, a.consts, W.limb);
  const Modulus m{T.q, a.consts[W.limb * 8 + 1], a.consts[W.limb * 8 + 2]};
  const uint64_t sc = a.msg_scale ? a.msg_scale[W.limb] : 1;
  const uint32_t bufU = sbase + S::kBuf;
  const uint32_t bufA = USCR ? bufU : bufU + unit_bytes(LOGN);
  uint64_t* uscr = USCR ? a.scratch + (size_t)blockIdx.x * (1u << unit_log(LOGN)) : nullptr;
  const uint64_t* pk0 = a.pkx + ((size_t)(0 * a.L + W.limb) * N) * 2;
  const uint64_t* pk1 = a.pkx + ((size_t)(1 * a.L + W.limb) * N) * 2;
  mbar_wait(&bars[0], 0);

  const int64_t units = (a.C + POLYS - 1) / POLYS;
  for (int64_t u = W.worker; u < units; u += W.nworkers) {
    const int64_t c_first = u * POLYS;
    uint32_t epack[PT][8];
    // ---- phase 1: u_hat = NTT(u), sampled straight into the registers of the first pass ----
#pragma unroll
    for (int j = 0; j < PT; ++j) {
      const G0 G(tid + j * kThreads);
      const uint32_t ctid = a.ct_offset + (uint32_t)(c_first + G.poly);
      uint64_t x[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const EncNoise z = sample_enc_noise(a.seed, ctid, G.coef + ((uint32_t)k << G0::TL));
        x[k] = lift_signed(z.u, T.q);
        const uint32_t pe = pack_e(z.e0, z.e1);
        if (k & 1) epack[j][k >> 1] |= pe << 16; else epack[j][k >> 1] = pe;
      }
      fwd_butterflies<G0::ST, G0::R>(x, G.high, T);
      group_store<LOGN, 0>(bufU, G, x);
    }
    compute_sync();
    fwd_pass_smem<LOGN, 1>(bufU, T);
    if constexpr (NP >= 4) fwd_pass_smem<LOGN, 2>(bufU, T);
    if constexpr (!USCR) {
      fwd_pass_smem<LOGN, NP - 1>(bufU, T);
    } else {
      // last pass straight to the global scratch row (same geometry as the epilogues that read it back)
      using GL = Geo<LOGN, NP - 1>;
#pragma unroll 1
      for (int j = 0; j < GL::PER_THREAD; ++j) {
        const GL G(tid + j * kThreads);
        uint64_t x[GL::E];
        group_load<LOGN, NP - 1>(bufU, G, x);
        fwd_butterflies<GL::ST, GL::R>(x, G.high, T);
#pragma unroll
        for (int v = 0; v < GL::E / 4; ++v) stg256(uscr + G.base + 4 * v, x[4 * v], x[4 * v + 1], x[4 * v + 2], x[4 * v + 3]);
      }
      compute_sync();
    }
    // ---- phase 2: c0 = u_hat * pk0 + NTT(e0 + m) ----
#pragma unroll
    for (int j = 0; j < PT; ++j) {
      const G0 G(tid + j * kThreads);
      uint64_t x[16];
      const int64_t c = c_first + G.poly;
      const bool have_msg = a.msg != nullptr && c < a.C;
      const int64_t* mrow = a.msg + (have_msg ? c * N : 0);
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint32_t pe = (k & 1) ? (epack[j][k >> 1] >> 16) : epack[j][k >> 1];
        uint64_t v = lift_signed(unpack_e0(pe), T.q);
        if (have_msg) {
          uint64_t mm = reduce_signed(mrow[G.coef + ((uint32_t)k << G0::TL)], m);
          if (sc != 1) mm = mul_mod(mm, sc, m);
          v += mm;                                 // < 2q: fine for the lazy butterflies
        }
        x[k] = v;
      }
      fwd_butterflies<G0::ST, G0::R>(x, G.high, T);
      group_store<LOGN, 0>(bufA, G, x);
    }
    compute_sync();
    if constexpr (NP >= 3) fwd_pass_smem<LOGN, 1>(bufA, T);
    if constexpr (NP >= 4) fwd_pass_smem<LOGN, 2>(bufA, T);
    enc_epilogue<LOGN, USCR>(bufA, bufU, uscr, T, pk0, a.ct, c_first, a.C, 0, a.L, W.limb, a.acc);
    // ---- phase 3: c1 = u_hat * pk1 + NTT(e1) ----
#pragma unroll
    for (int j = 0; j < PT; ++j) {
      const G0 G(tid + j * kThreads);
      uint64_t x[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint32_t pe = (k & 1) ? (epack[j][k >> 1] >> 16) : epack[j][k >> 1];
        x[k] = lift_signed(unpack_e1(pe), T.q);
      }
      fwd_butterflies<G0::ST, G0::R>(x, G.high, T);
      group_store<LOGN, 0>(bufA, G, x);
    }
    compute_sync();
    if constexpr (NP >= 3) fwd_pass_smem<LOGN, 1>(bufA, T);
    if constexpr (NP >= 4) fwd_pass_smem<LOGN, 2>(bufA, T);
    enc_epilogue<LOGN, USCR>(bufA, bufU, uscr, T, pk1, a.ct, c_first, a.C, 1, a.L, W.limb, a.acc);
  }
  cluster_sync_all();
}

// ------------------------------------------------------------------------------------------
// Fused decrypt
// ------------------------------------------------------------------------------------------
struct DecArgs {
  const uint64_t* ct;       // [C][2][Lct][N]
  const uint64_t* skx;      // [L][N][2]  (s, s')
  uint64_t* out;            // [C][k][N]
  const uint64_t* tw2;
  const uint64_t* consts;
  int Lct, k;
  int64_t C;
};

template <int LOGN, unsigned CORR>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads, 1)
decrypt2_kernel(const __grid_constant__ CUtensorMap tmap, DecArgs a) {
  constexpr int NP = num_passes(LOGN);
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  constexpr int N = 1 << LOGN;
  using S = Smem<LOGN, 1>;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBars);
  const int tid = threadIdx.x;
  const LimbWork W = limb_work(a.k);
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    fence_barrier_init();
  }
  cluster_sync_all();
  if (tid == 0) load_twiddles<LOGN>(smem + S::kTw, &bars[0], &tmap, (W.limb * 2 + 1) * (N * 16 / 128));
  const Limb T = make_limb(sbase + S::kTw, a.tw2 + (size_t)(W.limb * 2 + 1) * N * 2, a.consts, W.limb);
  const uint32_t buf = sbase + S::kBuf;
  const uint64_t* sx = a.skx + (size_t)W.limb * N * 2;
  mbar_wait(&bars[0], 0);

  const int64_t units = (a.C + POLYS - 1) / POLYS;
  for (int64_t u = W.worker; u < units; u += W.nworkers) {
    const int64_t c_first = u * POLYS;
    // first inverse pass (unit stride) fused with  x = c0 + c1 * s
    {
      using GG = Geo<LOGN, NP - 1>;
      constexpr int BIN = inv_bound_in<LOGN>(NP - 1, 4, CORR & ~(1u << (NP - 1)));
      static_assert(GG::TL == 0, "the first inverse pass must own contiguous coefficients");
#pragma unroll 1
      for (int j = 0; j < GG::PER_THREAD; ++j) {
        const GG G(tid + j * kThreads);
        int64_t c = c_first + G.poly;
        if (c >= a.C) c = a.C - 1;                 // tail of the last unit: recompute a valid one
        const uint64_t* c0 = a.ct + ((size_t)(c * 2 + 0) * a.Lct + W.limb) * N + G.coef;
        const uint64_t* c1 = a.ct + ((size_t)(c * 2 + 1) * a.Lct + W.limb) * N + G.coef;
        const uint64_t* sp = sx + (size_t)G.coef * 2;
        uint64_t x[GG::E];
#pragma unroll
        for (int v = 0; v < GG::E / 4; ++v) {
          uint64_t v0[4], v1[4], s[2][4];
          ldg256(c0 + 4 * v, v0);
          ldg256(c1 + 4 * v, v1);
          ldg256(sp + 8 * v, s[0]);
          ldg256(sp + 8 * v + 4, s[1]);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            x[4 * v + k] = v0[k] + mul_shoup_lazy(v1[k], s[k >> 1][(k & 1) * 2], s[k >> 1][(k & 1) * 2 + 1], T.q);
        }
        inv_butterflies<GG::ST, GG::R, BIN>(x, G.high, T);
        group_store<LOGN, NP - 1>(buf, G, x);
      }
      compute_sync();
    }
    if constexpr (NP >= 4) inv_pass_smem<LOGN, 2, 4, CORR>(buf, T);
    if constexpr (NP >= 3) inv_pass_smem<LOGN, 1, 4, CORR>(buf, T);
    {
      using GG = Geo<LOGN, 0>;
      constexpr int BIN = inv_bound_in<LOGN>(0, 4, CORR);
#pragma unroll 1
      for (int j = 0; j < GG::PER_THREAD; ++j) {
        const GG G(tid + j * kThreads);
        uint64_t x[GG::E];
        group_load<LOGN, 0>(buf, G, x);
        if constexpr (CORR & 1u) {
#pragma unroll
          for (int k = 0; k < GG::E; ++k) x[k] = lazy_reduce(x[k], T);
        }
        inv_butterflies<GG::ST, GG::R, BIN>(x, G.high, T);
        const int64_t c = c_first + G.poly;
        if (c < a.C) {
          uint64_t* o = a.out + ((size_t)c * a.k + W.limb) * N + G.coef;
#pragma unroll
          for (int k = 0; k < GG::E; ++k) o[(size_t)k << GG::TL] = mul_shoup(x[k], T.ninv, T.ninv_p, T.q);
        }
      }
      compute_sync();
    }
  }
  cluster_sync_all();
}

// (x, floor(x * 2^64 / q)) pairs for keys: one-time, per key.
__global__ void shoup_pairs_kernel(const uint64_t* __restrict__ x, uint64_t* __restrict__ out, int L, int n,
                                   const uint64_t* __restrict__ consts) {
  const int64_t row = blockIdx.y;
  const uint64_t* c = consts + (size_t)(row % L) * 8;
  const uint64_t q = c[0], rlo = c[1], rhi = c[2];   // floor(2^128 / q) = rhi:rlo
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t v = x[row * n + i];
    // candidate = floor(v * floor(2^128/q) / 2^64) is at most 1 below floor(v * 2^64 / q)
    uint64_t cand = v * rhi + mul_hi(v, rlo);
    // remainder of (v << 64) - cand * q, a 128-bit value known to be in [0, 2q)
    uint64_t plo, phi;
    mul_wide(cand, q, phi, plo);
    uint64_t rem_lo = 0 - plo;
    uint64_t rem_hi = v - phi - (plo != 0 ? 1 : 0);
    while (rem_hi != 0 || rem_lo >= q) {
      const uint64_t nl = rem_lo - q;
      rem_hi -= (rem_lo < q) ? 1 : 0;
      rem_lo = nl;
      ++cand;
    }
    out[(row * n + i) * 2] = v;
    out[(row * n + i) * 2 + 1] = cand;
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// u64 buffer of `bytes` bytes seen as [bytes/128][16]; copies move `box_rows` rows of 128 bytes.
CUtensorMap rows128_map(const void* ptr, uint64_t bytes, uint32_t box_rows) {
  return tensor_map(ptr, CU_TENSOR_MAP_DATA_TYPE_UINT64, {16, bytes / 128}, {128}, {16, box_rows},
                    CU_TENSOR_MAP_SWIZZLE_128B);
}

// Per-role CTA budgets (0 = every SM). The persistent kernels take one SM per CTA; when the pipelined FedAvg
// runs encrypt, the ciphertext all-reduce and decrypt on three streams they only overlap if each leaves SMs to
// the others, so the runner partitions the chip (set_cta_limits) instead of letting three full-chip kernels queue.
int g_limit[3] = {0, 0, 0};   // 0 ntt, 1 encrypt, 2 decrypt

int grid_ctas(int role = 0) {
  int n = device_sm_count() & ~1;
  if (g_limit[role] > 0 && g_limit[role] < n) n = g_limit[role] & ~1;
  return n < 2 ? 2 : n;
}

template <class K>
void set_smem(K kernel, int bytes) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

template <int LOGN, bool INV, unsigned CORR>
void launch_ntt2(uint64_t* data, int64_t rows, int L, const uint64_t* tw2, const uint64_t* consts, cudaStream_t st) {
  constexpr int NBUF = LOGN <= 13 ? 2 : 1;
  constexpr int N = 1 << LOGN;
  const CUtensorMap dmap = rows128_map(data, (uint64_t)rows * N * 8, Box<LOGN>::BOX);
  const CUtensorMap tmap = rows128_map(tw2, (uint64_t)L * 2 * N * 16, tw_rows(LOGN) / 2);
  NttArgs a{tw2, consts, L, rows};
  auto k = ntt2_kernel<LOGN, INV, CORR>;
  set_smem(k, Smem<LOGN, NBUF>::kTotal);
  k<<<grid_ctas(), kThreads + kProducerThreads, Smem<LOGN, NBUF>::kTotal, st>>>(dmap, tmap, a);
}

template <int LOGN>
bool dispatch_ntt2(uint64_t* data, int64_t rows, int L, const uint64_t* tw2, const uint64_t* consts, bool inverse,
                   int qbits, cudaStream_t st) {
  constexpr int NP = num_passes(LOGN);
  if (!inverse) {
    launch_ntt2<LOGN, false, 0u>(data, rows, L, tw2, consts, st);
    return true;
  }
  switch (pick_corr<LOGN>(qbits)) {
    case 0u: launch_ntt2<LOGN, true, 0u>(data, rows, L, tw2, consts, st); return true;
    case 1u << 1: launch_ntt2<LOGN, true, 1u << 1>(data, rows, L, tw2, consts, st); return true;
    case (1u << (NP - 1)) - 1u: launch_ntt2<LOGN, true, (1u << (NP - 1)) - 1u>(data, rows, L, tw2, consts, st); return true;
    default: return false;
  }
}

template <int LOGN>
void launch_encrypt2(EncArgs a, cudaStream_t st) {
  constexpr int N = 1 << LOGN;
  constexpr int NBUF = LOGN >= 14 ? 1 : 2;
  const CUtensorMap tmap = rows128_map(a.tw2, (uint64_t)a.L * 2 * N * 16, tw_rows(LOGN) / 2);
  auto k = encrypt2_kernel<LOGN>;
  set_smem(k, Smem<LOGN, NBUF>::kTotal);
  k<<<grid_ctas(1), kThreads, Smem<LOGN, NBUF>::kTotal, st>>>(tmap, a);
}

template <int LOGN, unsigned CORR>
void launch_decrypt2(const DecArgs& a, int Ltab, cudaStream_t st) {
  constexpr int N = 1 << LOGN;
  const CUtensorMap tmap = rows128_map(a.tw2, (uint64_t)Ltab * 2 * N * 16, tw_rows(LOGN) / 2);
  auto k = decrypt2_kernel<LOGN, CORR>;
  set_smem(k, Smem<LOGN, 1>::kTotal);
  k<<<grid_ctas(2), kThreads, Smem<LOGN, 1>::kTotal, st>>>(tmap, a);
}

template <int LOGN>
bool dispatch_decrypt2(const DecArgs& a, int Ltab, int qbits, cudaStream_t st) {
  constexpr int NP = num_passes(LOGN);
  switch (pick_corr<LOGN>(qbits)) {
    case 0u: launch_decrypt2<LOGN, 0u>(a, Ltab, st); return true;
    case 1u << 1: launch_decrypt2<LOGN, 1u << 1>(a, Ltab, st); return true;
    case (1u << (NP - 1)) - 1u: launch_decrypt2<LOGN, (1u << (NP - 1)) - 1u>(a, Ltab, st); return true;
    default: return false;
  }
}

}  // namespace

void shoup_pairs(const uint64_t* x, uint64_t* out, int64_t rows, int L, int n, const uint64_t* consts,
                 cudaStream_t st) {
  if (rows == 0) return;
  dim3 grid((n + 1023) / 1024, (unsigned)rows);
  shoup_pairs_kernel<<<grid, 256, 0, st>>>(x, out, L, n, consts);
  note_launch();
}

// The fast path needs every prime below 2^58 (lazy forward butterflies without correction), at
// most as many limbs as clusters, and 1024 <= N <= 16384.
bool ntt2_supported(int logn, int L, int qbits) {
  const int g = std::min(grid_ctas(0), std::min(grid_ctas(1), grid_ctas(2)));
  return logn >= 10 && logn <= 14 && qbits <= 58 && L <= g / 2;
}

void set_cta_limits(int ntt, int enc, int dec) {
  g_limit[0] = ntt;
  g_limit[1] = enc;
  g_limit[2] = dec;
}

bool ntt2(uint64_t* data, int64_t rows, int L, int logn, const uint64_t* tw2, const uint64_t* consts, int qbits,
          bool inverse, cudaStream_t st) {
  if (rows == 0) return true;
  if (!ntt2_supported(logn, L, qbits) || rows % L != 0) return false;
  bool ok = false;
  switch (logn) {
    case 10: ok = dispatch_ntt2<10>(data, rows, L, tw2, consts, inverse, qbits, st); break;
    case 11: ok = dispatch_ntt2<11>(data, rows, L, tw2, consts, inverse, qbits, st); break;
    case 12: ok = dispatch_ntt2<12>(data, rows, L, tw2, consts, inverse, qbits, st); break;
    case 13: ok = dispatch_ntt2<13>(data, rows, L, tw2, consts, inverse, qbits, st); break;
    case 14: ok = dispatch_ntt2<14>(data, rows, L, tw2, consts, inverse, qbits, st); break;
  }
  if (ok) note_launch();
  return ok;
}

int64_t encrypt2_scratch_words(int logn) { return logn >= 14 ? (int64_t)grid_ctas(1) << logn : 0; }

bool encrypt2(const int64_t* msg, const uint64_t* pkx, uint64_t* ct, int64_t C, int L, int logn, const uint64_t* tw2,
              const uint64_t* consts, const uint64_t* msg_scale, uint64_t seed, uint32_t ct_offset, int qbits,
              uint64_t* scratch, bool accumulate, cudaStream_t st) {
  if (C == 0) return true;
  if (!ntt2_supported(logn, L, qbits)) return false;
  if (logn >= 14 && scratch == nullptr) return false;
  {
    // A persistent CTA wants at least two units of 8192 coefficients: below that (the 109
    // ciphertexts of the medical CNN) the one-CTA-per-(ciphertext, limb) kernel fills the GPU
    // better (measured 0.107 vs 0.131 ms at n = 4096, L = 3, C = 109).
    const int64_t units = logn >= 13 ? C : (C * (1ll << logn) + 8191) / 8192;
    const int64_t workers = (grid_ctas(1) / 2 / L) * 2;
    if (units < 2 * workers) return false;
  }
  const EncArgs a{msg, pkx, ct, tw2, consts, msg_scale, seed, ct_offset, L, C, scratch, accumulate};
  switch (logn) {
    case 10: launch_encrypt2<10>(a, st); break;
    case 11: launch_encrypt2<11>(a, st); break;
    case 12: launch_encrypt2<12>(a, st); break;
    case 13: launch_encrypt2<13>(a, st); break;
    case 14: launch_encrypt2<14>(a, st); break;
  }
  note_launch();
  return true;
}

bool decrypt2(const uint64_t* ct, const uint64_t* skx, uint64_t* out, int64_t C, int Lct, int k, int logn,
              const uint64_t* tw2, const uint64_t* consts, int Ltab, int qbits, cudaStream_t st) {
  if (C == 0) return true;
  if (!ntt2_supported(logn, k, qbits)) return false;
  const DecArgs a{ct, skx, out, tw2, consts, Lct, k, C};
  bool ok = false;
  switch (logn) {
    case 10: ok = dispatch_decrypt2<10>(a, Ltab, qbits, st); break;
    case 11: ok = dispatch_decrypt2<11>(a, Ltab, qbits, st); break;
    case 12: ok = dispatch_decrypt2<12>(a, Ltab, qbits, st); break;
    case 13: ok = dispatch_decrypt2<13>(a, Ltab, qbits, st); break;
    case 14: ok = dispatch_decrypt2<14>(a, Ltab, qbits, st); break;
  }
  if (ok) note_launch();
  return ok;
}

}  // namespace cuda
}  // namespace hefl
