// Fused evaluation kernels on top of ntt2.cuh (SURVEY.md K9, K10):
//
//   rescale2_kernel    ct <- round(ct / q_last): INTT of the last limb, centred lift, NTT under every
//                      remaining prime, subtract, multiply by q_last^-1 -- one launch, no per-limb loop on the host
//   keyswitch2_kernel  sum over (source limb i, digit k) of NTT_j(digit_{i,k}(d2)) * evk[i][k], accumulated in
//                      shared memory per (ciphertext, target limb j), added onto (d0, d1) -- one launch
//   tensor3_kernel     (a0 b0, a0 b1 + a1 b0, a1 b1), element-wise
//
// These walk over several limbs inside one CTA, so the twiddles come from global memory (L2 resident) instead of a
// resident shared-memory table; they are API-parity paths (ct * float with rescale, ct * ct with relinearisation:
// FLPyfhelin.py:385, :357-364), not the FedAvg hot path.
#include <cuda.h>

#include <algorithm>
#include <cstdio>
#include <stdexcept>

#include "../kernels.h"
#include "ntt2.cuh"

namespace hefl {
namespace cuda {

using namespace hefl::dev2;
using namespace hefl::sm90;

namespace {

constexpr bool kG = true;   // global-memory twiddles

__device__ __forceinline__ Limb limb_global(const uint64_t* tw2, const uint64_t* consts, int limb, int inv, int n) {
  const uint64_t* c = consts + (size_t)limb * 8;
  Limb T;
  T.tw = 0;
  T.twg = tw2 + (size_t)(limb * 2 + inv) * n * 2;
  T.q = c[0];
  T.two_q = 2 * c[0];
  T.rhi = c[2];
  T.ninv = c[3];
  T.ninv_p = c[4];
  return T;
}

// ---- rescale ---------------------------------------------------------------------------------
struct RescaleArgs {
  const uint64_t* ct;     // [rows][lvl][N], rows = C * 2
  uint64_t* out;          // [rows][lvl - 1][N]
  const uint64_t* tw2;
  const uint64_t* consts;
  uint64_t inv[16], inv_p[16];   // q_last^-1 mod q_j, Shoup companion
  int lvl;
  int64_t rows;
};

template <int LOGN, unsigned CORR>
__global__ void __launch_bounds__(kThreads, 1) rescale2_kernel(RescaleArgs a) {
  constexpr int NP = num_passes(LOGN);
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  constexpr int N = 1 << LOGN;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t bufA = smem_u32(smem), bufB = bufA + unit_bytes(LOGN);
  const int tid = threadIdx.x;
  const int last = a.lvl - 1;
  const Limb TL = limb_global(a.tw2, a.consts, last, 1, N);
  const uint64_t half = TL.q >> 1;
  const int64_t units = (a.rows + POLYS - 1) / POLYS;
  for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
    const int64_t r_first = u * POLYS;
    // ---- coefficient form of the last limb, r = [c + q_last/2] mod q_last, kept in bufA ----
    {
      using GG = Geo<LOGN, NP - 1>;
      constexpr int BIN = inv_bound_in<LOGN>(NP - 1, 4, CORR & ~(1u << (NP - 1)));
#pragma unroll 1
      for (int j = 0; j < GG::PER_THREAD; ++j) {
        const GG G(tid + j * kThreads);
        int64_t r = r_first + G.poly;
        if (r >= a.rows) r = a.rows - 1;
        const uint64_t* src = a.ct + ((size_t)r * a.lvl + last) * N + G.coef;
        uint64_t x[GG::E];
#pragma unroll
        for (int v = 0; v < GG::E / 4; ++v) {
          uint64_t t[4];
          ldg256(src + 4 * v, t);
#pragma unroll
          for (int k = 0; k < 4; ++k) x[4 * v + k] = t[k];
        }
        inv_butterflies<GG::ST, GG::R, BIN, kG>(x, G.high, TL);
        group_store<LOGN, NP - 1>(bufA, G, x);
      }
      compute_sync();
    }
    if constexpr (NP >= 4) inv_pass_smem<LOGN, 2, 4, CORR, kG>(bufA, TL);
    if constexpr (NP >= 3) inv_pass_smem<LOGN, 1, 4, CORR, kG>(bufA, TL);
    {
      using GG = Geo<LOGN, 0>;
      constexpr int BIN = inv_bound_in<LOGN>(0, 4, CORR);
#pragma unroll 1
      for (int j = 0; j < GG::PER_THREAD; ++j) {
        const GG G(tid + j * kThreads);
        uint64_t x[GG::E];
        group_load<LOGN, 0>(bufA, G, x);
        if constexpr (CORR & 1u) {
#pragma unroll
          for (int k = 0; k < GG::E; ++k) x[k] = lazy_reduce(x[k], TL);
        }
        inv_butterflies<GG::ST, GG::R, BIN, kG>(x, G.high, TL);
#pragma unroll
        for (int k = 0; k < GG::E; ++k) x[k] = add_mod(mul_shoup(x[k], TL.ninv, TL.ninv_p, TL.q), half, TL.q);
        group_store<LOGN, 0>(bufA, G, x);
      }
      // no barrier: the forward first pass below has the same geometry (each thread re-reads its own words)
    }
    // ---- every remaining limb: t = NTT_j((r mod q_j) - (half mod q_j)); out = (c_j - t) * q_last^-1 ----
    for (int l = 0; l < last; ++l) {
      const Limb T = limb_global(a.tw2, a.consts, l, 0, N);
      const Modulus m{T.q, a.consts[l * 8 + 1], a.consts[l * 8 + 2]};
      const uint64_t half_l = barrett_reduce_64(half, m);
      {
        using GG = Geo<LOGN, 0>;
#pragma unroll 1
        for (int j = 0; j < GG::PER_THREAD; ++j) {
          const GG G(tid + j * kThreads);
          uint64_t x[GG::E];
          group_load<LOGN, 0>(bufA, G, x);
#pragma unroll
          for (int k = 0; k < GG::E; ++k) x[k] = sub_mod(barrett_reduce_64(x[k], m), half_l, T.q);
          fwd_butterflies<GG::ST, GG::R, kG>(x, G.high, T);
          group_store<LOGN, 0>(bufB, G, x);
        }
        compute_sync();
      }
      if constexpr (NP >= 3) fwd_pass_smem<LOGN, 1, kG>(bufB, T);
      if constexpr (NP >= 4) fwd_pass_smem<LOGN, 2, kG>(bufB, T);
      {
        using GG = Geo<LOGN, NP - 1>;
#pragma unroll 1
        for (int j = 0; j < GG::PER_THREAD; ++j) {
          const GG G(tid + j * kThreads);
          uint64_t x[GG::E];
          group_load<LOGN, NP - 1>(bufB, G, x);
          fwd_butterflies<GG::ST, GG::R, kG>(x, G.high, T);
          const int64_t r = r_first + G.poly;
          const int64_t rr = r < a.rows ? r : a.rows - 1;
          const uint64_t* cj = a.ct + ((size_t)rr * a.lvl + l) * N + G.coef;
          uint64_t* o = a.out + ((size_t)rr * last + l) * N + G.coef;
#pragma unroll
          for (int v = 0; v < GG::E / 4; ++v) {
            uint64_t c[4], res[4];
            ldg256(cj + 4 * v, c);
#pragma unroll
            for (int k = 0; k < 4; ++k)
              res[k] = mul_shoup(sub_mod(c[k], full_reduce(x[4 * v + k], T), T.q), a.inv[l], a.inv_p[l], T.q);
            if (r < a.rows) stg256(o + 4 * v, res[0], res[1], res[2], res[3]);
          }
        }
        compute_sync();
      }
    }
  }
}

// ---- key switch ------------------------------------------------------------------------------
struct KsArgs {
  const uint64_t* coef;   // [C][lvl][N]  d2 in coefficient form
  const uint64_t* evk;    // [E][2][Ltab][N]; entries of source limb i start at first[i]
  uint64_t* acc;          // [C][2][lvl][N]: (d0, d1) on entry, (d0 + r0, d1 + r1) on exit
  const uint64_t* tw2;
  const uint64_t* consts;
  int lvl, Ltab, digit_bits;
  int ndig[16], first[16];
  int64_t C;
};

template <int LOGN>
__global__ void __launch_bounds__(kThreads, 1) keyswitch2_kernel(KsArgs a) {
  constexpr int NP = num_passes(LOGN);
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  constexpr int N = 1 << LOGN;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t bufW = smem_u32(smem), bufR0 = bufW + unit_bytes(LOGN), bufR1 = bufR0 + unit_bytes(LOGN);
  const int tid = threadIdx.x;
  const int64_t groups = (a.C + POLYS - 1) / POLYS;
  const int64_t units = groups * a.lvl;
  const uint64_t mask = a.digit_bits >= 64 ? ~0ull : ((1ull << a.digit_bits) - 1);
  using GL = Geo<LOGN, NP - 1>;   // geometry of the accumulators: the last pass (contiguous per thread)
  for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
    const int jl = (int)(u % a.lvl);            // target limb
    const int64_t c_first = (u / a.lvl) * POLYS;
    const Limb T = limb_global(a.tw2, a.consts, jl, 0, N);
    const Modulus m{T.q, a.consts[jl * 8 + 1], a.consts[jl * 8 + 2]};
    // accumulators start from (d0, d1)
#pragma unroll 1
    for (int j = 0; j < GL::PER_THREAD; ++j) {
      const GL G(tid + j * kThreads);
      int64_t c = c_first + G.poly;
      if (c >= a.C) c = a.C - 1;
      uint64_t x[GL::E];
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const uint64_t* src = a.acc + ((size_t)(c * 2 + b) * a.lvl + jl) * N + G.coef;
#pragma unroll
        for (int v = 0; v < GL::E / 4; ++v) {
          uint64_t t[4];
          ldg256(src + 4 * v, t);
#pragma unroll
          for (int k = 0; k < 4; ++k) x[4 * v + k] = t[k];
        }
        group_store<LOGN, NP - 1>(b == 0 ? bufR0 : bufR1, G, x);
      }
    }
    for (int i = 0; i < a.lvl; ++i) {
      for (int kd = 0; kd < a.ndig[i]; ++kd) {
        const int shift = kd * a.digit_bits;
        const uint64_t* ek0 = a.evk + ((size_t)((a.first[i] + kd) * 2 + 0) * a.Ltab + jl) * N;
        const uint64_t* ek1 = a.evk + ((size_t)((a.first[i] + kd) * 2 + 1) * a.Ltab + jl) * N;
        {
          using GG = Geo<LOGN, 0>;
#pragma unroll 1
          for (int j = 0; j < GG::PER_THREAD; ++j) {
            const GG G(tid + j * kThreads);
            int64_t c = c_first + G.poly;
            if (c >= a.C) c = a.C - 1;
            const uint64_t* src = a.coef + ((size_t)c * a.lvl + i) * N + G.coef;
            uint64_t x[GG::E];
#pragma unroll
            for (int k = 0; k < GG::E; ++k) x[k] = (src[(size_t)k << GG::TL] >> shift) & mask;
            fwd_butterflies<GG::ST, GG::R, kG>(x, G.high, T);
            group_store<LOGN, 0>(bufW, G, x);
          }
          compute_sync();
        }
        if constexpr (NP >= 3) fwd_pass_smem<LOGN, 1, kG>(bufW, T);
        if constexpr (NP >= 4) fwd_pass_smem<LOGN, 2, kG>(bufW, T);
#pragma unroll 1
        for (int j = 0; j < GL::PER_THREAD; ++j) {
          const GL G(tid + j * kThreads);
          uint64_t x[GL::E], r[GL::E];
          group_load<LOGN, NP - 1>(bufW, G, x);
          fwd_butterflies<GL::ST, GL::R, kG>(x, G.high, T);
#pragma unroll
          for (int k = 0; k < GL::E; ++k) x[k] = full_reduce(x[k], T);
#pragma unroll
          for (int b = 0; b < 2; ++b) {
            const uint32_t bufR = b == 0 ? bufR0 : bufR1;
            const uint64_t* ek = (b == 0 ? ek0 : ek1) + G.coef;
            group_load<LOGN, NP - 1>(bufR, G, r);
#pragma unroll
            for (int v = 0; v < GL::E / 4; ++v) {
              uint64_t kk[4];
              ldg256(ek + 4 * v, kk);
#pragma unroll
              for (int k = 0; k < 4; ++k) r[4 * v + k] = mad_mod(x[4 * v + k], kk[k], r[4 * v + k], m);
            }
            group_store<LOGN, NP - 1>(bufR, G, r);
          }
        }
        compute_sync();
      }
    }
    // write (d0 + r0, d1 + r1) back
#pragma unroll 1
    for (int j = 0; j < GL::PER_THREAD; ++j) {
      const GL G(tid + j * kThreads);
      const int64_t c = c_first + G.poly;
      uint64_t x[GL::E];
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        group_load<LOGN, NP - 1>(b == 0 ? bufR0 : bufR1, G, x);
        if (c < a.C) {
          uint64_t* dst = a.acc + ((size_t)(c * 2 + b) * a.lvl + jl) * N + G.coef;
#pragma unroll
          for (int v = 0; v < GL::E / 4; ++v) stg256(dst + 4 * v, x[4 * v], x[4 * v + 1], x[4 * v + 2], x[4 * v + 3]);
        }
      }
    }
    compute_sync();
  }
}

// ---- tensor product --------------------------------------------------------------------------
__global__ void tensor3_kernel(const uint64_t* __restrict__ A, const uint64_t* __restrict__ B, uint64_t* __restrict__ d01,
                               uint64_t* __restrict__ d2, int64_t C, int lvl, int n, const uint64_t* __restrict__ consts) {
  const int64_t row = blockIdx.y;            // (c, limb)
  const int64_t c = row / lvl;
  const int l = (int)(row % lvl);
  const uint64_t* cc = consts + (size_t)l * 8;
  const Modulus m{cc[0], cc[1], cc[2]};
  const uint64_t* a0 = A + ((size_t)(c * 2 + 0) * lvl + l) * n;
  const uint64_t* a1 = A + ((size_t)(c * 2 + 1) * lvl + l) * n;
  const uint64_t* b0 = B + ((size_t)(c * 2 + 0) * lvl + l) * n;
  const uint64_t* b1 = B + ((size_t)(c * 2 + 1) * lvl + l) * n;
  uint64_t* o0 = d01 + ((size_t)(c * 2 + 0) * lvl + l) * n;
  uint64_t* o1 = d01 + ((size_t)(c * 2 + 1) * lvl + l) * n;
  uint64_t* o2 = d2 + ((size_t)c * lvl + l) * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t x0 = a0[i], x1 = a1[i], y0 = b0[i], y1 = b1[i];
    o0[i] = mul_mod(x0, y0, m);
    o1[i] = mad_mod(x0, y1, mul_mod(x1, y0, m), m);
    o2[i] = mul_mod(x1, y1, m);
  }
}

template <int LOGN>
bool launch_rescale(const RescaleArgs& a, int qbits, cudaStream_t st) {
  constexpr int NP = num_passes(LOGN);
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  const int smem = 2 * unit_bytes(LOGN);
  const int64_t units = (a.rows + POLYS - 1) / POLYS;
  const int grid = (int)std::min<int64_t>(units, device_sm_count());
  const unsigned corr = pick_corr<LOGN>(qbits);
  auto go = [&](auto k) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    k<<<grid, kThreads, smem, st>>>(a);
  };
  if (corr == 0u) go(rescale2_kernel<LOGN, 0u>);
  else if (corr == (1u << 1)) go(rescale2_kernel<LOGN, 1u << 1>);
  else if (corr == ((1u << (NP - 1)) - 1u)) go(rescale2_kernel<LOGN, (1u << (NP - 1)) - 1u>);
  else return false;
  return true;
}

template <int LOGN>
void launch_keyswitch(const KsArgs& a, cudaStream_t st) {
  constexpr int POLYS = (1 << unit_log(LOGN)) >> LOGN;
  const int smem = 3 * unit_bytes(LOGN);
  const int64_t units = ((a.C + POLYS - 1) / POLYS) * a.lvl;
  const int grid = (int)std::min<int64_t>(units, device_sm_count());
  auto k = keyswitch2_kernel<LOGN>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  k<<<grid, kThreads, smem, st>>>(a);
}

}  // namespace

bool rescale2(const uint64_t* ct, uint64_t* out, int64_t C, int lvl, int logn, const uint64_t* tw2, const uint64_t* consts,
              const uint64_t* inv, const uint64_t* inv_p, int qbits, cudaStream_t st) {
  if (C == 0) return true;
  if (logn < 10 || logn > 13 || qbits > 58 || lvl < 2 || lvl > 16) return false;
  RescaleArgs a{};
  a.ct = ct; a.out = out; a.tw2 = tw2; a.consts = consts; a.lvl = lvl; a.rows = C * 2;
  for (int l = 0; l < lvl - 1; ++l) { a.inv[l] = inv[l]; a.inv_p[l] = inv_p[l]; }
  bool ok = false;
  switch (logn) {
    case 10: ok = launch_rescale<10>(a, qbits, st); break;
    case 11: ok = launch_rescale<11>(a, qbits, st); break;
    case 12: ok = launch_rescale<12>(a, qbits, st); break;
    case 13: ok = launch_rescale<13>(a, qbits, st); break;
  }
  if (ok) note_launch();
  return ok;
}

bool keyswitch2(const uint64_t* coef, const uint64_t* evk, uint64_t* acc, int64_t C, int lvl, int Ltab, int logn,
                int digit_bits, const int* ndig, const int* first, const uint64_t* tw2, const uint64_t* consts, int qbits,
                cudaStream_t st) {
  if (C == 0) return true;
  if (logn < 10 || logn > 13 || qbits > 58 || lvl > 16) return false;
  KsArgs a{};
  a.coef = coef; a.evk = evk; a.acc = acc; a.tw2 = tw2; a.consts = consts;
  a.lvl = lvl; a.Ltab = Ltab; a.digit_bits = digit_bits; a.C = C;
  for (int i = 0; i < lvl; ++i) { a.ndig[i] = ndig[i]; a.first[i] = first[i]; }
  switch (logn) {
    case 10: launch_keyswitch<10>(a, st); break;
    case 11: launch_keyswitch<11>(a, st); break;
    case 12: launch_keyswitch<12>(a, st); break;
    case 13: launch_keyswitch<13>(a, st); break;
  }
  note_launch();
  return true;
}

void ct_tensor(const uint64_t* A, const uint64_t* B, uint64_t* d01, uint64_t* d2, int64_t C, int lvl, int n,
               const uint64_t* consts, cudaStream_t st) {
  if (C == 0) return;
  dim3 grid((n + 1023) / 1024, (unsigned)(C * lvl));
  tensor3_kernel<<<grid, 256, 0, st>>>(A, B, d01, d2, C, lvl, n, consts);
  note_launch();
}

}  // namespace cuda
}  // namespace hefl
