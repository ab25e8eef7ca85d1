// Second-generation negacyclic NTT device routines for sm_90a (SURVEY.md K3, K4).
//
// What changed against ntt.cuh (which stays as the path for N = 32768 and primes >= 2^58):
//
//  * the ring degree is a template parameter, so every stride, twiddle index and shared-memory
//    offset of a pass is an immediate;
//  * twiddles and their Shoup companions are interleaved (w, w') pairs that live in shared
//    memory: a TMA tensor copy with the 128-byte swizzle brings the first 4096 pairs of the
//    limb's table in ONCE per persistent CTA, multicast to the two CTAs of a cluster (both work
//    on the same limb); a butterfly fetches its twiddle with one LDS.128 instead of two __ldg;
//  * coefficient buffers use the same 128-byte swizzle (chunk ^= row & 7), which is what both
//    the TMA engine writes and what makes every pass -- including the unit-stride one, where a
//    thread owns 64 or 128 contiguous bytes -- free of bank conflicts without padding words;
//  * no conditional correction inside the forward butterfly: with q < 2^58 the lazy values
//    grow by 2q per stage and stay below 2^64 for all log2(N) <= 15 stages; the inverse
//    (Gentleman-Sande) doubles per stage and is corrected at pass boundaries chosen at
//    compile time from the head-room of the modulus;
//  * 512 threads x 16 coefficients per pass, radix-16 / radix-8 in registers: 3 passes for
//    N = 4096, 4 for N = 8192 / 16384.
//
// A "unit" is 8192 coefficients (16384 for N = 16384): 8192/N whole polynomials of the same
// limb processed together by one CTA.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../common/hopper.cuh"
#include "../modarith.h"

namespace hefl {
namespace dev2 {

constexpr int kThreads = 512;
constexpr int kTwLog = 12;  // twiddle pairs [0, 4096) are resident in shared memory

__host__ __device__ constexpr int unit_log(int logn) { return logn < 13 ? 13 : logn; }
__host__ __device__ constexpr int num_passes(int logn) { return logn <= 12 ? 3 : 4; }
// radix (log2) of forward pass p
__host__ __device__ constexpr int radix(int logn, int p) {
  return logn == 10   ? (p == 0 ? 4 : 3)    // 4,3,3
         : logn == 11 ? (p <= 1 ? 4 : 3)    // 4,4,3
         : logn == 12 ? 4                   // 4,4,4
         : logn == 13 ? (p == 0 ? 4 : 3)    // 4,3,3,3
                      : (p <= 1 ? 4 : 3);   // 14: 4,4,3,3
}
__host__ __device__ constexpr int stage0(int logn, int p) {
  int s = 0;
  for (int i = 0; i < p; ++i) s += radix(logn, i);
  return s;
}
__host__ __device__ constexpr int tw_rows(int logn) { return ((1 << (logn < kTwLog ? logn : kTwLog)) * 16) / 128; }
__host__ __device__ constexpr int tw_bytes(int logn) { return tw_rows(logn) * 128; }
__host__ __device__ constexpr int unit_bytes(int logn) { return (1 << unit_log(logn)) * 8; }

// byte offset inside a 1024-byte-aligned buffer -> swizzled byte offset (TMA SWIZZLE_128B)
__device__ __forceinline__ uint32_t swz(uint32_t o) { return o ^ ((o >> 3) & 0x70u); }

__device__ __forceinline__ uint64_t lds64(uint32_t a) {
  uint64_t v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts64(uint32_t a, uint64_t v) {
  asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory");
}
__device__ __forceinline__ void lds128(uint32_t a, uint64_t& x, uint64_t& y) {
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "r"(a));
}
__device__ __forceinline__ void sts128(uint32_t a, uint64_t x, uint64_t y) {
  asm volatile("st.shared.v2.u64 [%0], {%1, %2};" ::"r"(a), "l"(x), "l"(y) : "memory");
}
__device__ __forceinline__ void ldg128(const uint64_t* p, uint64_t& x, uint64_t& y) {
  asm volatile("ld.global.nc.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "l"(p));
}
// 32 bytes of global memory as two 16-byte accesses (sm_90 has no 256-bit ld/st.global)
__device__ __forceinline__ void ldg256(const uint64_t* p, uint64_t (&v)[4]) {
  ldg128(p, v[0], v[1]);
  ldg128(p + 2, v[2], v[3]);
}
__device__ __forceinline__ void stg256(uint64_t* p, uint64_t a, uint64_t b, uint64_t c, uint64_t d) {
  asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
  asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p + 2), "l"(c), "l"(d) : "memory");
}

// Per-limb state of a persistent CTA.
struct Limb {
  uint32_t tw;           // shared-memory address of the resident twiddle pairs (swizzled)
  const uint64_t* twg;   // the same table in global memory ([N][2]); used for indices >= 4096
  uint64_t q, two_q;
  uint64_t rhi;          // floor(2^64 / q): Shoup companion of 1
  uint64_t ninv, ninv_p;
};

// G = true: every stage reads the table from global memory (kernels that walk over several limbs per
// CTA -- rescale, key switch -- have no room for one resident table per limb; the tables stay in L2).
template <int STAGE, bool G = false>
__device__ __forceinline__ void tw_pair(const Limb& T, uint32_t ti, uint64_t& w, uint64_t& wp) {
  if constexpr (STAGE < kTwLog && !G) {
    lds128(T.tw + swz(ti << 4), w, wp);
  } else {
    ldg128(T.twg + 2 * (size_t)ti, w, wp);
  }
}

// x in [0, 2^64) -> [0, 2q), same residue
__device__ __forceinline__ uint64_t lazy_reduce(uint64_t x, const Limb& T) {
  return x - mul_hi(x, T.rhi) * T.q;
}
__device__ __forceinline__ uint64_t full_reduce(uint64_t x, const Limb& T) {
  uint64_t r = lazy_reduce(x, T);
  return r >= T.q ? r - T.q : r;
}

// R forward (Cooley-Tukey) stages ST .. ST+R-1 on the 2^R values of one group held in registers.
// `high` is the group's index above the stride (its twiddle selector). No correction: inputs
// below B*q give outputs below (B + 2R)*q.
template <int ST, int R, bool G = false>
__device__ __forceinline__ void fwd_butterflies(uint64_t (&x)[1 << R], uint32_t high, const Limb& T) {
  constexpr int E = 1 << R;
  const uint32_t idx0 = (1u << ST) + high;
#pragma unroll
  for (int u = 0; u < R; ++u) {
    const int half = E >> (u + 1);
#pragma unroll
    for (int k = 0; k < E; ++k) {
      if ((k & half) == 0) {
        uint64_t W, Wp;
        const uint32_t ti = (idx0 << u) + (uint32_t)(k >> (R - u));
        // the stage is ST + u: a compile-time value once the loop is unrolled
        if (ST + u < kTwLog) tw_pair<0, G>(T, ti, W, Wp); else tw_pair<kTwLog, G>(T, ti, W, Wp);
        const uint64_t Q = mul_shoup_lazy(x[k + half], W, Wp, T.q);
        const uint64_t X = x[k];
        x[k] = X + Q;
        x[k + half] = X + (T.two_q - Q);
      }
    }
  }
}

// R inverse (Gentleman-Sande) stages ST+R-1 .. ST. `bound` (compile time, in units of q) bounds
// the inputs; outputs are below bound * 2^R * q. Twiddles are the inverse table (same indexing).
template <int ST, int R, int BOUND, bool G = false>
__device__ __forceinline__ void inv_butterflies(uint64_t (&x)[1 << R], uint32_t high, const Limb& T) {
  constexpr int E = 1 << R;
  const uint32_t idx0 = (1u << ST) + high;
#pragma unroll
  for (int u = R - 1; u >= 0; --u) {
    const int half = E >> (u + 1);
    // inputs of this step are below (BOUND << (R-1-u)) * q
    const uint64_t bq = (uint64_t)(BOUND << (R - 1 - u)) * T.q;
#pragma unroll
    for (int k = 0; k < E; ++k) {
      if ((k & half) == 0) {
        uint64_t W, Wp;
        const uint32_t ti = (idx0 << u) + (uint32_t)(k >> (R - u));
        if (ST + u < kTwLog) tw_pair<0, G>(T, ti, W, Wp); else tw_pair<kTwLog, G>(T, ti, W, Wp);
        const uint64_t U = x[k], V = x[k + half];
        x[k] = U + V;
        x[k + half] = mul_shoup_lazy(U + (bq - V), W, Wp, T.q);
      }
    }
  }
}

// Geometry of group g (0 .. unit/2^R - 1) of pass P: which polynomial of the unit, the
// twiddle selector, and the unit-relative index of its first coefficient.
template <int LOGN, int P>
struct Geo {
  static constexpr int R = radix(LOGN, P);
  static constexpr int ST = stage0(LOGN, P);
  static constexpr int TL = LOGN - ST - R;   // log2 of the coefficient stride inside a group
  static constexpr int E = 1 << R;
  static constexpr int GROUPS = (1 << unit_log(LOGN)) >> R;
  static constexpr int PER_THREAD = GROUPS / kThreads;
  uint32_t poly, high, base, coef;           // coef: index of element 0 inside its polynomial
  __device__ __forceinline__ explicit Geo(uint32_t g) {
    const uint32_t gl = g & ((1u << (LOGN - R)) - 1);
    poly = g >> (LOGN - R);
    const uint32_t low = gl & ((1u << TL) - 1);
    high = gl >> TL;
    coef = (high << (TL + R)) + low;
    base = (poly << LOGN) + coef;
  }
};

// Load / store the 2^R values of a group from / to a swizzled unit buffer.
template <int LOGN, int P>
__device__ __forceinline__ void group_load(uint32_t buf, const Geo<LOGN, P>& G, uint64_t (&x)[1 << radix(LOGN, P)]) {
  using GG = Geo<LOGN, P>;
  if constexpr (GG::TL == 0) {
    // 2^R contiguous coefficients: 64 or 128 bytes inside one 128-byte row
    const uint32_t row = (G.base * 8u) & ~127u;
    const uint32_t c0 = ((G.base * 8u) >> 4) & 7u;     // first 16-byte chunk (0 or 4 for R = 3)
    const uint32_t rs = (row >> 7) & 7u;
#pragma unroll
    for (int c = 0; c < GG::E / 2; ++c) lds128(buf + row + (((c0 + c) ^ rs) << 4), x[2 * c], x[2 * c + 1]);
  } else {
#pragma unroll
    for (int k = 0; k < GG::E; ++k) x[k] = lds64(buf + swz((G.base + ((uint32_t)k << GG::TL)) * 8u));
  }
}
template <int LOGN, int P>
__device__ __forceinline__ void group_store(uint32_t buf, const Geo<LOGN, P>& G, const uint64_t (&x)[1 << radix(LOGN, P)]) {
  using GG = Geo<LOGN, P>;
  if constexpr (GG::TL == 0) {
    const uint32_t row = (G.base * 8u) & ~127u;
    const uint32_t c0 = ((G.base * 8u) >> 4) & 7u;
    const uint32_t rs = (row >> 7) & 7u;
#pragma unroll
    for (int c = 0; c < GG::E / 2; ++c) sts128(buf + row + (((c0 + c) ^ rs) << 4), x[2 * c], x[2 * c + 1]);
  } else {
#pragma unroll
    for (int k = 0; k < GG::E; ++k) sts64(buf + swz((G.base + ((uint32_t)k << GG::TL)) * 8u), x[k]);
  }
}

// Barrier over the 512 compute threads (kernels may carry an extra producer warp).
__device__ __forceinline__ void compute_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory"); }

// One in-place shared-memory forward pass over the whole unit. Ends with a compute barrier.
template <int LOGN, int P, bool TG = false>
__device__ __forceinline__ void fwd_pass_smem(uint32_t buf, const Limb& T) {
  using GG = Geo<LOGN, P>;
#pragma unroll 1
  for (int j = 0; j < GG::PER_THREAD; ++j) {
    const GG G(threadIdx.x + j * kThreads);
    uint64_t x[GG::E];
    group_load<LOGN, P>(buf, G, x);
    fwd_butterflies<GG::ST, GG::R, TG>(x, G.high, T);
    group_store<LOGN, P>(buf, G, x);
  }
  compute_sync();
}

// Bound (units of q) of the inverse values entering forward-numbered pass P when the inverse
// transform starts from values below B0*q and corrects to 2q before every pass in CORR (bit p).
template <int LOGN>
__host__ __device__ constexpr int inv_bound_in(int P, int B0, unsigned corr) {
  int b = B0;
  for (int p = num_passes(LOGN) - 1; p > P; --p) {
    if (corr & (1u << p)) b = 2;
    b <<= radix(LOGN, p);
  }
  if (corr & (1u << P)) b = 2;
  return b;
}

template <int LOGN, int P, int B0, unsigned CORR, bool TG = false>
__device__ __forceinline__ void inv_pass_smem(uint32_t buf, const Limb& T) {
  using GG = Geo<LOGN, P>;
  constexpr int BIN = inv_bound_in<LOGN>(P, B0, CORR);
#pragma unroll 1
  for (int j = 0; j < GG::PER_THREAD; ++j) {
    const GG G(threadIdx.x + j * kThreads);
    uint64_t x[GG::E];
    group_load<LOGN, P>(buf, G, x);
    if constexpr ((CORR >> P) & 1u) {
#pragma unroll
      for (int k = 0; k < GG::E; ++k) x[k] = lazy_reduce(x[k], T);
    }
    inv_butterflies<GG::ST, GG::R, BIN, TG>(x, G.high, T);
    group_store<LOGN, P>(buf, G, x);
  }
  compute_sync();
}

// Largest value bound (units of q) the inverse transform reaches; the caller picks CORR so that
// 2 * this * q < 2^64.
template <int LOGN>
__host__ __device__ constexpr int inv_bound_max(int B0, unsigned corr) {
  int worst = B0;
  for (int p = num_passes(LOGN) - 1; p >= 0; --p) {
    const int b = inv_bound_in<LOGN>(p, B0, corr) << radix(LOGN, p);
    if (b > worst) worst = b;
  }
  return worst;
}

// Cheapest inverse-correction schedule (bit p = reduce to [0, 2q) before pass p) whose largest intermediate,
// inv_bound_max * q from inputs below 4q, stays below 2^64 for primes of `qbits` bits; ~0u when none does. The
// inverse kernels are instantiated for these three schedules.
template <int LOGN>
unsigned pick_corr(int qbits) {
  constexpr int NP = num_passes(LOGN);
  const unsigned cands[3] = {0u, 1u << 1, (1u << (NP - 1)) - 1u};
  for (const unsigned corr : cands) {
    const long long worst = inv_bound_max<LOGN>(4, corr);
    int wb = 0;
    while ((1ll << wb) < worst) ++wb;
    if (wb + qbits <= 63) return corr;
  }
  return ~0u;
}

}  // namespace dev2
}  // namespace hefl
