// Shared-memory negacyclic NTT / INTT device routines for sm_90a (SURVEY.md K3, K4).
//
// One CTA transforms one contiguous block of 2^logb coefficients held in shared
// memory (the whole polynomial when logb == logn; N = 32768 is split into two
// 16384 blocks after one global-memory stage). Butterflies are Harvey lazy
// (values kept in [0,4q) forward, [0,2q) inverse) with Shoup twiddles, and up to
// three stages are merged per pass in registers (radix-8) so a 4096-point
// transform needs 4 block-wide barriers instead of 12.
//
// The routines are __device__ functions (not kernels) so that encrypt/decrypt
// fuse sampling, NTT and the public/secret-key multiply-add into one launch.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../modarith.h"

namespace hefl {
namespace dev {

// One padding word every 16 coefficients keeps the stride-1 radix-8 pass free of
// shared-memory bank conflicts (8 consecutive u64 per thread).
__device__ __forceinline__ int pad_idx(int i) { return i + (i >> 4); }
__host__ __device__ constexpr int padded_len(int n) { return n + (n >> 4); }

struct LimbTables {
  const uint64_t* w;    // psi powers, bit-reversed
  const uint64_t* wp;   // Shoup companions
  const uint64_t* iw;   // inverse psi powers, bit-reversed
  const uint64_t* iwp;
  uint64_t q, ratio_lo, ratio_hi, ninv, ninv_p;
};

__device__ __forceinline__ LimbTables load_limb(const uint64_t* tables, const uint64_t* consts,
                                                int l, int n) {
  LimbTables t;
  const uint64_t* base = tables + (size_t)l * 4 * n;
  t.w = base;
  t.wp = base + n;
  t.iw = base + 2 * n;
  t.iwp = base + 3 * n;
  const uint64_t* c = consts + (size_t)l * 8;
  t.q = c[0];
  t.ratio_lo = c[1];
  t.ratio_hi = c[2];
  t.ninv = c[3];
  t.ninv_p = c[4];
  return t;
}

// ---- generic radix-2^R pass over an indexable buffer --------------------------------------
// `Idx` maps a logical coefficient index to a storage index (padded shared memory or
// identity for global memory). `jg_base` is the global coefficient index of local index 0.

struct PadIdx {
  __device__ __forceinline__ int operator()(int i) const { return pad_idx(i); }
};
struct IdIdx {
  __device__ __forceinline__ int operator()(int i) const { return i; }
};

template <int R, class Idx>
__device__ __forceinline__ void fwd_pass(uint64_t* buf, int logn, int logb, int jg_base, int stage0,
                                         const LimbTables& T, int tid, int nthreads, Idx idx) {
  constexpr int E = 1 << R;
  const int tl = logn - stage0 - R;  // log2 of the element stride inside a group
  const int groups = (1 << logb) >> R;
  const uint64_t q = T.q, two_q = 2 * T.q;
  for (int g = tid; g < groups; g += nthreads) {
    const int low = g & ((1 << tl) - 1);
    const int high = g >> tl;
    const int base = (high << (tl + R)) + low;
    uint64_t x[E];
#pragma unroll
    for (int k = 0; k < E; ++k) x[k] = buf[idx(base + (k << tl))];
    const int idx0 = (1 << stage0) + ((jg_base + base) >> (logn - stage0));
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const int half = E >> (u + 1);
#pragma unroll
      for (int k = 0; k < E; ++k) {
        if ((k & half) == 0) {
          const int ti = (idx0 << u) + (k >> (R - u));
          const uint64_t W = __ldg(T.w + ti), Wp = __ldg(T.wp + ti);
          uint64_t X = x[k];
          if (X >= two_q) X -= two_q;
          const uint64_t Q = mul_shoup_lazy(x[k + half], W, Wp, q);
          x[k] = X + Q;
          x[k + half] = X - Q + two_q;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < E; ++k) buf[idx(base + (k << tl))] = x[k];
  }
}

template <int R, class Idx>
__device__ __forceinline__ void inv_pass(uint64_t* buf, int logn, int logb, int jg_base, int stage0,
                                         const LimbTables& T, int tid, int nthreads, Idx idx) {
  constexpr int E = 1 << R;
  const int tl = logn - stage0 - R;
  const int groups = (1 << logb) >> R;
  const uint64_t q = T.q, two_q = 2 * T.q;
  for (int g = tid; g < groups; g += nthreads) {
    const int low = g & ((1 << tl) - 1);
    const int high = g >> tl;
    const int base = (high << (tl + R)) + low;
    uint64_t x[E];
#pragma unroll
    for (int k = 0; k < E; ++k) x[k] = buf[idx(base + (k << tl))];
    const int idx0 = (1 << stage0) + ((jg_base + base) >> (logn - stage0));
#pragma unroll
    for (int u = R - 1; u >= 0; --u) {
      const int half = E >> (u + 1);
#pragma unroll
      for (int k = 0; k < E; ++k) {
        if ((k & half) == 0) {
          const int ti = (idx0 << u) + (k >> (R - u));
          const uint64_t W = __ldg(T.iw + ti), Wp = __ldg(T.iwp + ti);
          const uint64_t U = x[k], V = x[k + half];
          uint64_t s = U + V;
          if (s >= two_q) s -= two_q;
          x[k] = s;
          x[k + half] = mul_shoup_lazy(U - V + two_q, W, Wp, q);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < E; ++k) buf[idx(base + (k << tl))] = x[k];
  }
}

// Forward NTT of the block [blk*2^logb, (blk+1)*2^logb) held in padded shared memory.
// Input values < 4q (lazy); output values < 4q (caller reduces). Ends with __syncthreads().
__device__ __forceinline__ void ntt_fwd_block(uint64_t* s, int logn, int logb, int blk,
                                              const LimbTables& T) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int jg = blk << logb;
  int st = logn - logb;
  __syncthreads();
  while (logn - st >= 3) {
    fwd_pass<3>(s, logn, logb, jg, st, T, tid, nt, PadIdx());
    st += 3;
    __syncthreads();
  }
  if (logn - st == 2) {
    fwd_pass<2>(s, logn, logb, jg, st, T, tid, nt, PadIdx());
    __syncthreads();
  } else if (logn - st == 1) {
    fwd_pass<1>(s, logn, logb, jg, st, T, tid, nt, PadIdx());
    __syncthreads();
  }
}

// Inverse of ntt_fwd_block: undoes stages logn-1 .. logn-logb. Input < 2q, output < 2q,
// NOT yet scaled by N^-1 (caller folds that into its write-out).
__device__ __forceinline__ void ntt_inv_block(uint64_t* s, int logn, int logb, int blk,
                                              const LimbTables& T) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int jg = blk << logb;
  const int rem = logb % 3;
  int st = logn - rem;
  __syncthreads();
  if (rem == 2) {
    inv_pass<2>(s, logn, logb, jg, st, T, tid, nt, PadIdx());
    __syncthreads();
  } else if (rem == 1) {
    inv_pass<1>(s, logn, logb, jg, st, T, tid, nt, PadIdx());
    __syncthreads();
  }
  while (st - 3 >= logn - logb) {
    st -= 3;
    inv_pass<3>(s, logn, logb, jg, st, T, tid, nt, PadIdx());
    __syncthreads();
  }
}

__device__ __forceinline__ uint64_t reduce_4q(uint64_t x, uint64_t q) {
  if (x >= 2 * q) x -= 2 * q;
  if (x >= q) x -= q;
  return x;
}

}  // namespace dev
}  // namespace hefl
