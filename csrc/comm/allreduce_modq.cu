// Fused ciphertext all-reduce: coefficient-wise sum over ranks *modulo each RNS prime*,
// performed inside one kernel that reads/writes peer GPUs' memory over NVLink/NVSwitch.
// No NCCL call on this path (SURVEY.md §2.4 K1, §5.8; replaces the file-drop aggregation
// loop FLPyfhelin.py:372-381).
//
// Buffer layout on every rank: [C][2][L][N] u64 residues (< q_l < 2^61), symmetric address
// space (peer r's buffer is mapped at bufs[r]). Three algorithms:
//   two_shot  : rank r owns chunk r. It pulls chunk r from all P peers with 32-byte loads
//               (two 16-byte loads each, two per peer in flight), adds, reduces mod q_l in registers
//               and pushes the result into chunk r of all P buffers (in place). With a key
//               holder, that rank owns no chunk: it never reads un-aggregated ciphertext.
//   one_shot  : every rank pulls everything and writes a private output (latency-optimal for
//               small messages).
//   multimem  : as two_shot but the P-way add is done by the NVSwitch
//               (multimem.ld_reduce.add.u64) and the result is broadcast with multimem.st.
// Cross-GPU synchronisation uses per-block flags in a symmetric signal pad with
// release/acquire CAS at system scope; flags return to 0 so no reset/epoch is needed.
// All spins are bounded: on timeout the kernel records a diagnostic in `status` and exits
// (failure detection, SURVEY.md §5.3).
#include <cstdint>
#include <cuda_runtime.h>

#include "../he/kernels.h"
#include "../he/modarith.h"
#include "../he/philox.h"
#include "comm.h"

namespace hefl {
namespace comm {

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint32_t cas_release_sys(uint32_t* addr, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.global.release.sys.cas.b32 %0, [%1], %2, %3;"
               : "=r"(old) : "l"(addr), "r"(cmp), "r"(val) : "memory");
  return old;
}
__device__ __forceinline__ uint32_t cas_acquire_sys(uint32_t* addr, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], %2, %3;"
               : "=r"(old) : "l"(addr), "r"(cmp), "r"(val) : "memory");
  return old;
}

// Returns false on timeout.
__device__ __forceinline__ bool put_signal(uint32_t* addr, uint64_t deadline) {
  uint32_t spins = 0;
  while (cas_release_sys(addr, 0u, 1u) != 0u) {
    if ((++spins & 0x3FFu) == 0 && globaltimer_ns() > deadline) return false;
  }
  return true;
}
__device__ __forceinline__ bool wait_signal(uint32_t* addr, uint64_t deadline) {
  uint32_t spins = 0;
  while (cas_acquire_sys(addr, 1u, 0u) != 1u) {
    if ((++spins & 0x3FFu) == 0 && globaltimer_ns() > deadline) return false;
  }
  return true;
}

// Block-level barrier across ranks: block b of every rank meets block b of every other rank.
// slot selects one of two flag banks so consecutive barriers in one kernel never alias.
__device__ __forceinline__ bool block_barrier(const AllReduceArgs& a, int slot, uint64_t deadline) {
  __shared__ int ok_flag;
  if (threadIdx.x == 0) ok_flag = 1;
  __syncthreads();
  if (threadIdx.x < (unsigned)a.world) {
    const int peer = threadIdx.x;
    const size_t base = ((size_t)slot * gridDim.x + blockIdx.x) * a.world;
    bool ok = put_signal(a.sigs[peer] + base + a.rank, deadline);
    ok = ok && wait_signal(a.sigs[a.rank] + base + peer, deadline);
    if (!ok) {
      ok_flag = 0;
      if (a.status) atomicExch(a.status, 1u + (uint32_t)peer + ((uint32_t)slot << 8) + ((uint32_t)blockIdx.x << 16));
    }
  }
  __syncthreads();
  return ok_flag != 0;
}

// 32-byte peer accesses as two 16-byte ld/st.global.v2.u64 (sm_90 has no 256-bit global accesses). Relaxed at system scope: ordering
// against the other GPUs comes from the release/acquire flag barriers around the data phase.
struct U64x4 {
  uint64_t v[4];
};
__device__ __forceinline__ U64x4 ld32(const uint64_t* p) {
  U64x4 r;
  asm volatile("ld.global.relaxed.sys.v2.u64 {%0, %1}, [%2];" : "=l"(r.v[0]), "=l"(r.v[1]) : "l"(p) : "memory");
  asm volatile("ld.global.relaxed.sys.v2.u64 {%0, %1}, [%2];" : "=l"(r.v[2]), "=l"(r.v[3]) : "l"(p + 2) : "memory");
  return r;
}
__device__ __forceinline__ void st32(uint64_t* p, const U64x4& r) {
  asm volatile("st.global.relaxed.sys.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(r.v[0]), "l"(r.v[1]) : "memory");
  asm volatile("st.global.relaxed.sys.v2.u64 [%0], {%1, %2};" ::"l"(p + 2), "l"(r.v[2]), "l"(r.v[3]) : "memory");
}
__device__ __forceinline__ uint64_t mm_ld_add(const uint64_t* mc) {
  uint64_t v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.u64 %0, [%1];" : "=l"(v) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void mm_st(uint64_t* mc, uint64_t v) {
  asm volatile("multimem.st.relaxed.sys.global.u64 [%0], %1;" :: "l"(mc), "l"(v) : "memory");
}

__device__ __forceinline__ uint64_t mod_sum(uint64_t s, uint64_t q, uint64_t ratio_hi) {
  const uint64_t qhat = __umul64hi(s, ratio_hi);
  uint64_t r = s - qhat * q;
  if (r >= q) r -= q;
  if (r >= q) r -= q;
  return r;
}

// Work is cut into "quads" of 4 words (32 bytes). A quad never straddles a limb (N >= 1024),
// so q is fetched once per quad.
// Quads per thread per step in the P2P algorithms: U * P * 32 bytes in flight per thread. What matters is the
// number of REMOTE loads in flight per SM (peer latency is ~2.5 us): with two ranks a thread has one remote
// load per quad, with eight it has seven, so U shrinks as the world grows (and the registers stay <= 64 words).
constexpr int kMmUnroll = 2;    // quads per thread per step for multimem: 8 independent ld_reduce in flight

template <int ALGO, int kUnroll>  // ALGO: 0 two_shot, 1 one_shot, 2 multimem
__global__ void __launch_bounds__(512)
allreduce_modq_kernel(const __grid_constant__ AllReduceArgs a) {
  const uint64_t deadline = globaltimer_ns() + a.timeout_ns;
  if (!block_barrier(a, 0, deadline)) return;

  const int P = a.world;
  const int64_t quads = a.numel >> 2;
  int64_t lo = 0, hi = quads;
  if (ALGO != 1) {
    // Chunk ownership. With a key holder (a.no_owner >= 0) that rank owns nothing: it never
    // loads a peer's un-aggregated ciphertext, it only receives finished sums.
    const int owners = a.no_owner >= 0 ? P - 1 : P;
    const int me = a.no_owner >= 0 ? (a.rank == a.no_owner ? -1 : a.rank - (a.rank > a.no_owner ? 1 : 0)) : a.rank;
    if (me < 0) {
      lo = hi = 0;
    } else {
      const int64_t per = (quads + owners - 1) / owners;
      lo = per * me;
      hi = lo + per < quads ? lo + per : quads;
      if (lo > quads) lo = quads;
    }
  }
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
  const int logn = a.logn;
  uint32_t peer_loads = 0;

  if (ALGO == 2) {
    for (int64_t i0 = lo + tid; i0 < hi; i0 += nthreads * kMmUnroll) {
      uint64_t acc[kMmUnroll][4];
#pragma unroll
      for (int u = 0; u < kMmUnroll; ++u) {
        const int64_t i = i0 + u * nthreads;
        if (i < hi) {
          const uint64_t* mc = a.mc + (i << 2);
#pragma unroll
          for (int k = 0; k < 4; ++k) acc[u][k] = mm_ld_add(mc + k);
          ++peer_loads;
        }
      }
#pragma unroll
      for (int u = 0; u < kMmUnroll; ++u) {
        const int64_t i = i0 + u * nthreads;
        if (i < hi) {
          const int l = (int)(((i << 2) >> logn) % a.L);
          const uint64_t q = a.q[l], rh = a.ratio_hi[l];
          uint64_t* mc = a.mc + (i << 2);
#pragma unroll
          for (int k = 0; k < 4; ++k) mm_st(mc + k, mod_sum(acc[u][k], q, rh));
        }
      }
    }
  } else {
    for (int64_t i0 = lo + tid; i0 < hi; i0 += nthreads * kUnroll) {
      constexpr int kPeers = kMaxWorld / kUnroll;       // this instantiation serves worlds up to kPeers
      U64x4 v[kUnroll][kPeers];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t i = i0 + u * nthreads;
        if (i < hi) {
#pragma unroll
          for (int p = 0; p < kPeers; ++p)
            if (p < P) v[u][p] = ld32(a.bufs[(a.rank + p) % P] + (i << 2));  // stagger peers across ranks
          ++peer_loads;
        }
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t i = i0 + u * nthreads;
        if (i < hi) {
          const int l = (int)(((i << 2) >> logn) % a.L);
          const uint64_t q = a.q[l], rh = a.ratio_hi[l];
          U64x4 acc = v[u][0];
#pragma unroll
          for (int p = 1; p < kPeers; ++p)
            if (p < P) {
#pragma unroll
              for (int k = 0; k < 4; ++k) acc.v[k] += v[u][p].v[k];
            }
#pragma unroll
          for (int k = 0; k < 4; ++k) acc.v[k] = mod_sum(acc.v[k], q, rh);
          if (ALGO == 1) {
            st32(a.out + (i << 2), acc);
          } else {
#pragma unroll
            for (int p = 0; p < kMaxWorld; ++p)
              if (p < P) st32(a.bufs[(a.rank + p) % P] + (i << 2), acc);
          }
        }
      }
    }
  }
  if (a.stats && peer_loads) atomicAdd(a.stats, peer_loads);
  // make this block's peer stores visible before signalling completion
  __threadfence_system();
  block_barrier(a, 1, deadline);
}

template <int ALGO, int U>
static void launch_allreduce_u(const AllReduceArgs& args, int blocks, int threads, cudaStream_t st) {
  // Even grids go out as clusters of two CTAs: a cluster takes both SMs of a TPC, so a small grid (the
  // SM-partitioned pipeline gives the collective ~24 SMs) does not leave half-used TPCs that the cluster
  // kernels of encrypt / decrypt could no longer be placed on.
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3((unsigned)threads);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (blocks % 2 == 0) ? 2 : 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, allreduce_modq_kernel<ALGO, U>, args);
}

template <int ALGO>
static void launch_allreduce(const AllReduceArgs& args, int blocks, int threads, cudaStream_t st) {
  if (ALGO == 2 || args.world > 4) launch_allreduce_u<ALGO, 1>(args, blocks, threads, st);
  else if (args.world > 2) launch_allreduce_u<ALGO, 2>(args, blocks, threads, st);
  else launch_allreduce_u<ALGO, 4>(args, blocks, threads, st);
}

void allreduce_modq(const AllReduceArgs& args, int algo, int blocks, int threads, cudaStream_t st) {
  switch (algo) {
    case 0: launch_allreduce<0>(args, blocks, threads, st); break;
    case 1: launch_allreduce<1>(args, blocks, threads, st); break;
    default: launch_allreduce<2>(args, blocks, threads, st); break;
  }
  hefl::cuda::note_launch();
}

// Pairwise additive masks (secure-aggregation style): for every peer j the word w of this rank's
// ciphertext gets +PRG(seed_ij, w) if sign_j > 0 and -PRG(seed_ij, w) if sign_j < 0, modulo the
// limb prime. Rank i uses sign(+) for j > i and (-) for j < i with the SAME pair seed, so the masks
// cancel in the sum over ranks while every individual buffer is uniformly random to anybody who
// does not hold all of that rank's pair seeds. One Philox call yields the masks of two words.
__global__ void __launch_bounds__(256)
pairwise_mask_kernel(uint64_t* __restrict__ data, int64_t numel, int L, int logn, MaskArgs m) {
  const int64_t pairs = numel >> 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = i << 1;
    const int l = (int)((e >> logn) % L);
    const Modulus mod{m.q[l], m.ratio_lo[l], m.ratio_hi[l]};
    ulonglong2 v = *reinterpret_cast<ulonglong2*>(data + e);
    for (int j = 0; j < m.npeers; ++j) {
      const Philox4 r = philox4x32_10((uint32_t)i, (uint32_t)(i >> 32), m.round, 9u, (uint32_t)m.seed[j],
                                      (uint32_t)(m.seed[j] >> 32));
      const uint64_t a0 = barrett_reduce_64(((uint64_t)r.x << 32) | r.y, mod);
      const uint64_t a1 = barrett_reduce_64(((uint64_t)r.z << 32) | r.w, mod);
      if (m.sign[j] > 0) {
        v.x = add_mod(v.x, a0, mod.q);
        v.y = add_mod(v.y, a1, mod.q);
      } else {
        v.x = sub_mod(v.x, a0, mod.q);
        v.y = sub_mod(v.y, a1, mod.q);
      }
    }
    *reinterpret_cast<ulonglong2*>(data + e) = v;
  }
}

void pairwise_mask(uint64_t* data, int64_t numel, int L, int logn, const MaskArgs& m, cudaStream_t st) {
  if (numel == 0 || m.npeers == 0) return;
  int blocks = (int)(((numel >> 1) + 255) / 256);
  if (blocks > hefl::cuda::device_sm_count() * 8) blocks = hefl::cuda::device_sm_count() * 8;
  pairwise_mask_kernel<<<blocks, 256, 0, st>>>(data, numel, L, logn, m);
  hefl::cuda::note_launch();
}

// Local K-way modular sum of K buffers living on ONE device (loopback transport on a single
// GPU, and the aggregation step of the file-based compat path). The accumulator is reduced after
// every 7 addends: a reduced accumulator (< q) plus 7 residues stays <= 8 (q - 1) < 2^64 for q <= 2^61,
// while plus 8 residues it can exceed 2^64 under a 61-bit prime.
__global__ void local_sum_modq_kernel(const uint64_t* const* __restrict__ srcs, int K,
                                      uint64_t* __restrict__ out, int64_t numel, int logn, int L,
                                      const uint64_t* __restrict__ consts) {
  const int64_t pairs = numel >> 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < pairs;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = i << 1;
    const int l = (int)((e >> logn) % L);
    const uint64_t q = consts[l * 8], rh = consts[l * 8 + 2];
    ulonglong2 acc = make_ulonglong2(0, 0);
    for (int k = 0; k < K; ++k) {
      const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(srcs[k] + e);
      acc.x += v.x;
      acc.y += v.y;
      if (k % 7 == 6) { acc.x = mod_sum(acc.x, q, rh); acc.y = mod_sum(acc.y, q, rh); }
    }
    acc.x = mod_sum(acc.x, q, rh);
    acc.y = mod_sum(acc.y, q, rh);
    *reinterpret_cast<ulonglong2*>(out + e) = acc;
  }
}

void local_sum_modq(const uint64_t* const* srcs_dev, int K, uint64_t* out, int64_t numel, int logn,
                    int L, const uint64_t* consts, cudaStream_t st) {
  int blocks = (int)(((numel >> 1) + 255) / 256);
  if (blocks > hefl::cuda::device_sm_count() * 8) blocks = hefl::cuda::device_sm_count() * 8;
  if (blocks < 1) blocks = 1;
  local_sum_modq_kernel<<<blocks, 256, 0, st>>>(srcs_dev, K, out, numel, logn, L, consts);
  hefl::cuda::note_launch();
}

}  // namespace comm
}  // namespace hefl
