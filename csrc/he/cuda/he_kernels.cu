// sm_90a HE kernels: NTT/INTT, pointwise modular ops, CKKS encode/decode (special FFT),
// fused public-key encrypt, fused decrypt, CRT centring, BFV fractional codec.
// SURVEY.md §2.4 K3-K9, K11. Every kernel has a CPU twin in ../host_math.cpp and is
// tested bit-exact (integer kernels) or to 1 ulp-of-rounding (FFT) against it.
#include <atomic>
#include <cstdio>

#include "../kernels.h"
#include "../philox.h"
#include <stdexcept>
#include <string>

#include "ntt.cuh"

namespace hefl {
namespace cuda {

int device_sm_count() {
  static int counts[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!counts[dev]) cudaDeviceGetAttribute(&counts[dev], cudaDevAttrMultiProcessorCount, dev);
  return counts[dev];
}

static std::atomic<uint64_t> g_launches{0};
uint64_t launch_count() { return g_launches.load(); }
// Called by every host launcher right after its launch(es): counts our kernels (bench.py gpu_launches) and
// turns a failed launch (bad configuration, missing sm_90a image, sticky asynchronous error) into an exception
// instead of a silent no-op — the ops must fail loudly.
void note_launch(uint64_t n) {
  g_launches.fetch_add(n);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    throw std::runtime_error(std::string("hefl: CUDA kernel launch failed: ") + cudaGetErrorName(e) + " (" +
                             cudaGetErrorString(e) + ")");
}

using namespace hefl::dev;

static inline int ntt_threads(int logb) {
  int t = (1 << logb) >> 3;
  if (t > 1024) t = 1024;
  if (t < 32) t = 32;
  return t;
}
static inline size_t ntt_smem_bytes(int logb) { return (size_t)padded_len(1 << logb) * 8; }
// Largest block that fits one CTA's shared memory (227 KB): 16384 coefficients.
static inline int block_log(int logn) { return logn > 14 ? 14 : logn; }

template <class K>
static void set_smem(K kernel, size_t bytes) {
  static thread_local size_t configured = 0;
  (void)configured;
  if (bytes > 48 * 1024)
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

// ------------------------------------------------------------------------------------------
// NTT kernels
// ------------------------------------------------------------------------------------------

template <bool INVERSE, bool SCALE>
__global__ void __launch_bounds__(1024)
ntt_block_kernel(uint64_t* __restrict__ data, int L, int logn, int logb,
                 const uint64_t* __restrict__ tables, const uint64_t* __restrict__ consts) {
  extern __shared__ uint64_t smem[];
  const int nblk_log = logn - logb;
  const int row = blockIdx.x >> nblk_log;
  const int blk = blockIdx.x & ((1 << nblk_log) - 1);
  const int n = 1 << logn, nb = 1 << logb;
  const LimbTables T = load_limb(tables, consts, row % L, n);
  uint64_t* g = data + (size_t)row * n + ((size_t)blk << logb);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) smem[pad_idx(i)] = g[i];
  if (!INVERSE) {
    ntt_fwd_block(smem, logn, logb, blk, T);
    for (int i = threadIdx.x; i < nb; i += blockDim.x) g[i] = reduce_4q(smem[pad_idx(i)], T.q);
  } else {
    ntt_inv_block(smem, logn, logb, blk, T);
    for (int i = threadIdx.x; i < nb; i += blockDim.x) {
      uint64_t x = smem[pad_idx(i)];
      if (SCALE) x = mul_shoup(x, T.ninv, T.ninv_p, T.q);
      g[i] = x;  // when !SCALE the value stays lazy (< 2q) for the global stages
    }
  }
}

// First (forward) or last (inverse) R = logn - logb stages straight on global memory.
template <int R, bool INVERSE>
__global__ void ntt_global_kernel(uint64_t* __restrict__ data, int L, int logn,
                                  const uint64_t* __restrict__ tables,
                                  const uint64_t* __restrict__ consts) {
  const int n = 1 << logn;
  const int row = blockIdx.y;
  const LimbTables T = load_limb(tables, consts, row % L, n);
  uint64_t* g = data + (size_t)row * n;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nt = gridDim.x * blockDim.x;
  if (!INVERSE) {
    fwd_pass<R>(g, logn, logn, 0, 0, T, tid, nt, IdIdx());
  } else {
    inv_pass<R>(g, logn, logn, 0, 0, T, tid, nt, IdIdx());
  }
}

__global__ void scale_ninv_kernel(uint64_t* __restrict__ data, int L, int n,
                                  const uint64_t* __restrict__ consts) {
  const int row = blockIdx.y;
  const uint64_t* c = consts + (size_t)(row % L) * 8;
  const uint64_t q = c[0], ninv = c[3], ninv_p = c[4];
  uint64_t* g = data + (size_t)row * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    g[i] = mul_shoup(g[i], ninv, ninv_p, q);
}

__global__ void reduce4q_kernel(uint64_t* __restrict__ data, int L, int n,
                                const uint64_t* __restrict__ consts) {
  const int row = blockIdx.y;
  const uint64_t q = consts[(size_t)(row % L) * 8];
  uint64_t* g = data + (size_t)row * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    g[i] = reduce_4q(g[i], q);
}

void ntt(uint64_t* data, int64_t rows, int L, int logn, const uint64_t* tables,
         const uint64_t* consts, bool inverse, cudaStream_t st) {
  if (rows == 0) return;
  const int logb = block_log(logn);
  const int nblk = 1 << (logn - logb);
  const int threads = ntt_threads(logb);
  const size_t smem = ntt_smem_bytes(logb);
  const int n = 1 << logn;
  if (logb == logn) {
    if (!inverse) {
      set_smem(ntt_block_kernel<false, false>, smem);
      ntt_block_kernel<false, false><<<(unsigned)rows, threads, smem, st>>>(data, L, logn, logb, tables, consts);
    } else {
      set_smem(ntt_block_kernel<true, true>, smem);
      ntt_block_kernel<true, true><<<(unsigned)rows, threads, smem, st>>>(data, L, logn, logb, tables, consts);
    }
    note_launch();
    return;
  }
  // N = 32768: one global radix-2 stage + two 16384-point shared-memory blocks.
  const int R = logn - logb;  // == 1 with the current block_log
  dim3 ggrid((n >> R) / 256, (unsigned)rows);
  dim3 egrid(n / 1024, (unsigned)rows);
  if (!inverse) {
    if (R == 1) ntt_global_kernel<1, false><<<ggrid, 256, 0, st>>>(data, L, logn, tables, consts);
    set_smem(ntt_block_kernel<false, false>, smem);
    // values are lazy (< 4q) after the global stage; the block kernel accepts that
    ntt_block_kernel<false, false><<<(unsigned)(rows * nblk), threads, smem, st>>>(data, L, logn, logb, tables, consts);
    note_launch(2);
  } else {
    set_smem(ntt_block_kernel<true, false>, smem);
    ntt_block_kernel<true, false><<<(unsigned)(rows * nblk), threads, smem, st>>>(data, L, logn, logb, tables, consts);
    if (R == 1) ntt_global_kernel<1, true><<<ggrid, 256, 0, st>>>(data, L, logn, tables, consts);
    scale_ninv_kernel<<<egrid, 256, 0, st>>>(data, L, n, consts);
    note_launch(3);
  }
  (void)reduce4q_kernel;
}

// ------------------------------------------------------------------------------------------
// Pointwise modular ops
// ------------------------------------------------------------------------------------------

__global__ void pointwise_kernel(uint64_t* __restrict__ out, const uint64_t* __restrict__ a,
                                 const uint64_t* __restrict__ b, int64_t brows, int L, int n,
                                 const uint64_t* __restrict__ consts, int op) {
  const int64_t row = blockIdx.y;
  const int l = (int)(row % L);
  const uint64_t* c = consts + (size_t)l * 8;
  const Modulus m{c[0], c[1], c[2]};
  const uint64_t* ar = a + row * n;
  const uint64_t* br = (op == 4 || op == 5) ? nullptr : b + (row % brows) * n;
  uint64_t* o = out + row * n;
  const uint64_t scalar = op == 5 ? b[l] : 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    uint64_t r;
    switch (op) {
      case 0: r = add_mod(ar[i], br[i], m.q); break;
      case 1: r = sub_mod(ar[i], br[i], m.q); break;
      case 2: r = mul_mod(ar[i], br[i], m); break;
      case 3: r = mad_mod(ar[i], br[i], o[i], m); break;
      case 4: r = neg_mod(ar[i], m.q); break;
      default: r = mul_mod(ar[i], scalar, m); break;
    }
    o[i] = r;
  }
}

void pointwise(uint64_t* out, const uint64_t* a, const uint64_t* b, int64_t rows, int64_t brows,
               int L, int n, const uint64_t* consts, int op, cudaStream_t st) {
  if (rows == 0) return;
  dim3 grid((n + 1023) / 1024, (unsigned)rows);
  pointwise_kernel<<<grid, 256, 0, st>>>(out, a, b, brows, L, n, consts, op);
  note_launch();
}

__global__ void reduce_mod_kernel(uint64_t* __restrict__ data, int L, int n,
                                  const uint64_t* __restrict__ consts) {
  const int64_t row = blockIdx.y;
  const uint64_t* c = consts + (size_t)(row % L) * 8;
  const Modulus m{c[0], c[1], c[2]};
  ulonglong2* g = reinterpret_cast<ulonglong2*>(data + row * n);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n / 2; i += gridDim.x * blockDim.x) {
    ulonglong2 v = g[i];
    v.x = barrett_reduce_64(v.x, m);
    v.y = barrett_reduce_64(v.y, m);
    g[i] = v;
  }
}

void reduce_mod(uint64_t* data, int64_t rows, int L, int n, const uint64_t* consts,
                cudaStream_t st) {
  if (rows == 0) return;
  dim3 grid((n / 2 + 255) / 256, (unsigned)rows);
  reduce_mod_kernel<<<grid, 256, 0, st>>>(data, L, n, consts);
  note_launch();
}

// ------------------------------------------------------------------------------------------
// CKKS special FFT (fp64). One CTA per ciphertext; N/2 complex points in shared memory
// (N <= 16384) or in a global scratch row (N = 32768).
// ------------------------------------------------------------------------------------------

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__device__ void fft_special_inv_dev(double2* v, int lognh, int m, const int32_t* __restrict__ rot,
                                    const double2* __restrict__ ksi) {
  const int nh = 1 << lognh;
  for (int ll = lognh; ll >= 1; --ll) {  // len = 1 << ll
    const int lh = ll - 1;
    const int lenq = 4 << ll;
    const int gap = m / lenq;
    for (int b = threadIdx.x; b < nh / 2; b += blockDim.x) {
      const int j = b & ((1 << lh) - 1);
      const int i = (b >> lh) << ll;
      const int idx = (lenq - (rot[j] & (lenq - 1))) * gap;
      const double2 x = v[i + j], y = v[i + j + (1 << lh)];
      const double2 u = make_double2(x.x + y.x, x.y + y.y);
      const double2 w = cmul(make_double2(x.x - y.x, x.y - y.y), ksi[idx]);
      v[i + j] = u;
      v[i + j + (1 << lh)] = w;
    }
    __syncthreads();
  }
}

__device__ void fft_special_dev(double2* v, int lognh, int m, const int32_t* __restrict__ rot,
                                const double2* __restrict__ ksi) {
  const int nh = 1 << lognh;
  for (int ll = 1; ll <= lognh; ++ll) {
    const int lh = ll - 1;
    const int lenq = 4 << ll;
    const int gap = m / lenq;
    for (int b = threadIdx.x; b < nh / 2; b += blockDim.x) {
      const int j = b & ((1 << lh) - 1);
      const int i = (b >> lh) << ll;
      const int idx = (rot[j] & (lenq - 1)) * gap;
      const double2 u = v[i + j];
      const double2 w = cmul(v[i + j + (1 << lh)], ksi[idx]);
      v[i + j] = make_double2(u.x + w.x, u.y + w.y);
      v[i + j + (1 << lh)] = make_double2(u.x - w.x, u.y - w.y);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024)
ckks_encode_kernel(const float* __restrict__ vf, const double* __restrict__ vd, int64_t nvals,
                   int logn, double scale, const int32_t* __restrict__ rot,
                   const double2* __restrict__ ksi, int64_t* __restrict__ msg,
                   double2* __restrict__ scratch) {
  extern __shared__ double2 fsm[];
  const int n = 1 << logn, nh = n >> 1, lognh = logn - 1;
  const int64_t c = blockIdx.x;
  double2* v = scratch ? scratch + c * nh : fsm;
  for (int i = threadIdx.x; i < nh; i += blockDim.x) {
    const int64_t g = c * nh + i;
    double x = 0.0;
    if (g < nvals) x = vf ? (double)vf[g] : vd[g];
    v[i] = make_double2(x, 0.0);
  }
  __syncthreads();
  fft_special_inv_dev(v, lognh, 2 * n, rot, ksi);
  const double s = scale / (double)nh;
  int64_t* o = msg + c * n;
  for (int i = threadIdx.x; i < nh; i += blockDim.x) {
    const int r = (int)(__brev((unsigned)i) >> (32 - lognh));
    const double2 w = v[i];
    o[r] = __double2ll_rn(w.x * s);
    o[r + nh] = __double2ll_rn(w.y * s);
  }
}

static inline int fft_threads(int logn) {
  int t = (1 << logn) >> 2;
  if (t > 1024) t = 1024;
  if (t < 32) t = 32;
  return t;
}

void ckks_encode(const float* vals_f32, const double* vals_f64, int64_t C, int64_t nvals_total,
                 int logn, double scale, const int32_t* rot_group, const double* ksi, int64_t* msg,
                 double* scratch, cudaStream_t st) {
  if (C == 0) return;
  const size_t smem = logn <= 14 ? (size_t)(1 << (logn - 1)) * 16 : 0;
  set_smem(ckks_encode_kernel, smem);
  ckks_encode_kernel<<<(unsigned)C, fft_threads(logn), smem, st>>>(
      vals_f32, vals_f64, nvals_total, logn, scale, rot_group,
      reinterpret_cast<const double2*>(ksi), msg,
      logn <= 14 ? nullptr : reinterpret_cast<double2*>(scratch));
  note_launch();
}

struct CrtParams {
  uint64_t q0, q1, q1_ratio_lo, q1_ratio_hi, q0_inv_q1;
  int k;
};

__device__ __forceinline__ double crt_center_one(uint64_t x0, uint64_t x1, const CrtParams& p) {
  if (p.k == 1) return x0 > p.q0 / 2 ? -(double)(p.q0 - x0) : (double)x0;
  const Modulus m1{p.q1, p.q1_ratio_lo, p.q1_ratio_hi};
  const uint64_t x0r = barrett_reduce_64(x0, m1);
  const uint64_t d = mul_mod(sub_mod(x1, x0r, p.q1), p.q0_inv_q1, m1);
  // x = x0 + q0*d  in [0, q0*q1)
  uint64_t hi, lo;
  mul_wide(p.q0, d, hi, lo);
  uint64_t xl = lo + x0;
  uint64_t xh = hi + (xl < lo ? 1 : 0);
  uint64_t Qh, Ql;
  mul_wide(p.q0, p.q1, Qh, Ql);
  // half = Q >> 1
  const uint64_t hh = Qh >> 1, hl = (Ql >> 1) | (Qh << 63);
  const bool neg = xh > hh || (xh == hh && xl > hl);
  if (neg) {  // x = Q - x
    const uint64_t nl = Ql - xl;
    const uint64_t nh = Qh - xh - (Ql < xl ? 1 : 0);
    return -((double)nh * 18446744073709551616.0 + (double)nl);
  }
  return (double)xh * 18446744073709551616.0 + (double)xl;
}

__global__ void crt_center_kernel(const uint64_t* __restrict__ res, int64_t C, int n, CrtParams p,
                                  double* __restrict__ out) {
  const int64_t total = C * n;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total;
       g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = g / n, i = g % n;
    const uint64_t x0 = res[(c * p.k) * n + i];
    const uint64_t x1 = p.k > 1 ? res[(c * p.k + 1) * n + i] : 0;
    out[g] = crt_center_one(x0, x1, p);
  }
}

void crt_center(const uint64_t* res, int64_t C, int k, int n, uint64_t q0, uint64_t q1,
                uint64_t q1_ratio_lo, uint64_t q1_ratio_hi, uint64_t q0_inv_q1, double* out,
                cudaStream_t st) {
  if (C == 0) return;
  CrtParams p{q0, q1, q1_ratio_lo, q1_ratio_hi, q0_inv_q1, k};
  const int64_t total = C * n;
  int blocks = (int)((total + 255) / 256);
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  crt_center_kernel<<<blocks, 256, 0, st>>>(res, C, n, p, out);
  note_launch();
}

// One server-optimizer step on a decoded average a (fp64) at flat index g (DESIGN.md §8). fp32 throughout
// after d = (float)(a - x); __fmul_rn / __fadd_rn keep nvcc from contracting into FMAs, so the step rounds
// exactly like its host twin (host::ckks_decode_server_step). sqrtf and '/' are IEEE (no fast-math).
template <int OPT>
__device__ __forceinline__ float server_step_one(double a, int64_t g, const ServerStep& s) {
  if (g >= s.n_trainable) return (float)a;              // BatchNorm running statistics: plain FedAvg
  const float x = s.x_t[g];
  const float d = (float)(a - (double)x);
  float m = s.m[g];
  if (OPT == kFedAvgM) {
    m = __fadd_rn(__fmul_rn(s.beta1, m), d);
    s.m[g] = m;
    return __fadd_rn(x, __fmul_rn(s.lr, m));
  }
  m = __fadd_rn(__fmul_rn(s.beta1, m), __fmul_rn(__fsub_rn(1.0f, s.beta1), d));
  const float d2 = __fmul_rn(d, d);
  float v = s.v[g];
  if (OPT == kFedAdagrad) {
    v = __fadd_rn(v, d2);
  } else if (OPT == kFedYogi) {
    const float t = __fsub_rn(v, d2);
    const float sg = t > 0.0f ? 1.0f : (t < 0.0f ? -1.0f : 0.0f);
    v = __fsub_rn(v, __fmul_rn(__fmul_rn(__fsub_rn(1.0f, s.beta2), d2), sg));
  } else {                                              // kFedAdam
    v = __fadd_rn(__fmul_rn(s.beta2, v), __fmul_rn(__fsub_rn(1.0f, s.beta2), d2));
  }
  s.m[g] = m;
  s.v[g] = v;
  return __fadd_rn(x, __fdiv_rn(__fmul_rn(s.lr, m), __fadd_rn(__fsqrt_rn(v), s.tau)));
}

// Decode straight from decrypted residues: CRT centre -> /(scale*K) -> special FFT -> real part.
// OPT = 0 writes the average; OPT = 1..4 (FedAvgM, FedAdagrad, FedYogi, FedAdam) apply the server step to it
// in the same pass, so the average itself never goes to memory unless ServerStep::avg_* asks for it.
template <int OPT>
__device__ __forceinline__ void decode_res_body(const uint64_t* __restrict__ res, const double* __restrict__ coeffs,
                                                int logn, const CrtParams& p, double inv_scale,
                                                const int32_t* __restrict__ rot, const double2* __restrict__ ksi,
                                                float* __restrict__ out_f32, double* __restrict__ out_f64,
                                                int64_t nvals, double2* __restrict__ scratch, const ServerStep& sv) {
  extern __shared__ double2 fsm[];
  const int n = 1 << logn, nh = n >> 1, lognh = logn - 1;
  const int64_t c = blockIdx.x;
  double2* v = scratch ? scratch + c * nh : fsm;
  for (int i = threadIdx.x; i < nh; i += blockDim.x) {
    double re, im;
    if (res) {
      const uint64_t* r0 = res + (c * p.k) * n;
      const uint64_t* r1 = p.k > 1 ? r0 + n : r0;
      re = crt_center_one(r0[i], r1[i], p);
      im = crt_center_one(r0[i + nh], r1[i + nh], p);
    } else {
      re = coeffs[c * n + i];
      im = coeffs[c * n + i + nh];
    }
    const int r = (int)(__brev((unsigned)i) >> (32 - lognh));
    v[r] = make_double2(re * inv_scale, im * inv_scale);
  }
  __syncthreads();
  fft_special_dev(v, lognh, 2 * n, rot, ksi);
  if constexpr (OPT == 0) {
    for (int i = threadIdx.x; i < nh; i += blockDim.x) {
      const int64_t g = c * nh + i;
      if (g < nvals) {
        if (out_f32) out_f32[g] = (float)v[i].x;
        if (out_f64) out_f64[g] = v[i].x;
      }
    }
  } else {
    for (int i = threadIdx.x; i < nh; i += blockDim.x) {
      const int64_t g = c * nh + i;
      if (g < nvals) {
        const double a = v[i].x;
        const int64_t gg = sv.g0 + g;
        if (sv.avg_f32) sv.avg_f32[gg] = (float)a;
        if (sv.avg_f64) sv.avg_f64[gg] = a;
        sv.x_new[gg] = server_step_one<OPT>(a, gg, sv);
      }
    }
  }
}

__global__ void __launch_bounds__(1024)
ckks_decode_res_kernel(const uint64_t* __restrict__ res, const double* __restrict__ coeffs,
                       int logn, CrtParams p, double inv_scale, const int32_t* __restrict__ rot,
                       const double2* __restrict__ ksi, float* __restrict__ out_f32,
                       double* __restrict__ out_f64, int64_t nvals, double2* __restrict__ scratch) {
  decode_res_body<kFedAvg>(res, coeffs, logn, p, inv_scale, rot, ksi, out_f32, out_f64, nvals, scratch, ServerStep{});
}

// The decode with a server-optimizer step (OPT = 1..4) in its output loop.
template <int OPT>
__global__ void __launch_bounds__(1024)
ckks_decode_step_kernel(const uint64_t* __restrict__ res, int logn, CrtParams p, double inv_scale,
                        const int32_t* __restrict__ rot, const double2* __restrict__ ksi, int64_t nvals,
                        double2* __restrict__ scratch, ServerStep sv) {
  decode_res_body<OPT>(res, nullptr, logn, p, inv_scale, rot, ksi, nullptr, nullptr, nvals, scratch, sv);
}

void ckks_decode_residues(const uint64_t* res, int64_t C, int k, int logn, uint64_t q0, uint64_t q1,
                          uint64_t q1_ratio_lo, uint64_t q1_ratio_hi, uint64_t q0_inv_q1,
                          double inv_scale, const int32_t* rot_group, const double* ksi,
                          float* out, int64_t nvals_total, double* scratch, cudaStream_t st) {
  if (C == 0) return;
  CrtParams p{q0, q1, q1_ratio_lo, q1_ratio_hi, q0_inv_q1, k};
  const size_t smem = logn <= 14 ? (size_t)(1 << (logn - 1)) * 16 : 0;
  set_smem(ckks_decode_res_kernel, smem);
  ckks_decode_res_kernel<<<(unsigned)C, fft_threads(logn), smem, st>>>(
      res, nullptr, logn, p, inv_scale, rot_group, reinterpret_cast<const double2*>(ksi), out,
      nullptr, nvals_total, logn <= 14 ? nullptr : reinterpret_cast<double2*>(scratch));
  note_launch();
}

template <int OPT>
static void launch_decode_step(const uint64_t* res, int64_t C, int logn, const CrtParams& p, double inv_scale,
                               const int32_t* rot_group, const double* ksi, int64_t nvals, double* scratch,
                               const ServerStep& sv, cudaStream_t st) {
  const size_t smem = logn <= 14 ? (size_t)(1 << (logn - 1)) * 16 : 0;
  set_smem(ckks_decode_step_kernel<OPT>, smem);
  ckks_decode_step_kernel<OPT><<<(unsigned)C, fft_threads(logn), smem, st>>>(
      res, logn, p, inv_scale, rot_group, reinterpret_cast<const double2*>(ksi), nvals,
      logn <= 14 ? nullptr : reinterpret_cast<double2*>(scratch), sv);
}

void ckks_decode_server_step(const uint64_t* res, int64_t C, int k, int logn, uint64_t q0, uint64_t q1,
                             uint64_t q1_ratio_lo, uint64_t q1_ratio_hi, uint64_t q0_inv_q1,
                             double inv_scale, const int32_t* rot_group, const double* ksi,
                             int64_t nvals, const ServerStep& sv, int opt, double* scratch, cudaStream_t st) {
  if (C == 0) return;
  CrtParams p{q0, q1, q1_ratio_lo, q1_ratio_hi, q0_inv_q1, k};
  switch (opt) {
    case kFedAvgM: launch_decode_step<kFedAvgM>(res, C, logn, p, inv_scale, rot_group, ksi, nvals, scratch, sv, st); break;
    case kFedAdagrad: launch_decode_step<kFedAdagrad>(res, C, logn, p, inv_scale, rot_group, ksi, nvals, scratch, sv, st); break;
    case kFedYogi: launch_decode_step<kFedYogi>(res, C, logn, p, inv_scale, rot_group, ksi, nvals, scratch, sv, st); break;
    case kFedAdam: launch_decode_step<kFedAdam>(res, C, logn, p, inv_scale, rot_group, ksi, nvals, scratch, sv, st); break;
    default: throw std::invalid_argument("ckks_decode_server_step: opt must be 1..4, got " + std::to_string(opt));
  }
  note_launch();
}

void ckks_decode(const double* coeffs, int64_t C, int logn, double inv_scale,
                 const int32_t* rot_group, const double* ksi, float* out_f32, double* out_f64,
                 double* scratch, cudaStream_t st) {
  if (C == 0) return;
  CrtParams p{1, 1, 0, 0, 0, 1};
  const size_t smem = logn <= 14 ? (size_t)(1 << (logn - 1)) * 16 : 0;
  set_smem(ckks_decode_res_kernel, smem);
  ckks_decode_res_kernel<<<(unsigned)C, fft_threads(logn), smem, st>>>(
      nullptr, coeffs, logn, p, inv_scale, rot_group, reinterpret_cast<const double2*>(ksi),
      out_f32, out_f64, C * (int64_t)(1 << (logn - 1)),
      logn <= 14 ? nullptr : reinterpret_cast<double2*>(scratch));
  note_launch();
}

__global__ void coeff_encode_kernel(const float* __restrict__ vals, int64_t total, int64_t nvals,
                                    double scale, int64_t* __restrict__ msg) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total;
       g += (int64_t)gridDim.x * blockDim.x)
    msg[g] = g < nvals ? __double2ll_rn((double)vals[g] * scale) : 0;
}

void coeff_encode(const float* vals, int64_t C, int64_t nvals_total, int n, double scale,
                  int64_t* msg, cudaStream_t st) {
  if (C == 0) return;
  const int64_t total = C * n;
  int blocks = (int)((total + 255) / 256);
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  coeff_encode_kernel<<<blocks, 256, 0, st>>>(vals, total, nvals_total, scale, msg);
  note_launch();
}

// ------------------------------------------------------------------------------------------
// Fused public-key encryption (K6): sample -> NTT -> multiply-add with pk, one CTA per
// (ciphertext, limb). TWO_BUF keeps NTT(u) in a second shared buffer so each output word is
// written exactly once; for N = 16384 one buffer is used and the partial products make a
// round trip through L2. acc: ct = (ct + Enc(m)) mod q, the old word read where it is stored.
// ------------------------------------------------------------------------------------------

template <bool TWO_BUF>
__global__ void __launch_bounds__(1024)
encrypt_kernel(const int64_t* __restrict__ msg, const uint64_t* __restrict__ pk,
               uint64_t* __restrict__ ct, int L, int logn, const uint64_t* __restrict__ tables,
               const uint64_t* __restrict__ consts, const uint64_t* __restrict__ msg_scale,
               uint64_t seed, uint32_t ct_offset, bool acc) {
  extern __shared__ uint64_t smem[];
  const int n = 1 << logn;
  const int64_t c = blockIdx.x / L;
  const int l = blockIdx.x % L;
  const LimbTables T = load_limb(tables, consts, l, n);
  const Modulus m{T.q, T.ratio_lo, T.ratio_hi};
  uint64_t* bufA = smem;
  uint64_t* bufU = TWO_BUF ? smem + padded_len(n) : smem;
  const uint32_t cid = ct_offset + (uint32_t)c;
  uint64_t* c0 = ct + ((c * 2 + 0) * L + l) * n;
  uint64_t* c1 = ct + ((c * 2 + 1) * L + l) * n;
  const uint64_t* pk0 = pk + (size_t)(0 * L + l) * n;
  const uint64_t* pk1 = pk + (size_t)(1 * L + l) * n;
  const uint64_t sc = msg_scale ? msg_scale[l] : 1;

  // pass 1: u
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    bufU[pad_idx(i)] = lift_signed(sample_enc_noise(seed, cid, (uint32_t)i).u, T.q);
  }
  ntt_fwd_block(bufU, logn, logn, 0, T);
  if (!TWO_BUF) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const uint64_t uh = reduce_4q(bufU[pad_idx(i)], T.q);
      c0[i] = mad_mod(uh, pk0[i], acc ? c0[i] : 0, m);
      c1[i] = mad_mod(uh, pk1[i], acc ? c1[i] : 0, m);
    }
    __syncthreads();
  }
  // pass 2: e0 + scale*m
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    uint64_t mm = msg ? reduce_signed(msg[c * n + i], m) : 0;
    if (sc != 1) mm = mul_mod(mm, sc, m);
    bufA[pad_idx(i)] = add_mod(lift_signed(sample_enc_noise(seed, cid, (uint32_t)i).e0, T.q), mm, T.q);
  }
  ntt_fwd_block(bufA, logn, logn, 0, T);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t a = reduce_4q(bufA[pad_idx(i)], T.q);
    if (TWO_BUF) {
      const uint64_t uh = reduce_4q(bufU[pad_idx(i)], T.q);
      c0[i] = mad_mod(uh, pk0[i], acc ? add_mod(a, c0[i], T.q) : a, m);
    } else {
      c0[i] = add_mod(c0[i], a, T.q);
    }
  }
  __syncthreads();
  // pass 3: e1
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    bufA[pad_idx(i)] = lift_signed(sample_enc_noise(seed, cid, (uint32_t)i).e1, T.q);
  }
  ntt_fwd_block(bufA, logn, logn, 0, T);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t b = reduce_4q(bufA[pad_idx(i)], T.q);
    if (TWO_BUF) {
      const uint64_t uh = reduce_4q(bufU[pad_idx(i)], T.q);
      c1[i] = mad_mod(uh, pk1[i], acc ? add_mod(b, c1[i], T.q) : b, m);
    } else {
      c1[i] = add_mod(c1[i], b, T.q);
    }
  }
}

// Unfused pieces for N = 32768 (a polynomial does not fit one CTA).
__global__ void enc_sample_kernel(const int64_t* __restrict__ msg, uint64_t* __restrict__ u,
                                  uint64_t* __restrict__ a, uint64_t* __restrict__ b, int L, int n,
                                  const uint64_t* __restrict__ consts,
                                  const uint64_t* __restrict__ msg_scale, uint64_t seed,
                                  uint32_t ct_offset) {
  const int64_t c = blockIdx.y / L;
  const int l = blockIdx.y % L;
  const uint64_t* cc = consts + (size_t)l * 8;
  const Modulus m{cc[0], cc[1], cc[2]};
  const uint64_t sc = msg_scale ? msg_scale[l] : 1;
  const size_t row = (size_t)blockIdx.y * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const EncNoise z = sample_enc_noise(seed, ct_offset + (uint32_t)c, (uint32_t)i);
    u[row + i] = lift_signed(z.u, m.q);
    uint64_t mm = msg ? reduce_signed(msg[c * n + i], m) : 0;
    if (sc != 1) mm = mul_mod(mm, sc, m);
    a[row + i] = add_mod(lift_signed(z.e0, m.q), mm, m.q);
    b[row + i] = lift_signed(z.e1, m.q);
  }
}

__global__ void enc_combine_kernel(const uint64_t* __restrict__ u, const uint64_t* __restrict__ a,
                                   const uint64_t* __restrict__ b, const uint64_t* __restrict__ pk,
                                   uint64_t* __restrict__ ct, int L, int n,
                                   const uint64_t* __restrict__ consts, bool acc) {
  const int64_t c = blockIdx.y / L;
  const int l = blockIdx.y % L;
  const uint64_t* cc = consts + (size_t)l * 8;
  const Modulus m{cc[0], cc[1], cc[2]};
  const size_t row = (size_t)blockIdx.y * n;
  uint64_t* c0 = ct + ((c * 2 + 0) * L + l) * n;
  uint64_t* c1 = ct + ((c * 2 + 1) * L + l) * n;
  const uint64_t* pk0 = pk + (size_t)(0 * L + l) * n;
  const uint64_t* pk1 = pk + (size_t)(1 * L + l) * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t uh = u[row + i];
    c0[i] = mad_mod(uh, pk0[i], acc ? add_mod(a[row + i], c0[i], m.q) : a[row + i], m);
    c1[i] = mad_mod(uh, pk1[i], acc ? add_mod(b[row + i], c1[i], m.q) : b[row + i], m);
  }
}

void encrypt(const int64_t* msg, const uint64_t* pk, uint64_t* ct, int64_t C, int L, int logn,
             const uint64_t* tables, const uint64_t* consts, const uint64_t* msg_scale,
             uint64_t seed, uint32_t ct_offset, bool accumulate, cudaStream_t st) {
  if (C == 0) return;
  const int n = 1 << logn;
  if (logn <= 14) {
    const int threads = ntt_threads(logn);
    const bool two = logn <= 13;
    const size_t smem = ntt_smem_bytes(logn) * (two ? 2 : 1);
    if (two) {
      set_smem(encrypt_kernel<true>, smem);
      encrypt_kernel<true><<<(unsigned)(C * L), threads, smem, st>>>(msg, pk, ct, L, logn, tables, consts, msg_scale, seed,
                                                                     ct_offset, accumulate);
    } else {
      set_smem(encrypt_kernel<false>, smem);
      encrypt_kernel<false><<<(unsigned)(C * L), threads, smem, st>>>(msg, pk, ct, L, logn, tables, consts, msg_scale, seed,
                                                                      ct_offset, accumulate);
    }
    note_launch();
    return;
  }
  // Large-N path: scratch lives in a stream-ordered allocation.
  const size_t bytes = (size_t)C * L * n * 8;
  uint64_t *u, *a, *b;
  cudaMallocAsync(&u, bytes * 3, st);
  a = u + (size_t)C * L * n;
  b = a + (size_t)C * L * n;
  dim3 grid(n / 1024, (unsigned)(C * L));
  enc_sample_kernel<<<grid, 256, 0, st>>>(msg, u, a, b, L, n, consts, msg_scale, seed, ct_offset);
  note_launch();
  ntt(u, 3 * C * L, L, logn, tables, consts, false, st);  // rows keep (row % L) == limb
  enc_combine_kernel<<<grid, 256, 0, st>>>(u, a, b, pk, ct, L, n, consts, accumulate);
  note_launch();
  cudaFreeAsync(u, st);
}

// ------------------------------------------------------------------------------------------
// Fused decrypt (K7): (c0 + c1*s) -> INTT, one CTA per (ciphertext, limb < k).
// ------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(1024)
decrypt_kernel(const uint64_t* __restrict__ ct, const uint64_t* __restrict__ sk,
               uint64_t* __restrict__ out, int Lct, int k, int logn,
               const uint64_t* __restrict__ tables, const uint64_t* __restrict__ consts) {
  extern __shared__ uint64_t smem[];
  const int n = 1 << logn;
  const int64_t c = blockIdx.x / k;
  const int l = blockIdx.x % k;
  const LimbTables T = load_limb(tables, consts, l, n);
  const Modulus m{T.q, T.ratio_lo, T.ratio_hi};
  const uint64_t* c0 = ct + ((c * 2 + 0) * Lct + l) * n;
  const uint64_t* c1 = ct + ((c * 2 + 1) * Lct + l) * n;
  const uint64_t* s = sk + (size_t)l * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) smem[pad_idx(i)] = mad_mod(c1[i], s[i], c0[i], m);
  ntt_inv_block(smem, logn, logn, 0, T);
  uint64_t* o = out + (c * k + l) * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    o[i] = mul_shoup(smem[pad_idx(i)], T.ninv, T.ninv_p, T.q);
}

__global__ void dec_combine_kernel(const uint64_t* __restrict__ ct, const uint64_t* __restrict__ sk,
                                   uint64_t* __restrict__ out, int Lct, int k, int n,
                                   const uint64_t* __restrict__ consts) {
  const int64_t c = blockIdx.y / k;
  const int l = blockIdx.y % k;
  const uint64_t* cc = consts + (size_t)l * 8;
  const Modulus m{cc[0], cc[1], cc[2]};
  const uint64_t* c0 = ct + ((c * 2 + 0) * Lct + l) * n;
  const uint64_t* c1 = ct + ((c * 2 + 1) * Lct + l) * n;
  const uint64_t* s = sk + (size_t)l * n;
  uint64_t* o = out + (c * k + l) * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    o[i] = mad_mod(c1[i], s[i], c0[i], m);
}

void decrypt(const uint64_t* ct, const uint64_t* sk, uint64_t* out, int64_t C, int Lct, int k,
             int logn, const uint64_t* tables, const uint64_t* consts, cudaStream_t st) {
  if (C == 0) return;
  const int n = 1 << logn;
  if (logn <= 14) {
    const size_t smem = ntt_smem_bytes(logn);
    set_smem(decrypt_kernel, smem);
    decrypt_kernel<<<(unsigned)(C * k), ntt_threads(logn), smem, st>>>(ct, sk, out, Lct, k, logn, tables, consts);
    note_launch();
    return;
  }
  dim3 grid(n / 1024, (unsigned)(C * k));
  dec_combine_kernel<<<grid, 256, 0, st>>>(ct, sk, out, Lct, k, n, consts);
  note_launch();
  ntt(out, C * k, k, logn, tables, consts, true, st);
}

// ------------------------------------------------------------------------------------------
// BFV fractional codec (compat path, K11) and helpers
// ------------------------------------------------------------------------------------------

__global__ void frac_encode_kernel(const double* __restrict__ vals, int64_t C, int n,
                                   int int_digits, int frac_digits, int64_t* __restrict__ msg) {
  // one warp per scalar: zero the row, then lane 0 writes the (at most 96) digits
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  int64_t* o = msg + c * n;
  for (int i = lane; i < n; i += 32) o[i] = 0;
  __syncwarp();
  if (lane == 0) {
    double v = vals[c];
    const int sgn = v < 0 ? -1 : 1;
    v = fabs(v);
    double ip = floor(v);
    double fp = v - ip;
    for (int i = 0; i < int_digits && ip > 0; ++i) {
      const double half = floor(ip * 0.5);
      const int bit = (int)(ip - 2.0 * half);
      o[i] = sgn * bit;
      ip = half;
    }
    for (int i = 1; i <= frac_digits; ++i) {
      fp *= 2.0;
      const int bit = fp >= 1.0 ? 1 : 0;
      fp -= bit;
      o[n - i] = -sgn * bit;
    }
  }
}

void frac_encode(const double* vals, int64_t C, int n, int int_digits, int frac_digits,
                 int64_t* msg, cudaStream_t st) {
  if (C == 0) return;
  const int64_t threads = C * 32;
  frac_encode_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(vals, C, n, int_digits, frac_digits, msg);
  note_launch();
}

__global__ void frac_decode_kernel(const int64_t* __restrict__ coeffs, int64_t C, int n,
                                   int int_digits, int frac_digits, double* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int64_t* x = coeffs + c * n;
  double acc = 0.0, w = 1.0;
  for (int i = 0; i < int_digits; ++i) { acc += (double)x[i] * w; w *= 2.0; }
  w = 0.5;
  for (int i = 1; i <= frac_digits; ++i) { acc -= (double)x[n - i] * w; w *= 0.5; }
  out[c] = acc;
}

void frac_decode(const int64_t* coeffs, int64_t C, int n, int int_digits, int frac_digits,
                 double* out, cudaStream_t st) {
  if (C == 0) return;
  frac_decode_kernel<<<(unsigned)((C + 127) / 128), 128, 0, st>>>(coeffs, C, n, int_digits, frac_digits, out);
  note_launch();
}

__global__ void bfv_scale_round_kernel(const uint64_t* __restrict__ x, int64_t total, uint64_t q,
                                       uint64_t p, int64_t* __restrict__ out) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total;
       g += (int64_t)gridDim.x * blockDim.x) {
    const unsigned __int128 num = (unsigned __int128)x[g] * p + q / 2;
    const uint64_t mval = (uint64_t)(num / q) % p;
    out[g] = mval > p / 2 ? (int64_t)mval - (int64_t)p : (int64_t)mval;
  }
}

void bfv_scale_round(const uint64_t* x, int64_t C, int n, uint64_t q, uint64_t p, int64_t* out,
                     cudaStream_t st) {
  if (C == 0) return;
  const int64_t total = C * n;
  int blocks = (int)((total + 255) / 256);
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  bfv_scale_round_kernel<<<blocks, 256, 0, st>>>(x, total, q, p, out);
  note_launch();
}

__global__ void digit_extract_kernel(const uint64_t* __restrict__ x, int64_t total, int shift,
                                     uint64_t mask, uint64_t* __restrict__ out) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total;
       g += (int64_t)gridDim.x * blockDim.x)
    out[g] = (x[g] >> shift) & mask;
}

void digit_extract(const uint64_t* x, int64_t rows, int n, int shift, int bits, uint64_t* out,
                   cudaStream_t st) {
  if (rows == 0) return;
  const int64_t total = rows * n;
  int blocks = (int)((total + 255) / 256);
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  const uint64_t mask = bits >= 64 ? ~0ull : ((1ull << bits) - 1);
  digit_extract_kernel<<<blocks, 256, 0, st>>>(x, total, shift, mask, out);
  note_launch();
}

// ------------------------------------------------------------------------------------------
// Key generation on the device (SURVEY X1.b / X1.c). Same counter-based streams as the host twin
// (host::sample_secret / host::gen_public), so the keys are bit-identical for a given seed; the NTTs in
// between are the regular batched kernels. Reference: HE.keyGen() / relinKeyGen (FLPyfhelin.py:340, :362).
// ------------------------------------------------------------------------------------------
// mode 0: ternary secret, out [L][n]; mode 1: centred-binomial error of key idx0 + e, out = pk [E][2][L][n], slot [e][0]
__global__ void keygen_sample_kernel(uint64_t* __restrict__ out, int L, int n, const uint64_t* __restrict__ consts,
                                     uint64_t seed, uint32_t idx0, int mode) {
  const int l = blockIdx.y, e = blockIdx.z;
  const uint64_t q = consts[(size_t)l * 8];
  uint64_t* o = out + ((size_t)e * (mode ? 2 : 1) * L + l) * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    o[i] = mode ? lift_signed(sample_cbd(seed, STREAM_PK_E, idx0 + (uint32_t)e, (uint32_t)i), q)
                : lift_signed(sample_ternary(seed, STREAM_SK, (uint32_t)i), q);
}

// pk [E][2][L][n] with NTT(e) in slot 0: slot 1 <- a (uniform), slot 0 <- -(a s + e)
__global__ void keygen_finish_kernel(const uint64_t* __restrict__ sk, uint64_t* __restrict__ pk, int L, int n,
                                     const uint64_t* __restrict__ consts, uint64_t seed, uint32_t idx0) {
  const int l = blockIdx.y, e = blockIdx.z;
  const uint64_t* c = consts + (size_t)l * 8;
  const Modulus m{c[0], c[1], c[2]};
  uint64_t* b = pk + ((size_t)e * 2 * L + l) * n;
  uint64_t* a = b + (size_t)L * n;
  const uint64_t* s = sk + (size_t)l * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t ai = sample_uniform(seed, idx0 + (uint32_t)e, (uint32_t)l, (uint32_t)i, m);
    a[i] = ai;
    b[i] = neg_mod(mad_mod(ai, s[i], b[i], m), m.q);
  }
}

// evaluation keys: evk[e][0][limb_of[e]] += w[e] * s2[limb_of[e]]  (the CRT-basis message term of digit e)
__global__ void relin_message_kernel(uint64_t* __restrict__ evk, const uint64_t* __restrict__ s2,
                                     const int* __restrict__ limb_of, const uint64_t* __restrict__ w, int L, int n,
                                     const uint64_t* __restrict__ consts) {
  const int e = blockIdx.y, l = limb_of[e];
  const uint64_t* c = consts + (size_t)l * 8;
  const Modulus m{c[0], c[1], c[2]};
  uint64_t* b = evk + ((size_t)e * 2 * L + l) * n;
  const uint64_t* s = s2 + (size_t)l * n;
  const uint64_t we = w[e];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    b[i] = add_mod(b[i], mul_mod(we, s[i], m), m.q);
}

void keygen_sample(uint64_t* out, int E, int L, int n, const uint64_t* consts, uint64_t seed, uint32_t idx0, int mode,
                   cudaStream_t st) {
  dim3 grid((n + 1023) / 1024, L, E);
  keygen_sample_kernel<<<grid, 256, 0, st>>>(out, L, n, consts, seed, idx0, mode);
  note_launch();
}

void keygen_finish(const uint64_t* sk, uint64_t* pk, int E, int L, int n, const uint64_t* consts, uint64_t seed,
                   uint32_t idx0, cudaStream_t st) {
  dim3 grid((n + 1023) / 1024, L, E);
  keygen_finish_kernel<<<grid, 256, 0, st>>>(sk, pk, L, n, consts, seed, idx0);
  note_launch();
}

void relin_message(uint64_t* evk, const uint64_t* s2, const int* limb_of, const uint64_t* w, int E, int L, int n,
                   const uint64_t* consts, cudaStream_t st) {
  dim3 grid((n + 1023) / 1024, E);
  relin_message_kernel<<<grid, 256, 0, st>>>(evk, s2, limb_of, w, L, n, consts);
  note_launch();
}

}  // namespace cuda
}  // namespace hefl
