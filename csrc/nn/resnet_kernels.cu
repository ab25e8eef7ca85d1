// ResNet building blocks for sm_90a (SURVEY.md K18): training-mode BatchNorm over NHWC bf16 with
// fused residual add and ReLU (forward and backward), and global average pooling. Activations are
// [P = B*H*W pixels, C channels] bf16, statistics and parameters fp32.
//
//   forward : bn_stats (per-channel sum / sum-of-squares, one fp32 atomic per channel per CTA)
//             bn_apply (finalises the statistics per CTA, normalise, scale/shift, + residual, ReLU; CTA 0
//                       publishes mean / invstd and updates the running statistics)
//   backward: bn_bwd_reduce (dbeta, dgamma with the ReLU mask recomputed from the output)
//             bn_bwd_apply  (dx, and the gradient that flows into the residual branch)
#include <cuda_bf16.h>

#include "../he/kernels.h"
#include "nn.h"

namespace hefl {
namespace nn {

// Each CTA reduces a slab of rows for 8-channel groups; threads = (row lane, channel group).
__global__ void bn_stats_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ sums, int64_t P, int C) {
  const int groups = C >> 3;
  const int cg = threadIdx.x % groups;
  const int rl = threadIdx.x / groups;
  const int rows_per_iter = blockDim.x / groups;
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = q[i] = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * rows_per_iter + rl; r < P; r += (int64_t)gridDim.x * rows_per_iter) {
    const uint4 v = *reinterpret_cast<const uint4*>(x + r * C + cg * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float a = __uint_as_float(w[i] << 16), b = __uint_as_float(w[i] & 0xFFFF0000u);
      s[2 * i] += a; q[2 * i] += a * a;
      s[2 * i + 1] += b; q[2 * i + 1] += b * b;
    }
  }
  extern __shared__ float red[];   // [2][C]
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    atomicAdd(&red[cg * 8 + i], s[i]);
    atomicAdd(&red[C + cg * 8 + i], q[i]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) atomicAdd(&sums[i], red[i]);
}

// Normalise + scale/shift (+ residual) (+ ReLU). Every CTA derives the per-channel scale/shift from the raw
// sums into shared memory; CTA 0 also publishes mean / invstd (saved for backward) and the running statistics.
__global__ void bn_apply_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                                const float* __restrict__ sums, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float* __restrict__ mean_out,
                                float* __restrict__ invstd_out, float* __restrict__ run_mean,
                                float* __restrict__ run_var, __nv_bfloat16* __restrict__ y, int64_t P, int C,
                                float momentum, float eps, int relu) {
  extern __shared__ float ss[];   // [C] scale, [C] shift
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float m = sums[c] / (float)P;
    const float var = fmaxf(sums[C + c] / (float)P - m * m, 0.f);
    const float is = rsqrtf(var + eps);
    const float sc = gamma[c] * is;
    ss[c] = sc;
    ss[C + c] = beta[c] - m * sc;
    if (blockIdx.x == 0) {
      mean_out[c] = m;
      invstd_out[c] = is;
      if (run_mean) {
        run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * m;
        run_var[c] = (1.f - momentum) * run_var[c] + momentum * var * ((float)P / (float)(P > 1 ? P - 1 : 1));
      }
    }
  }
  __syncthreads();
  // thread = (row lane, 8-channel group): no division inside the loop (a 64-bit t / groups per element cost
  // more than the loads)
  const int groups = C >> 3;
  const int cg = threadIdx.x % groups;
  const int rows_per_iter = blockDim.x / groups;
  for (int64_t row = (int64_t)blockIdx.x * rows_per_iter + threadIdx.x / groups; row < P;
       row += (int64_t)gridDim.x * rows_per_iter) {
    const int64_t o = row * C + cg * 8;
    const uint4 v = *reinterpret_cast<const uint4*>(x + o);
    uint4 rv = make_uint4(0u, 0u, 0u, 0u);
    if (res) rv = *reinterpret_cast<const uint4*>(res + o);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
    uint32_t ow[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float a[2] = {__uint_as_float(w[i] << 16), __uint_as_float(w[i] & 0xFFFF0000u)};
      const float r[2] = {__uint_as_float(rw[i] << 16), __uint_as_float(rw[i] & 0xFFFF0000u)};
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = cg * 8 + 2 * i + j;
        float z = fmaf(a[j], ss[c], ss[C + c]) + r[j];
        if (relu) z = z > 0.f ? z : 0.f;
        a[j] = z;
      }
      const __nv_bfloat162 pk = __floats2bfloat162_rn(a[0], a[1]);
      ow[i] = *reinterpret_cast<const uint32_t*>(&pk);
    }
    *reinterpret_cast<uint4*>(y + o) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
  }
}

// sums[0..C) = dbeta = sum dy', sums[C..2C) = dgamma = sum dy' * xhat, with dy' = dy * (y > 0) if relu.
__global__ void bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                     const __nv_bfloat16* __restrict__ y, const float* __restrict__ mean,
                                     const float* __restrict__ invstd, float* __restrict__ sums, int64_t P, int C,
                                     int relu) {
  const int groups = C >> 3;
  const int cg = threadIdx.x % groups;
  const int rl = threadIdx.x / groups;
  const int rows_per_iter = blockDim.x / groups;
  float s[8], q[8], mu[8], is[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = q[i] = 0.f; mu[i] = mean[cg * 8 + i]; is[i] = invstd[cg * 8 + i]; }
  for (int64_t r = (int64_t)blockIdx.x * rows_per_iter + rl; r < P; r += (int64_t)gridDim.x * rows_per_iter) {
    const int64_t o = r * C + cg * 8;
    const uint4 dv = *reinterpret_cast<const uint4*>(dy + o);
    const uint4 xv = *reinterpret_cast<const uint4*>(x + o);
    uint4 yv = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
    if (relu) yv = *reinterpret_cast<const uint4*>(y + o);
    const uint32_t dw[4] = {dv.x, dv.y, dv.z, dv.w}, xw[4] = {xv.x, xv.y, xv.z, xv.w}, yw[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int k = 2 * i + j;
        const uint32_t sh = j ? 0u : 16u;
        const float d = __uint_as_float(j ? (dw[i] & 0xFFFF0000u) : (dw[i] << 16));
        const float xx = __uint_as_float(j ? (xw[i] & 0xFFFF0000u) : (xw[i] << 16));
        const uint32_t yb = j ? (yw[i] >> 16) : (yw[i] & 0xFFFFu);
        (void)sh;
        const bool on = !relu || (yb != 0u && (yb & 0x8000u) == 0u);
        const float dd = on ? d : 0.f;
        s[k] += dd;
        q[k] += dd * (xx - mu[k]) * is[k];
      }
    }
  }
  extern __shared__ float red[];
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    atomicAdd(&red[cg * 8 + i], s[i]);
    atomicAdd(&red[C + cg * 8 + i], q[i]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) atomicAdd(&sums[i], red[i]);
}

// dx = gamma*invstd * (dy' - dbeta/P - xhat*dgamma/P); dres = dy' (gradient into the residual branch).
// Per channel: dx = a*dy' + b*x + c with a = gamma*invstd, b = -a*invstd*dgamma/P, c = -a*dbeta/P - b*mean.
__global__ void bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                    const __nv_bfloat16* __restrict__ y, const float* __restrict__ mean,
                                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                                    const float* __restrict__ sums, __nv_bfloat16* __restrict__ dx,
                                    __nv_bfloat16* __restrict__ dres, int64_t P, int C, int relu) {
  extern __shared__ float ss[];   // [3][C]
  const float invP = 1.f / (float)P;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float a = gamma[c] * invstd[c];
    const float b = -a * invstd[c] * sums[C + c] * invP;
    ss[c] = a;
    ss[C + c] = b;
    ss[2 * C + c] = -a * sums[c] * invP - b * mean[c];
  }
  __syncthreads();
  // thread = (row lane, 8-channel group): no division inside the loop (a 64-bit t / groups per element cost
  // more than the loads)
  const int groups = C >> 3;
  const int cg = threadIdx.x % groups;
  const int rows_per_iter = blockDim.x / groups;
  for (int64_t row = (int64_t)blockIdx.x * rows_per_iter + threadIdx.x / groups; row < P;
       row += (int64_t)gridDim.x * rows_per_iter) {
    const int64_t o = row * C + cg * 8;
    const uint4 dv = *reinterpret_cast<const uint4*>(dy + o);
    const uint4 xv = *reinterpret_cast<const uint4*>(x + o);
    uint4 yv = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
    if (relu) yv = *reinterpret_cast<const uint4*>(y + o);
    const uint32_t dw[4] = {dv.x, dv.y, dv.z, dv.w}, xw[4] = {xv.x, xv.y, xv.z, xv.w}, yw[4] = {yv.x, yv.y, yv.z, yv.w};
    uint32_t ow[4], rw[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float od[2], rd[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = cg * 8 + 2 * i + j;
        const float d = __uint_as_float(j ? (dw[i] & 0xFFFF0000u) : (dw[i] << 16));
        const float xx = __uint_as_float(j ? (xw[i] & 0xFFFF0000u) : (xw[i] << 16));
        const uint32_t yb = j ? (yw[i] >> 16) : (yw[i] & 0xFFFFu);
        const bool on = !relu || (yb != 0u && (yb & 0x8000u) == 0u);
        const float dd = on ? d : 0.f;
        od[j] = fmaf(ss[c], dd, fmaf(ss[C + c], xx, ss[2 * C + c]));
        rd[j] = dd;
      }
      const __nv_bfloat162 p0 = __floats2bfloat162_rn(od[0], od[1]);
      const __nv_bfloat162 p1 = __floats2bfloat162_rn(rd[0], rd[1]);
      ow[i] = *reinterpret_cast<const uint32_t*>(&p0);
      rw[i] = *reinterpret_cast<const uint32_t*>(&p1);
    }
    *reinterpret_cast<uint4*>(dx + o) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    if (dres) *reinterpret_cast<uint4*>(dres + o) = make_uint4(rw[0], rw[1], rw[2], rw[3]);
  }
}

static inline int blocks_for(int64_t work, int per_block, int cap) {
  int64_t b = (work + per_block - 1) / per_block;
  if (b > cap) b = cap;
  return b < 1 ? 1 : (int)b;
}

void bn_forward(const void* x, const void* res, const float* gamma, const float* beta, float* run_mean, float* run_var,
                float* mean, float* invstd, float* sums, void* y, int64_t P, int C, float momentum, float eps, int relu,
                cudaStream_t st) {
  cudaMemsetAsync(sums, 0, 2 * C * sizeof(float), st);
  const int threads = 256 - 256 % (C / 8 > 256 ? 256 : (C / 8));   // multiple of the channel-group count
  const int rows_per_iter = threads / (C / 8);
  bn_stats_kernel<<<blocks_for(P, rows_per_iter * 8, hefl::cuda::device_sm_count() * 4), threads, 2 * C * 4, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), sums, P, C);
  bn_apply_kernel<<<blocks_for(P, rows_per_iter * 4, hefl::cuda::device_sm_count() * 8), threads, 2 * C * 4, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(res), sums, gamma, beta, mean,
      invstd, run_mean, run_var, reinterpret_cast<__nv_bfloat16*>(y), P, C, momentum, eps, relu);
  hefl::cuda::note_launch(2);
}

void bn_backward(const void* dy, const void* x, const void* y, const float* mean, const float* invstd,
                 const float* gamma, float* sums, void* dx, void* dres, int64_t P, int C, int relu, cudaStream_t st) {
  cudaMemsetAsync(sums, 0, 2 * C * sizeof(float), st);
  const int threads = 256 - 256 % (C / 8 > 256 ? 256 : (C / 8));
  const int rows_per_iter = threads / (C / 8);
  bn_bwd_reduce_kernel<<<blocks_for(P, rows_per_iter * 8, hefl::cuda::device_sm_count() * 4), threads, 2 * C * 4, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(x),
      reinterpret_cast<const __nv_bfloat16*>(y), mean, invstd, sums, P, C, relu);
  bn_bwd_apply_kernel<<<blocks_for(P, rows_per_iter * 4, hefl::cuda::device_sm_count() * 8), threads, 3 * C * 4, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(x),
      reinterpret_cast<const __nv_bfloat16*>(y), mean, invstd, gamma, sums, reinterpret_cast<__nv_bfloat16*>(dx),
      reinterpret_cast<__nv_bfloat16*>(dres), P, C, relu);
  hefl::cuda::note_launch(2);
}

// Global average pool over HW: x [B, HW, C] bf16 -> out [B, C] fp32 (forward) and the broadcast back.
__global__ void avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, int HW, int C) {
  const int b = blockIdx.y;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int p = 0; p < HW; ++p) acc += __bfloat162float(x[((int64_t)b * HW + p) * C + c]);
    out[b * C + c] = acc / (float)HW;
  }
}
__global__ void avgpool_bwd_kernel(const float* __restrict__ dout, __nv_bfloat16* __restrict__ dx, int HW, int C,
                                   int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t b = i / ((int64_t)HW * C);
    dx[i] = __float2bfloat16(dout[b * C + c] / (float)HW);
  }
}
void avgpool_forward(const void* x, float* out, int B, int HW, int C, cudaStream_t st) {
  dim3 grid((C + 127) / 128, B);
  avgpool_fwd_kernel<<<grid, 128, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), out, HW, C);
  hefl::cuda::note_launch();
}
void avgpool_backward(const float* dout, void* dx, int B, int HW, int C, cudaStream_t st) {
  const int64_t total = (int64_t)B * HW * C;
  avgpool_bwd_kernel<<<blocks_for(total, 256, hefl::cuda::device_sm_count() * 8), 256, 0, st>>>(dout, reinterpret_cast<__nv_bfloat16*>(dx), HW, C, total);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl

// ------------------------------------------------------------------------------------------
// FP8 (e4m3) quantisation with delayed scaling for the 1x1 convolutions of ResNet-50 (BASELINE configs[4]:
// "ResNet-50 fp8 local training"). One pass: q = sat_e4m3(x * scale) with the scale derived from the PREVIOUS
// step's amax, and this step's amax recorded for the next one. The GEMM itself is a plain library GEMM
// (cuBLASLt fp8 through torch._scaled_mm); this kernel replaces the amax + scale + cast passes around it.
// ------------------------------------------------------------------------------------------
#include <cuda_fp8.h>

namespace hefl {
namespace nn {

__global__ void fp8_quantize_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                    const float* __restrict__ scale, float* __restrict__ amax, int64_t n8) {
  const float s = *scale;
  float local = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t out[2] = {0u, 0u};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = __uint_as_float(w[k] << 16), b = __uint_as_float(w[k] & 0xFFFF0000u);
      local = fmaxf(local, fmaxf(fabsf(a), fabsf(b)));
      const __nv_fp8x2_storage_t p = __nv_cvt_float2_to_fp8x2(make_float2(a * s, b * s), __NV_SATFINITE, __NV_E4M3);
      out[k >> 1] |= (uint32_t)p << ((k & 1) * 16);
    }
    reinterpret_cast<uint2*>(q)[i] = make_uint2(out[0], out[1]);
  }
  for (int off = 16; off; off >>= 1) local = fmaxf(local, __shfl_xor_sync(0xffffffffu, local, off));
  if ((threadIdx.x & 31) == 0 && local > 0.f) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(local));   // non-negative floats order as ints
}

// MX (block-scaled) e4m3 quantiser: one UE8M0 scale per row and per 32 consecutive elements of K. One thread per
// block of 32 (64 bytes in, 32 bytes out); consecutive lanes take consecutive blocks of a row. The scale bytes are
// written straight in the tile order the tensor core consumes (gemm_tcgen05.cu, MxArgs): per (128-row block,
// 128-element k-group) 512 bytes [lane l][row quarter i][k-block kb] for row 32*i + l.
__global__ void mxfp8_quantize_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf,
                                      int64_t R, int K) {
  const int kblocks = K >> 5, kgroups = K >> 7;
  const int64_t total = R * kblocks;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / kblocks;
    const int kbk = (int)(t - r * kblocks);
    const uint4* src = reinterpret_cast<const uint4*>(x + r * K + kbk * 32);
    uint4 v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = src[i];
    float f[32];
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        f[8 * i + 2 * j] = __uint_as_float(w[j] << 16);
        f[8 * i + 2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
        amax = fmaxf(amax, fmaxf(fabsf(f[8 * i + 2 * j]), fabsf(f[8 * i + 2 * j + 1])));
      }
    }
    // smallest e with amax * 2^-e <= 448 (the largest e4m3 magnitude)
    int e = -127;
    if (amax > 0.f) {
      e = (int)((__float_as_uint(amax) >> 23) & 0xFFu) - 127 - 8;
      if (e < -127) e = -127;
      const float probe = amax * __uint_as_float((uint32_t)(127 - e) << 23);
      if (probe > 448.f) ++e;
      if (e > 127) e = 127;
    }
    const float inv = __uint_as_float((uint32_t)(127 - e) << 23);        // 2^-e
    uint32_t out[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(f[4 * i] * inv, f[4 * i + 1] * inv), __NV_SATFINITE, __NV_E4M3);
      const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(f[4 * i + 2] * inv, f[4 * i + 3] * inv), __NV_SATFINITE, __NV_E4M3);
      out[i] = (uint32_t)lo | ((uint32_t)hi << 16);
    }
    uint4* dst = reinterpret_cast<uint4*>(q + r * K + kbk * 32);
    dst[0] = make_uint4(out[0], out[1], out[2], out[3]);
    dst[1] = make_uint4(out[4], out[5], out[6], out[7]);
    const int64_t mb = r >> 7;
    const int rr = (int)(r & 127), l = rr & 31, qi = rr >> 5;
    sf[((mb * kgroups + (kbk >> 2)) * 32 + l) * 16 + qi * 4 + (kbk & 3)] = (uint8_t)(e + 127);
  }
}

void mxfp8_quantize(const void* x, uint8_t* q, uint8_t* sf, int64_t R, int K, cudaStream_t st) {
  const int64_t total = R * (K >> 5);
  mxfp8_quantize_kernel<<<blocks_for(total, 256, hefl::cuda::device_sm_count() * 16), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), q, sf, R, K);
  hefl::cuda::note_launch();
}

// Delayed scaling bookkeeping of one tensor role in ONE tiny launch (was six ATen element-wise kernels per
// tensor and step): scale <- (448 / margin) / amax_prev (kept when amax_prev == 0), inv <- 1 / scale, amax <- 0.
__global__ void fp8_scale_update_kernel(float* __restrict__ amax, float* __restrict__ scale, float* __restrict__ inv,
                                        float target) {
  const float a = *amax;
  float s = *scale;
  if (a > 0.f) s = target / fmaxf(a, 1e-12f);
  *scale = s;
  *inv = 1.0f / s;
  *amax = 0.f;
}

void fp8_scale_update(float* amax, float* scale, float* inv, float target, cudaStream_t st) {
  fp8_scale_update_kernel<<<1, 1, 0, st>>>(amax, scale, inv, target);
  hefl::cuda::note_launch();
}

void fp8_quantize(const void* x, uint8_t* q, const float* scale, float* amax, int64_t n, cudaStream_t st) {
  const int64_t n8 = n / 8;
  fp8_quantize_kernel<<<blocks_for(n8, 256 * 4, hefl::cuda::device_sm_count() * 8), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), q, scale,
                                                                       amax, n8);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl
