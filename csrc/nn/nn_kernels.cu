// Small fused NN kernels for sm_90a: Adam (+ bf16 weight shadow), input preprocessing,
// un-pooling of gradients. SURVEY.md §2.4 K17.
#include <cuda_bf16.h>

#include "../he/kernels.h"
#include "../he/philox.h"
#include "nn.h"
#include "launch.cuh"

namespace hefl {
namespace nn {

// PROX: FedProx local objective, the gradient of (mu/2)*||p - anchor||^2 is added to g before the moments
// (anchor = the round's global model). The extra arguments come last so that <false> keeps today's code.
template <bool PROX>
__global__ void adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, __nv_bfloat16* __restrict__ shadow, int64_t n,
                            const int64_t* __restrict__ step, const float* __restrict__ lr_scale,
                            float lr, float decay, float beta1, float beta2, float eps,
                            const float* __restrict__ anchor, float mu) {
  pdl_wait();   // parameter writer: no early trigger (see launch.cuh)
  const float t = (float)(*step);
  const float lr_t = lr * (lr_scale ? *lr_scale : 1.0f) / (1.0f + decay * (t - 1.0f));
  const float bc1 = 1.0f - powf(beta1, t);
  const float bc2 = 1.0f - powf(beta2, t);
  const float alpha = lr_t * sqrtf(bc2) / bc1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i];
    if (PROX) gi += mu * (p[i] - anchor[i]);
    const float mi = beta1 * m[i] + (1.0f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.0f - beta2) * gi * gi;
    const float pi = p[i] - alpha * mi / (sqrtf(vi) + eps);
    m[i] = mi;
    v[i] = vi;
    p[i] = pi;
    g[i] = 0.0f;
    if (shadow) shadow[i] = __float2bfloat16(pi);
  }
}

void adam_step(float* p, float* g, float* m, float* v, void* shadow_bf16, int64_t n,
               const int64_t* step, const float* lr_scale, float lr, float decay, float beta1,
               float beta2, float eps, const float* anchor, float mu, cudaStream_t st) {
  if (n == 0) return;
  int blocks = (int)((n + 255) / 256);
  if (blocks > hefl::cuda::device_sm_count() * 8) blocks = hefl::cuda::device_sm_count() * 8;
  launch_pdl(anchor && mu != 0.0f ? adam_kernel<true> : adam_kernel<false>, dim3(blocks), dim3(256), 0, st, p, g, m, v,
             reinterpret_cast<__nv_bfloat16*>(shadow_bf16), n, step, lr_scale, lr, decay, beta1, beta2, eps, anchor, mu);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl

// ------------------------------------------------------------------------------------------
// Data-movement kernels around the tcgen05 convolutions
// ------------------------------------------------------------------------------------------
namespace hefl {
namespace nn {

// Per-sample affine warp of the pre-processing: theta[b] if given, else (aug_seed != 0) Keras
// ImageDataGenerator(shear_range=0.2 deg, zoom_range=0.2, horizontal_flip) drawn per sample from a counter-based
// generator keyed by (seed, optimiser step, sample). Returns false when the image is not warped.
__device__ __forceinline__ bool preprocess_theta(const float* __restrict__ theta, uint64_t aug_seed,
                                                 const int64_t* __restrict__ step, int b, float tl[6]) {
  bool warp_img = theta != nullptr;
  if (theta) {
#pragma unroll
    for (int i = 0; i < 6; ++i) tl[i] = theta[b * 6 + i];
  } else if (aug_seed != 0) {
    const uint64_t st = step ? (uint64_t)*step : 0ull;
    const Philox4 r = philox4x32_10((uint32_t)b, (uint32_t)st, (uint32_t)(st >> 32), 7u, (uint32_t)aug_seed,
                                    (uint32_t)(aug_seed >> 32));
    const float u0 = r.x * 2.3283064e-10f, u1 = r.y * 2.3283064e-10f, u2 = r.z * 2.3283064e-10f;
    const float sh = (u0 * 2.f - 1.f) * 0.2f * 0.017453292f;
    const float zx = 1.f + (u1 * 2.f - 1.f) * 0.2f, zy = 1.f + (u2 * 2.f - 1.f) * 0.2f;
    const float flip = (r.w & 1u) ? -1.f : 1.f;
    tl[0] = zx * flip; tl[1] = -sinf(sh) * zx; tl[2] = 0.f;
    tl[3] = 0.f; tl[4] = cosf(sh) * zy; tl[5] = 0.f;
    warp_img = true;
  }
  return warp_img;
}

// uint8 NHWC (3 channels) -> bf16 [P,16] (channels 3..15 zero), with 1/255 rescale and an optional per-sample affine warp (Keras shear/zoom/flip,
// FLPyfhelin.py:80-86) sampled bilinearly with border clamp (torch.grid_sample semantics,
// align_corners=False). With `compact` the output is [P,4] instead: R, G, B, 0 — one 8-byte store per pixel, the
// same values as channels 0-2 of the other layouts.
__global__ void preprocess_u8_kernel(const uint8_t* __restrict__ x, const float* __restrict__ theta,
                                     __nv_bfloat16* __restrict__ X, int B, int H, int W, uint64_t aug_seed,
                                     const int64_t* __restrict__ step, int spack, int compact) {
  pdl_prologue();
  const int b = blockIdx.y;
  float tl[6];
  const bool warp_img = preprocess_theta(theta, aug_seed, step, b, tl);
  // One warp = one run of consecutive pixels of an image row. With `spack` (s-packed layer-1 input: channels
  // 0-2 = this pixel, 3-5 = pixel w+1, 6-8 = pixel w+2, so the three horizontal filter taps become part of the
  // GEMM K dimension) a warp stores 30 pixels and lanes 30/31 only feed their values to the shuffles.
  const int lane = threadIdx.x & 31;
  const int PW = spack && !compact ? 30 : 32;
  const int chunks = (W + PW - 1) / PW;
  const int tasks = H * chunks;
  const int wpb = blockDim.x >> 5;
  const uint8_t* img = x + (int64_t)b * H * W * 3;
  for (int task = blockIdx.x * wpb + (threadIdx.x >> 5); task < tasks; task += gridDim.x * wpb) {
    const int h = task / chunks;
    const int w = (task - h * chunks) * PW + lane;
    const int wc = w < W ? w : W - 1;
    float c[3];
    if (warp_img) {
      const float* t = tl;
      const float xn = (2.f * wc + 1.f) / W - 1.f, yn = (2.f * h + 1.f) / H - 1.f;
      const float sx = t[0] * xn + t[1] * yn + t[2], sy = t[3] * xn + t[4] * yn + t[5];
      float ix = ((sx + 1.f) * W - 1.f) * 0.5f, iy = ((sy + 1.f) * H - 1.f) * 0.5f;
      ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));
      iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
      const int x0 = (int)floorf(ix), y0 = (int)floorf(iy);
      const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
      const float fx = ix - x0, fy = iy - y0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float v00 = img[((int64_t)y0 * W + x0) * 3 + k], v01 = img[((int64_t)y0 * W + x1) * 3 + k];
        const float v10 = img[((int64_t)y1 * W + x0) * 3 + k], v11 = img[((int64_t)y1 * W + x1) * 3 + k];
        c[k] = ((v00 * (1.f - fx) + v01 * fx) * (1.f - fy) + (v10 * (1.f - fx) + v11 * fx) * fy) * (1.f / 255.f);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) c[k] = (float)img[((int64_t)h * W + wc) * 3 + k] * (1.f / 255.f);
    }
    uint32_t p01 = (uint32_t)__bfloat16_as_ushort(__float2bfloat16(c[0])) |
                   ((uint32_t)__bfloat16_as_ushort(__float2bfloat16(c[1])) << 16);
    uint32_t p2 = __bfloat16_as_ushort(__float2bfloat16(c[2]));
    if (compact) {
      if (w < W) *reinterpret_cast<uint2*>(X + ((int64_t)(b * H + h) * W + w) * 4) = make_uint2(p01, p2);
      continue;
    }
    if (w >= W) { p01 = 0u; p2 = 0u; }                       // past the row end: zero neighbours
    const uint32_t n1_01 = __shfl_down_sync(0xffffffffu, p01, 1), n1_2 = __shfl_down_sync(0xffffffffu, p2, 1);
    const uint32_t n2_01 = __shfl_down_sync(0xffffffffu, p01, 2), n2_2 = __shfl_down_sync(0xffffffffu, p2, 2);
    if (lane < PW && w < W) {
      uint4* dst = reinterpret_cast<uint4*>(X + ((int64_t)(b * H + h) * W + w) * 16);
      if (spack) {
        dst[0] = make_uint4(p01, p2 | (n1_01 << 16), (n1_01 >> 16) | (n1_2 << 16), n2_01);
        dst[1] = make_uint4(n2_2, 0u, 0u, 0u);
      } else {
        dst[0] = make_uint4(p01, p2, 0u, 0u);
        dst[1] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
}

// One-channel (grayscale) input: the same scaling, warp and Philox keying as preprocess_u8_kernel. With `spack`
// it writes the rs-packed layer-1 input: channel 3r + s holds pixel (h + r, w + s), 0 past the bottom or right
// edge, channels 9..15 zero — the whole 3x3 neighbourhood, so layer 1 is a single K = 16 GEMM. Without it,
// channel 0 = pixel and the rest zero. Each warp samples its own three rows (h, h+1, h+2) with the code that
// samples row h + r as channel 0, so channel 3r + s is bit-identical to channel 0 of pixel (h + r, w + s).
__global__ void preprocess_u8_gray_kernel(const uint8_t* __restrict__ x, const float* __restrict__ theta,
                                          __nv_bfloat16* __restrict__ X, int B, int H, int W, uint64_t aug_seed,
                                          const int64_t* __restrict__ step, int spack) {
  pdl_prologue();
  const int b = blockIdx.y;
  float tl[6];
  const bool warp_img = preprocess_theta(theta, aug_seed, step, b, tl);
  const int lane = threadIdx.x & 31;
  const int PW = spack ? 30 : 32;
  const int NR = spack ? 3 : 1;
  const int chunks = (W + PW - 1) / PW;
  const int tasks = H * chunks;
  const int wpb = blockDim.x >> 5;
  const uint8_t* img = x + (int64_t)b * H * W;
  for (int task = blockIdx.x * wpb + (threadIdx.x >> 5); task < tasks; task += gridDim.x * wpb) {
    const int h = task / chunks;
    const int w = (task - h * chunks) * PW + lane;
    const int wc = w < W ? w : W - 1;
    uint32_t v[3] = {0u, 0u, 0u};                            // bf16 bits of pixel (h + r, w)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hh = h + r;
      if (r >= NR || hh >= H) continue;                      // rows below the image: zero
      float c;
      if (warp_img) {
        const float xn = (2.f * wc + 1.f) / W - 1.f, yn = (2.f * hh + 1.f) / H - 1.f;
        const float sx = tl[0] * xn + tl[1] * yn + tl[2], sy = tl[3] * xn + tl[4] * yn + tl[5];
        float ix = ((sx + 1.f) * W - 1.f) * 0.5f, iy = ((sy + 1.f) * H - 1.f) * 0.5f;
        ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));
        iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
        const int x0 = (int)floorf(ix), y0 = (int)floorf(iy);
        const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
        const float fx = ix - x0, fy = iy - y0;
        const float v00 = img[(int64_t)y0 * W + x0], v01 = img[(int64_t)y0 * W + x1];
        const float v10 = img[(int64_t)y1 * W + x0], v11 = img[(int64_t)y1 * W + x1];
        c = ((v00 * (1.f - fx) + v01 * fx) * (1.f - fy) + (v10 * (1.f - fx) + v11 * fx) * fy) * (1.f / 255.f);
      } else {
        c = (float)img[(int64_t)hh * W + wc] * (1.f / 255.f);
      }
      v[r] = w < W ? (uint32_t)__bfloat16_as_ushort(__float2bfloat16(c)) : 0u;   // past the row end: zero
    }
    if (spack) {
      uint32_t k[9];                                         // channel 3r + s = pixel (h + r, w + s)
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        k[3 * r] = v[r];
        k[3 * r + 1] = __shfl_down_sync(0xffffffffu, v[r], 1);
        k[3 * r + 2] = __shfl_down_sync(0xffffffffu, v[r], 2);
      }
      if (lane < PW && w < W) {
        uint4* dst = reinterpret_cast<uint4*>(X + ((int64_t)(b * H + h) * W + w) * 16);
        dst[0] = make_uint4(k[0] | (k[1] << 16), k[2] | (k[3] << 16), k[4] | (k[5] << 16), k[6] | (k[7] << 16));
        dst[1] = make_uint4(k[8], 0u, 0u, 0u);
      }
    } else if (w < W) {
      uint4* dst = reinterpret_cast<uint4*>(X + ((int64_t)(b * H + h) * W + w) * 16);
      dst[0] = make_uint4(v[0], 0u, 0u, 0u);
      dst[1] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

void preprocess_u8(const uint8_t* x, const float* theta, void* X, int B, int H, int W, int C, uint64_t aug_seed,
                   const int64_t* step, int spack, int compact, cudaStream_t st) {
  const int pw = spack && !compact ? 30 : 32;
  const int tasks = H * ((W + pw - 1) / pw);
  int bx = (tasks + 7) / 8;
  if (bx > 64) bx = 64;
  dim3 grid(bx, B);
  if (C == 1)
    launch_pdl(preprocess_u8_gray_kernel, dim3(grid), dim3(256), 0, st, x, theta, reinterpret_cast<__nv_bfloat16*>(X),
               B, H, W, aug_seed, step, spack);
  else
    launch_pdl(preprocess_u8_kernel, dim3(grid), dim3(256), 0, st, x, theta, reinterpret_cast<__nv_bfloat16*>(X), B,
               H, W, aug_seed, step, spack, compact);
  hefl::cuda::note_launch();
}

// Gradient of (ReLU -> 2x2 max-pool): scatter the pooled gradient to the arg-max position on the
// conv-input grid, zero elsewhere (including the invalid border). Output [P, Co] bf16 feeds both
// dgrad (K-major A operand) and wgrad (MN-major B operand). One thread = one pixel x 8 channels.
__global__ void unpool_relu_kernel(const __nv_bfloat16* __restrict__ g, const uint8_t* __restrict__ amax,
                                   const __nv_bfloat16* __restrict__ ypool, __nv_bfloat16* __restrict__ dY, int B,
                                   int H, int W, int Hp, int Wp, int Co) {
  pdl_prologue();
  // One thread = one 2x2 window x 8 channels: reads the pooled data once, writes all four
  // positions (windows outside the pooled grid write zeros so the whole H x W grid is defined).
  const int groups = Co >> 3;
  const int Wh = (W + 1) >> 1;
  const int rowp = blockIdx.y;                // b*Hh + hh, Hh = ceil(H/2)
  const int Hh = (H + 1) >> 1;
  const int b = rowp / Hh, hh = rowp - b * Hh;
  const int per_row = Wh * groups;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < per_row; t += gridDim.x * blockDim.x) {
    const int ww = t / groups;
    const int cg = t - ww * groups;
    uint32_t ow[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int i = 0; i < 4; ++i) ow[q][i] = 0u;
    if (hh < Hp && ww < Wp) {
      const int64_t o = (((int64_t)b * Hp + hh) * Wp + ww) * Co + cg * 8;
      const uint4 gv = *reinterpret_cast<const uint4*>(g + o);
      const uint4 yv = *reinterpret_cast<const uint4*>(ypool + o);
      const uint2 av = *reinterpret_cast<const uint2*>(amax + o);
      const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
      const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w};
      const uint32_t aw[2] = {av.x, av.y};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int c = i * 2 + j;
          const uint32_t a8 = (aw[c >> 2] >> ((c & 3) * 8)) & 3u;
          const uint32_t yb = (yw[i] >> (16 * j)) & 0xFFFFu;
          const bool on = yb != 0u && (yb & 0x8000u) == 0u;             // pooled > 0
          const uint32_t val = on ? (((gw[i] >> (16 * j)) & 0xFFFFu) << (16 * j)) : 0u;
#pragma unroll
          for (int q = 0; q < 4; ++q) ow[q][i] |= (a8 == (uint32_t)q) ? val : 0u;
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int h = 2 * hh + (q >> 1), w = 2 * ww + (q & 1);
      if (h < H && w < W)
        *reinterpret_cast<uint4*>(dY + (((int64_t)b * H + h) * W + w) * Co + cg * 8) =
            make_uint4(ow[q][0], ow[q][1], ow[q][2], ow[q][3]);
    }
  }
}

void unpool_relu(const void* g, const uint8_t* amax, const void* ypool, void* dY, int B, int H, int W, int Hp,
                 int Wp, int Co, cudaStream_t st) {
  const int per_row = ((W + 1) / 2) * (Co / 8);
  dim3 grid((per_row + 127) / 128, B * ((H + 1) / 2));
  launch_pdl(unpool_relu_kernel, dim3(grid), dim3(128), 0, st, reinterpret_cast<const __nv_bfloat16*>(g), amax,
                                           reinterpret_cast<const __nv_bfloat16*>(ypool),
                                           reinterpret_cast<__nv_bfloat16*>(dY), B, H, W, Hp, Wp, Co);
  hefl::cuda::note_launch();
}

// bf16 shadow of the flat parameters ([Co][Ci][3][3] per conv) -> Wf [tap][Co][CK] (forward B
// operand, channel-padded) and Wd [tap][Ci][Co] (dgrad B operand).
__global__ void conv_weight_relayout_kernel(const __nv_bfloat16* __restrict__ shadow, const ConvLayerTable t,
                                            __nv_bfloat16* __restrict__ Wf, __nv_bfloat16* __restrict__ Wd, int l0,
                                            int spack0, int compact0) {
  pdl_wait();   // parameter writer: no early trigger (see launch.cuh)
  const int l = blockIdx.y + l0;
  const int Ci = t.Ci[l], CK = t.CK[l], Co = t.Co[l];
  const __nv_bfloat16* w = shadow + t.w_off[l];
  if (l == 0 && compact0) {
    // compact RGB layer 1 ([P,4] input, pixels 2j..2j+3 x (R, G, B, 0) form one K = 16 row): Wf [3 r][2 dx][Co][16]
    // after the s-packed [3][Co][CK] (written below too: the 16-channel kernels may be selected at any time), k =
    // 4 * slot + ci with slot = s + dx, so column parity dx is a choice of weights, not of input address
    const int nf = 6 * Co * CK;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) {
      const int k = i % CK, co = (i / CK) % Co, rd = i / (CK * Co);
      const int r = rd >> 1, sx = (k >> 2) - (rd & 1), ci = k & 3;
      Wf[t.wf_off[l] + 3 * Co * CK + i] =
          sx >= 0 && sx < 3 && ci < Ci ? w[(co * Ci + ci) * 9 + r * 3 + sx] : __float2bfloat16(0.f);
    }
  }
  if (l == 0 && spack0 && Ci == 1) {
    // rs-packed one-channel layer 1: Wf [1][Co][CK], k = 3r + s (the input carries the whole 3x3 neighbourhood)
    const int nf = Co * CK;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) {
      const int k = i % CK, co = i / CK;
      Wf[t.wf_off[l] + i] = k < 9 ? w[co * 9 + k] : __float2bfloat16(0.f);
    }
    return;
  }
  if (l == 0 && spack0) {
    // s-packed layer 1: Wf [3 filter rows][Co][CK], k = s*Ci + ci (the input carries pixels w, w+1, w+2)
    const int nf = 3 * Co * CK;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) {
      const int k = i % CK, co = (i / CK) % Co, r = i / (CK * Co);
      const int sx = k / Ci, ci = k - sx * Ci;
      Wf[t.wf_off[l] + i] = k < 3 * Ci ? w[(co * Ci + ci) * 9 + r * 3 + sx] : __float2bfloat16(0.f);
    }
    return;
  }
  const int nf = 9 * Co * CK;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) {
    const int ck = i % CK, co = (i / CK) % Co, tap = i / (CK * Co);
    Wf[t.wf_off[l] + i] = ck < Ci ? w[(co * Ci + ck) * 9 + tap] : __float2bfloat16(0.f);
  }
  if (l > 0) {
    const int nd = 9 * Ci * Co;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nd; i += gridDim.x * blockDim.x) {
      const int co = i % Co, ci = (i / Co) % Ci, tap = i / (Co * Ci);
      Wd[t.wd_off[l] + i] = w[(co * Ci + ci) * 9 + tap];
    }
  }
}

void conv_weight_relayout(const void* shadow, const ConvLayerTable& t, void* Wf, void* Wd, int l0, int l1,
                          int spack0, int compact0, cudaStream_t st) {
  if (l1 <= l0) return;
  dim3 grid(32, l1 - l0);
  launch_pdl(conv_weight_relayout_kernel, dim3(grid), dim3(256), 0, st, reinterpret_cast<const __nv_bfloat16*>(shadow), t,
                                                    reinterpret_cast<__nv_bfloat16*>(Wf),
                                                    reinterpret_cast<__nv_bfloat16*>(Wd), l0, spack0, compact0);
  hefl::cuda::note_launch();
}

// dW32 [9*CK+1][Co] (wgrad output, row 9*CK = bias gradient) -> flat fp32 gradient in the
// parameter layout ([Co][Ci][3][3], then bias); clears dW32 for the next step.
__global__ void conv_grad_finalize_kernel(float* __restrict__ dW32, const ConvLayerTable t,
                                          float* __restrict__ grad, int l0) {
  pdl_prologue();
  const int l = blockIdx.y + l0;
  const int Ci = t.Ci[l], CK = t.CK[l], Co = t.Co[l];
  float* src = dW32 + t.dw_off[l];
  const int nw = Co * Ci * 9;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nw; i += gridDim.x * blockDim.x) {
    const int tap = i % 9, ci = (i / 9) % Ci, co = i / (9 * Ci);
    grad[t.w_off[l] + i] = src[(size_t)(tap * CK + ci) * Co + co];
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Co; i += gridDim.x * blockDim.x)
    grad[t.b_off[l] + i] = src[(size_t)9 * CK * Co + i];
}
__global__ void zero_f32_kernel(float* __restrict__ p, int64_t n) {
  pdl_prologue();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = 0.f;
}

void conv_grad_finalize(float* dW32, const ConvLayerTable& t, float* grad, int l0, int l1, cudaStream_t st) {
  if (l1 <= l0) return;
  dim3 grid(32, l1 - l0);
  launch_pdl(conv_grad_finalize_kernel, dim3(grid), dim3(256), 0, st, dW32, t, grad, l0);
  const int l = l1 - 1;
  const int64_t begin = t.dw_off[l0];
  const int64_t total = t.dw_off[l] + (int64_t)(9 * t.CK[l] + 1) * t.Co[l] - begin;
  launch_pdl(zero_f32_kernel, dim3(64), dim3(256), 0, st, dW32 + begin, total);
  hefl::cuda::note_launch(2);
}

}  // namespace nn
}  // namespace hefl

// ------------------------------------------------------------------------------------------
// Dense head of the sequential CNNs: Flatten -> Dense(H1, ReLU) -> Dense(H2, ReLU) -> Dense(C)
// -> softmax cross-entropy (FLPyfhelin.py:133-136, :141), forward AND backward in four launches
// (K16/K17). ~13 MFLOP at batch 32: latency- and shared-memory-bound, so the work is spread over
// many CTAs per phase, operands are staged with all loads in flight, and every thread reuses
// each shared-memory operand for several FMAs.
//   k1  h1 = relu(feat W1^T + b1)                                  grid H1/4
//   k2  h2, logits, loss, dlogits, dW3, db3, dh2                   1 CTA (0.3 MFLOP)
//   k3  dW2, db2, dh1 (column slices of 16)                        grid H1/16
//   k4  dW1, db1, dfeat (column slices of 16)                      grid F/16
// A head-only step (depth 2 / 3 / 4, DESIGN.md §10) skips dfeat, k4, or k3 and k4 with k2's dh2. Grad-CAM
// (kHeadSaliency, DESIGN.md §11) seeds k2's dlogits with a one-hot target, writes the logits and runs k3 and k4 without
// their dW / db (null gradient pointers). Federated evaluation (kHeadScore, DESIGN.md §13) runs k1 and k2 up to the
// logits, which it writes, and nothing after them.
// ------------------------------------------------------------------------------------------
namespace hefl {
namespace nn {

// k1: one CTA = 4 neurons; thread = (sample b, neuron jj); feat and the 4 weight rows in smem.
__global__ void __launch_bounds__(128)
head_fc1_fwd_kernel(const __nv_bfloat16* __restrict__ feat, const float* __restrict__ W1,
                    const float* __restrict__ b1, float* __restrict__ h1, int B, int F, int H1) {
  pdl_trigger();
  extern __shared__ float sm1[];
  const int FP = F + 1;
  float* fs = sm1;                 // [B][F+1]
  float* ws = fs + B * FP;         // [4][F+1]
  const int j0 = blockIdx.x * 4;
  const int F8 = F >> 3, F4 = F >> 2;
  const uint4* src = reinterpret_cast<const uint4*>(feat);
  // weights first: they do not depend on the previous kernel, so this overlaps its tail (PDL)
#pragma unroll 4
  for (int i = threadIdx.x; i < 4 * F4; i += blockDim.x) {
    const int jj = i / F4, k4 = i - jj * F4;
    const float4 v = (j0 + jj) < H1 ? reinterpret_cast<const float4*>(W1 + (size_t)(j0 + jj) * F)[k4]
                                     : make_float4(0.f, 0.f, 0.f, 0.f);
    float* dst = ws + jj * FP + k4 * 4;
    dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
  }
  pdl_wait();
#pragma unroll 8
  for (int i = threadIdx.x; i < B * F8; i += blockDim.x) {   // B*F/8 16-byte loads, 8+ in flight per thread
    const uint4 v = src[i];
    const int b = i / F8, k8 = i - b * F8;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float* dst = fs + b * FP + k8 * 8;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      dst[2 * q] = __uint_as_float(w[q] << 16);
      dst[2 * q + 1] = __uint_as_float(w[q] & 0xFFFF0000u);
    }
  }
  __syncthreads();
  const int b = threadIdx.x >> 2, jj = threadIdx.x & 3;
  if (b < B && j0 + jj < H1) {
    const float* fr = fs + b * FP;
    const float* wr = ws + jj * FP;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = 0;
#pragma unroll 4
    for (; k + 4 <= F; k += 4) {
      a0 = fmaf(fr[k], wr[k], a0);
      a1 = fmaf(fr[k + 1], wr[k + 1], a1);
      a2 = fmaf(fr[k + 2], wr[k + 2], a2);
      a3 = fmaf(fr[k + 3], wr[k + 3], a3);
    }
    for (; k < F; ++k) a0 = fmaf(fr[k], wr[k], a0);
    const float acc = (a0 + a1) + (a2 + a3) + b1[j0 + jj];
    h1[b * H1 + j0 + jj] = acc > 0.f ? acc : 0.f;
  }
}

struct HeadMidArgs {
  const float* h1;      // [B][H1]
  const float *W2, *b2, *W3, *b3;
  const int64_t* y;     // [B]
  float *gW3, *gb3;
  float* dh2;           // [B][H2] out
  float* out;           // [2]: loss, ncorrect
  float* logits;        // [B][C], kHeadSaliency and kHeadScore only
  int B, H1, H2, C, depth;
};

// k2: fc2 (each thread: 2 samples x 4 neurons, operands reused from registers), fc3, loss, dW3, dh2.
__global__ void __launch_bounds__(256)
head_mid_kernel(const HeadMidArgs a) {
  pdl_trigger();
  extern __shared__ float sm[];
  const int B = a.B, H1 = a.H1, H2 = a.H2, C = a.C;
  float* h1 = sm;                       // [B][H1+1]
  float* W2 = h1 + B * (H1 + 1);        // [H2][H1+1]
  float* h2 = W2 + H2 * (H1 + 1);       // [B][H2+1]
  float* lg = h2 + B * (H2 + 1);        // [B][C]  logits -> dlogits
  float* red = lg + B * C;              // [2*B]
  float* W3 = red + 2 * B;              // [C][H2]
  const int tid = threadIdx.x, nt = blockDim.x;
  const int H14 = H1 >> 2;
#pragma unroll 8
  for (int i = tid; i < H2 * H14; i += nt) {
    const float4 v = reinterpret_cast<const float4*>(a.W2)[i];
    float* d = W2 + (i / H14) * (H1 + 1) + (i % H14) * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
  for (int i = tid; i < C * H2; i += nt) W3[i] = a.W3[i];
  pdl_wait();          // weights staged above overlap the previous kernel; activations only from here
#pragma unroll 4
  for (int i = tid; i < B * H14; i += nt) {
    const float4 v = reinterpret_cast<const float4*>(a.h1)[i];
    float* d = h1 + (i / H14) * (H1 + 1) + (i % H14) * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
  __syncthreads();
  {  // fc2: tiles of 2 samples x 4 neurons
    const int tiles_j = H2 >> 2, tiles = (B >> 1) * tiles_j;
    for (int t = tid; t < tiles; t += nt) {
      const int b0 = (t / tiles_j) * 2, j0 = (t % tiles_j) * 4;
      float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      for (int i = 0; i < H1; ++i) {
        const float x0 = h1[b0 * (H1 + 1) + i], x1 = h1[(b0 + 1) * (H1 + 1) + i];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float w = W2[(j0 + q) * (H1 + 1) + i];
          acc[0][q] = fmaf(x0, w, acc[0][q]);
          acc[1][q] = fmaf(x1, w, acc[1][q]);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float bb = a.b2[j0 + q];
        const float y0 = acc[0][q] + bb, y1 = acc[1][q] + bb;
        h2[b0 * (H2 + 1) + j0 + q] = y0 > 0.f ? y0 : 0.f;
        h2[(b0 + 1) * (H2 + 1) + j0 + q] = y1 > 0.f ? y1 : 0.f;
      }
    }
  }
  __syncthreads();
  for (int o = tid; o < B * C; o += nt) {                      // fc3
    const int b = o / C, c = o % C;
    float a0 = a.b3[c], a1 = 0.f;
    int j = 0;
    for (; j + 2 <= H2; j += 2) {
      a0 = fmaf(h2[b * (H2 + 1) + j], W3[c * H2 + j], a0);
      a1 = fmaf(h2[b * (H2 + 1) + j + 1], W3[c * H2 + j + 1], a1);
    }
    for (; j < H2; ++j) a0 = fmaf(h2[b * (H2 + 1) + j], W3[c * H2 + j], a0);
    lg[o] = a0 + a1;
  }
  __syncthreads();
  if (tid < 32) {                                              // warp 0: softmax cross-entropy, one lane per sample
    float l = 0.f, nc = 0.f;
    if (tid < B) {
      float mx = -1e30f;
      int am = 0;
      for (int c = 0; c < C; ++c) if (lg[tid * C + c] > mx) { mx = lg[tid * C + c]; am = c; }
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += __expf(lg[tid * C + c] - mx);
      if (a.depth == kHeadScore) {                             // logits only: no labels, loss or backward
        for (int c = 0; c < C; ++c) a.logits[tid * C + c] = lg[tid * C + c];
      } else if (a.depth == kHeadSaliency) {                   // d logits[b, target] / d logits: one-hot
        const int yy = (int)a.y[tid];
        const int tt = yy < 0 ? am : yy;
        for (int c = 0; c < C; ++c) {
          a.logits[tid * C + c] = lg[tid * C + c];
          lg[tid * C + c] = c == tt ? 1.f : 0.f;
        }
      } else {
        const int yy = (int)a.y[tid];
        l = -(lg[tid * C + yy] - mx - __logf(s));
        nc = am == yy ? 1.f : 0.f;
        const float invB = 1.f / B;
        for (int c = 0; c < C; ++c) {
          const float p = __expf(lg[tid * C + c] - mx) / s;
          lg[tid * C + c] = (p - (c == yy ? 1.f : 0.f)) * invB;   // dlogits
        }
      }
    }
    for (int off = 16; off; off >>= 1) {                       // all 32 lanes take part (B <= 32)
      l += __shfl_xor_sync(0xffffffffu, l, off);
      nc += __shfl_xor_sync(0xffffffffu, nc, off);
    }
    if (tid == 0 && a.depth < kHeadSaliency) {
      a.out[0] = l / B;
      a.out[1] = nc;
    }
  }
  __syncthreads();
  if (!a.depth || a.depth == kHeadScore) return;
  for (int o = tid; a.depth != kHeadSaliency && o < C * H2 + C; o += nt) {   // dW3, db3
    if (o < C * H2) {
      const int c = o / H2, j = o % H2;
      float acc = 0.f;
      for (int b = 0; b < B; ++b) acc = fmaf(lg[b * C + c], h2[b * (H2 + 1) + j], acc);
      a.gW3[o] = acc;
    } else {
      const int c = o - C * H2;
      float acc = 0.f;
      for (int b = 0; b < B; ++b) acc += lg[b * C + c];
      a.gb3[c] = acc;
    }
  }
  if (a.depth == 4) return;
  for (int o = tid; o < B * H2; o += nt) {                     // dh2 -> global for k3
    const int b = o / H2, j = o % H2;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fmaf(lg[b * C + c], W3[c * H2 + j], acc);
    a.dh2[o] = h2[b * (H2 + 1) + j] > 0.f ? acc : 0.f;
  }
}

// k3: one CTA owns 16 columns i of layer 2's input: dW2[:, i], dh1[:, i]; CTA 0 also db2.
__global__ void __launch_bounds__(256)
head_fc2_bwd_kernel(const float* __restrict__ dh2g, const float* __restrict__ h1g, const float* __restrict__ W2,
                    float* __restrict__ gW2, float* __restrict__ gb2, float* __restrict__ dh1, int B, int H1, int H2) {
  pdl_trigger();
  extern __shared__ float sm[];
  float* d = sm;                       // [B][H2+1]
  float* hs = d + B * (H2 + 1);        // [B][16]
  float* ws = hs + B * 16;             // [H2][17]
  const int tid = threadIdx.x, nt = blockDim.x;
  const int i0 = blockIdx.x * 16;
#pragma unroll 4
  for (int i = tid; i < H2 * 16; i += nt) ws[(i >> 4) * 17 + (i & 15)] = (i0 + (i & 15)) < H1 ? W2[(size_t)(i >> 4) * H1 + i0 + (i & 15)] : 0.f;
  pdl_wait();
#pragma unroll 4
  for (int i = tid; i < B * H2; i += nt) d[(i / H2) * (H2 + 1) + i % H2] = dh2g[i];
#pragma unroll 2
  for (int i = tid; i < B * 16; i += nt) hs[i] = (i0 + (i & 15)) < H1 ? h1g[(i >> 4) * H1 + i0 + (i & 15)] : 0.f;
  __syncthreads();
  for (int o = tid; gW2 != nullptr && o < H2 * 16; o += nt) {  // dW2[j][i0+k]
    const int j = o >> 4, k = o & 15;
    float a0 = 0.f, a1 = 0.f;
    int b = 0;
    for (; b + 2 <= B; b += 2) {
      a0 = fmaf(d[b * (H2 + 1) + j], hs[b * 16 + k], a0);
      a1 = fmaf(d[(b + 1) * (H2 + 1) + j], hs[(b + 1) * 16 + k], a1);
    }
    for (; b < B; ++b) a0 = fmaf(d[b * (H2 + 1) + j], hs[b * 16 + k], a0);
    if (i0 + k < H1) gW2[(size_t)j * H1 + i0 + k] = a0 + a1;
  }
  for (int o = tid; o < B * 16; o += nt) {                     // dh1[b][i0+k]
    const int b = o >> 4, k = o & 15;
    float a0 = 0.f, a1 = 0.f;
    int j = 0;
    for (; j + 2 <= H2; j += 2) {
      a0 = fmaf(d[b * (H2 + 1) + j], ws[j * 17 + k], a0);
      a1 = fmaf(d[b * (H2 + 1) + j + 1], ws[(j + 1) * 17 + k], a1);
    }
    for (; j < H2; ++j) a0 = fmaf(d[b * (H2 + 1) + j], ws[j * 17 + k], a0);
    if (i0 + k < H1) dh1[b * H1 + i0 + k] = hs[b * 16 + k] > 0.f ? (a0 + a1) : 0.f;
  }
  if (blockIdx.x == 0 && gb2 != nullptr) {
    for (int j = tid; j < H2; j += nt) {
      float acc = 0.f;
      for (int b = 0; b < B; ++b) acc += d[b * (H2 + 1) + j];
      gb2[j] = acc;
    }
  }
}

// k4: dW1[j][k] = sum_b dh1[b][j] feat[b][k]; db1[j] = sum_b dh1[b][j]; dfeat[b][k] = sum_j dh1[b][j] W1[j][k].
// One CTA owns 16 input columns k.
__global__ void __launch_bounds__(256)
head_fc1_bwd_kernel(const float* __restrict__ dh1, const __nv_bfloat16* __restrict__ feat,
                    const float* __restrict__ W1, float* __restrict__ gW1, float* __restrict__ gb1,
                    __nv_bfloat16* __restrict__ dfeat, int B, int F, int H1) {
  pdl_trigger();
  extern __shared__ float sm[];
  float* d = sm;                       // [B][H1+1]
  float* fs = d + B * (H1 + 1);        // [B][16]
  float* ws = fs + B * 16;             // [H1][17]
  const int tid = threadIdx.x, nt = blockDim.x;
  const int k0 = blockIdx.x * 16;
#pragma unroll 8
  for (int i = tid; i < H1 * 16; i += nt) {
    const int j = i >> 4, k = i & 15;
    ws[j * 17 + k] = k0 + k < F ? W1[(size_t)j * F + k0 + k] : 0.f;
  }
  pdl_wait();
#pragma unroll 8
  for (int i = tid; i < B * H1; i += nt) d[(i / H1) * (H1 + 1) + i % H1] = dh1[i];
#pragma unroll 2
  for (int i = tid; i < B * 16; i += nt) {
    const int b = i >> 4, k = i & 15;
    fs[i] = k0 + k < F ? __bfloat162float(feat[b * F + k0 + k]) : 0.f;
  }
  __syncthreads();
  for (int o = tid; gW1 != nullptr && o < H1 * 16; o += nt) {
    const int j = o >> 4, k = o & 15;
    float a0 = 0.f, a1 = 0.f;
    int b = 0;
    for (; b + 2 <= B; b += 2) {
      a0 = fmaf(d[b * (H1 + 1) + j], fs[b * 16 + k], a0);
      a1 = fmaf(d[(b + 1) * (H1 + 1) + j], fs[(b + 1) * 16 + k], a1);
    }
    for (; b < B; ++b) a0 = fmaf(d[b * (H1 + 1) + j], fs[b * 16 + k], a0);
    if (k0 + k < F) gW1[(size_t)j * F + k0 + k] = a0 + a1;
  }
  for (int o = tid; dfeat != nullptr && o < B * 16; o += nt) {
    const int b = o >> 4, k = o & 15;
    float a0 = 0.f, a1 = 0.f;
    int j = 0;
    for (; j + 2 <= H1; j += 2) {
      a0 = fmaf(d[b * (H1 + 1) + j], ws[j * 17 + k], a0);
      a1 = fmaf(d[b * (H1 + 1) + j + 1], ws[(j + 1) * 17 + k], a1);
    }
    for (; j < H1; ++j) a0 = fmaf(d[b * (H1 + 1) + j], ws[j * 17 + k], a0);
    if (k0 + k < F) dfeat[b * F + k0 + k] = __float2bfloat16(a0 + a1);
  }
  if (blockIdx.x == 0 && gb1 != nullptr) {
    for (int j = tid; j < H1; j += nt) {
      float acc = 0.f;
      for (int b = 0; b < B; ++b) acc += d[b * (H1 + 1) + j];
      gb1[j] = acc;
    }
  }
}

void head_forward_backward(const void* feat, const float* W1, const float* b1, const float* W2, const float* b2,
                           const float* W3, const float* b3, const int64_t* y, float* gW1, float* gb1, float* gW2,
                           float* gb2, float* gW3, float* gb3, void* dfeat, float* h1_buf, float* dh1_buf,
                           float* out, float* logits, int B, int F, int H1, int H2, int C, int depth,
                           cudaStream_t st) {
  const auto* f = reinterpret_cast<const __nv_bfloat16*>(feat);
  const bool saliency = depth == kHeadSaliency;
  float* dh2_buf = dh1_buf + (size_t)B * H1;                  // scratch tail: [B][H2]
  const int smem_a = (B + 4) * (F + 1) * 4;
  cudaFuncSetAttribute(head_fc1_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_a);
  launch_pdl(head_fc1_fwd_kernel, dim3((H1 + 3) / 4), dim3(128), smem_a, st, f, W1, b1, h1_buf, B, F, H1);
  HeadMidArgs a{h1_buf, W2, b2, W3, b3, y, gW3, gb3, dh2_buf, out, logits, B, H1, H2, C, depth};
  const int smem_b = (B * (H1 + 1) + H2 * (H1 + 1) + B * (H2 + 1) + B * C + 2 * B + C * H2) * 4;
  cudaFuncSetAttribute(head_mid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_b);
  launch_pdl(head_mid_kernel, dim3(1), dim3(256), smem_b, st, a);
  hefl::cuda::note_launch(2);
  if ((depth >= 1 && depth <= 3) || saliency) {
    const int smem_c = (B * (H2 + 1) + B * 16 + H2 * 17) * 4;
    launch_pdl(head_fc2_bwd_kernel, dim3((H1 + 15) / 16), dim3(256), smem_c, st, dh2_buf, h1_buf, W2,
               saliency ? nullptr : gW2, saliency ? nullptr : gb2, dh1_buf, B, H1, H2);
    hefl::cuda::note_launch();
  }
  if (depth == 1 || depth == 2 || saliency) {
    const int smem_d = (B * (H1 + 1) + B * 16 + H1 * 17) * 4;
    cudaFuncSetAttribute(head_fc1_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_d);
    launch_pdl(head_fc1_bwd_kernel, dim3((F + 15) / 16), dim3(256), smem_d, st, dh1_buf, f, W1,
               saliency ? nullptr : gW1, saliency ? nullptr : gb1,
               depth == 2 ? nullptr : reinterpret_cast<__nv_bfloat16*>(dfeat), B, F, H1);
    hefl::cuda::note_launch();
  }
}

}  // namespace nn
}  // namespace hefl
