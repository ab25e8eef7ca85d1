// Dense head of the medical CNN — Flatten -> Dense(128, ReLU) -> Dense(64, ReLU) -> Dense(C) -> softmax
// cross-entropy (FLPyfhelin.py:133-136, :141) — forward AND backward in ONE launch on a thread-block
// cluster of 8 CTAs (K16/K17).
//
// ~13 MFLOP at batch 32: pure latency. The 4-kernel version measured 50 us in the step graph (4 launch
// ramps, 4 rounds of staging, one single-CTA phase). Here the 8 CTAs of a cluster each own a slice of
// every layer and exchange the small activations through distributed shared memory:
//   P0  (before griddepcontrol.wait, overlapping the last conv kernel) stage this CTA's weight slices:
//       W1 rows of its 16 neurons, W1 columns of its 64 input features, W2 rows / columns, W3
//   P1  h1[:, own 16]  = relu(feat W1^T + b1)            -> written into all 8 CTAs' h1 (DSMEM), cluster.sync
//   P2  h2[:, own 8]   = relu(h1 W2^T + b2)              -> all-gather, cluster.sync
//   P3  logits, loss, accuracy, dlogits (every CTA, 64 outputs); CTA 0 writes loss / dW3 / db3;
//       dh2[:, own 8]                                     -> all-gather, cluster.sync
//   P4  dW2 / db2 (own rows), dh1[:, own 16]              -> all-gather (transposed), cluster.sync
//   P5  dW1 / db1 (own rows), dfeat[:, own 64 features]   (needs all dh1 and the W1 column slice)
// ``depth`` says how far the backward runs: 0 eval (P3's loss only), 1 everything, and for a head-only step of
// personalised federated learning (DESIGN.md §10) 2 = P5 without dfeat, 3 = up to P4's dW2 / db2, 4 = up to P3's
// dW3 / db3. Every early exit follows the last cluster barrier after which no CTA writes into another's shared memory.
// depth 5 (kHeadSaliency, Grad-CAM, DESIGN.md §11) seeds the backward with the one-hot of a target class (-1: the
// arg-max of the logits) instead of p - y, CTA 0 writes the logits, and P3-P5 skip every dW / db: dfeat only.
// depth 6 (kHeadScore, federated evaluation, DESIGN.md §13) runs P1-P3, CTA 0 writes the logits, and the kernel exits
// where depth 0 exits: no label is read and no loss, gradient or dfeat is written.
// Four cluster barriers replace three kernel boundaries; nothing but parameters gradients, dfeat and the
// two result scalars touches global memory.
#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include "../he/kernels.h"
#include "launch.cuh"
#include "nn.h"

namespace cg = cooperative_groups;

namespace hefl {
namespace nn {

namespace hc {
constexpr int R = 8;              // cluster size
constexpr int F = 512, H1 = 128, H2 = 64;
constexpr int J1 = H1 / R;        // 16 fc1 neurons per CTA
constexpr int J2 = H2 / R;        // 8 fc2 neurons per CTA
constexpr int KS = F / R;         // 64 input features per CTA (dfeat slice)
constexpr int BM = 32;            // max batch
constexpr int CM = 4;             // max classes
constexpr int FP = F + 4;         // padded row pitches (floats): float4 rows land on distinct banks
constexpr int H1P = H1 + 4;
constexpr int H2P = H2 + 4;
constexpr int NT = 256;
// shared-memory layout (floats)
constexpr int O_FEAT = 0;                          // [BM][FP]
constexpr int O_W1R = O_FEAT + BM * FP;            // [J1][FP]     W1 rows of the own neurons
constexpr int O_W1C = O_W1R + J1 * FP;             // [H1][KS]     W1[:, own 64 features]
constexpr int O_W2R = O_W1C + H1 * KS;             // [J2][H1P]    W2 rows of the own fc2 neurons
constexpr int O_W2C = O_W2R + J2 * H1P;            // [H2][J1]     W2[:, own 16 fc1 neurons]
constexpr int O_W3 = O_W2C + H2 * J1;              // [CM][H2]
constexpr int O_H1 = O_W3 + CM * H2;               // [BM][H1P]    full h1 (all-gathered)
constexpr int O_H2 = O_H1 + BM * H1P;              // [BM][H2P]
constexpr int O_LG = O_H2 + BM * H2P;              // [BM][CM]     logits -> dlogits
constexpr int O_DH2 = O_LG + BM * CM;              // [BM][H2P]
constexpr int O_DH1 = O_DH2 + BM * H2P;            // [H1][BM]     dh1 transposed
constexpr int TOTAL = O_DH1 + H1 * BM;
constexpr int SMEM_BYTES = TOTAL * 4;
}  // namespace hc

struct HeadClusterArgs {
  const __nv_bfloat16* feat;   // [B][F]
  const float *W1, *b1, *W2, *b2, *W3, *b3;
  const int64_t* y;
  float *gW1, *gb1, *gW2, *gb2, *gW3, *gb3;
  __nv_bfloat16* dfeat;        // [B][F]
  float* out;                  // [2] loss, ncorrect
  float* logits;               // [B][C], kHeadSaliency and kHeadScore only
  int B, C, depth;           // 0 eval, 1 full backward, 2 / 3 / 4 stop after dW1 / dW2 / dW3 (no dfeat), kHeadSaliency,
                             // kHeadScore
};

__global__ void __launch_bounds__(hc::NT, 1) head_cluster_kernel(const HeadClusterArgs a) {
  using namespace hc;
  extern __shared__ __align__(16) float sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int r = (int)cluster.block_rank();
  const int t = threadIdx.x;
  const int B = a.B, C = a.C;
  float* featS = sm + O_FEAT;
  float* w1r = sm + O_W1R;
  float* w1c = sm + O_W1C;
  float* w2r = sm + O_W2R;
  float* w2c = sm + O_W2C;
  float* w3 = sm + O_W3;
  float* h1S = sm + O_H1;
  float* h2S = sm + O_H2;
  float* lgS = sm + O_LG;
  float* dh2S = sm + O_DH2;
  float* dh1S = sm + O_DH1;

  // ---- P0: weight slices (parameters are only written by kernels that never trigger early: launch.cuh)
  pdl_trigger();
  {
    const float4* src = reinterpret_cast<const float4*>(a.W1 + (size_t)r * J1 * F);     // 16 contiguous rows
#pragma unroll 4
    for (int i = t; i < J1 * F / 4; i += NT) {
      const int row = i / (F / 4), c4 = i - row * (F / 4);
      *reinterpret_cast<float4*>(w1r + row * FP + c4 * 4) = __ldg(src + i);
    }
#pragma unroll 4
    for (int i = t; i < H1 * KS / 4; i += NT) {                                           // 128 rows x 16 float4
      const int j = i / (KS / 4), c4 = i - j * (KS / 4);
      *reinterpret_cast<float4*>(w1c + j * KS + c4 * 4) =
          __ldg(reinterpret_cast<const float4*>(a.W1 + (size_t)j * F + r * KS) + c4);
    }
    for (int i = t; i < J2 * H1 / 4; i += NT) {
      const int row = i / (H1 / 4), c4 = i - row * (H1 / 4);
      *reinterpret_cast<float4*>(w2r + row * H1P + c4 * 4) =
          __ldg(reinterpret_cast<const float4*>(a.W2 + (size_t)(r * J2 + row) * H1) + c4);
    }
    for (int i = t; i < H2 * J1 / 4; i += NT) {
      const int j = i / (J1 / 4), c4 = i - j * (J1 / 4);
      *reinterpret_cast<float4*>(w2c + j * J1 + c4 * 4) =
          __ldg(reinterpret_cast<const float4*>(a.W2 + (size_t)j * H1 + r * J1) + c4);
    }
    for (int i = t; i < C * H2; i += NT) w3[i] = __ldg(a.W3 + i);
  }
  pdl_wait();
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.feat);
#pragma unroll 4
    for (int i = t; i < B * F / 8; i += NT) {
      const uint4 v = src[i];
      const int b = i / (F / 8), k8 = i - b * (F / 8);
      float* dst = featS + b * FP + k8 * 8;
      *reinterpret_cast<float4*>(dst) = make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xFFFF0000u),
                                                    __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xFFFF0000u));
      *reinterpret_cast<float4*>(dst + 4) = make_float4(__uint_as_float(v.z << 16), __uint_as_float(v.z & 0xFFFF0000u),
                                                        __uint_as_float(v.w << 16), __uint_as_float(v.w & 0xFFFF0000u));
    }
  }
  // every CTA of the cluster has started (its shared memory is live) before anyone writes into it
  cluster.sync();

  // ---- P1: h1[:, own 16]. Register-tiled: every lane owns a 4-sample x 4-neuron tile and every warp one
  // eighth of K (8 LDS.128 per 64 FMAs; the first version did 3 LDS.128 per 8 FMAs and spent 30 % of the
  // kernel here, shared-memory bound). Partial sums of the 8 warps meet in shared memory (the dh1 buffer is
  // idle until P4).
  {
    const int lane = t & 31, warp = t >> 5;
    const int bi = lane >> 2, ji = lane & 3;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const float* fbase = featS + (4 * bi) * FP + warp * (F / 8);
    const float* wbase = w1r + (4 * ji) * FP + warp * (F / 8);
#pragma unroll 2
    for (int k = 0; k < F / 8; k += 4) {
      float4 f[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        f[i] = *reinterpret_cast<const float4*>(fbase + i * FP + k);
        w[i] = *reinterpret_cast<const float4*>(wbase + i * FP + k);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[i][j] = fmaf(f[i].x, w[j].x, acc[i][j]);
          acc[i][j] = fmaf(f[i].y, w[j].y, acc[i][j]);
          acc[i][j] = fmaf(f[i].z, w[j].z, acc[i][j]);
          acc[i][j] = fmaf(f[i].w, w[j].w, acc[i][j]);
        }
    }
    float* part = dh1S + warp * (BM * J1);                    // [8 warps][32 samples][16 neurons]
#pragma unroll
    for (int i = 0; i < 4; ++i)
      *reinterpret_cast<float4*>(part + (4 * bi + i) * J1 + 4 * ji) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    __syncthreads();
    const int b = t >> 3, jq = t & 7;
    if (b < B) {
      float v0 = 0.f, v1 = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        v0 += dh1S[w * (BM * J1) + b * J1 + jq];
        v1 += dh1S[w * (BM * J1) + b * J1 + jq + 8];
      }
      const int j0 = r * J1 + jq, j1 = j0 + 8;
      v0 += __ldg(a.b1 + j0);
      v1 += __ldg(a.b1 + j1);
      v0 = v0 > 0.f ? v0 : 0.f;
      v1 = v1 > 0.f ? v1 : 0.f;
#pragma unroll
      for (int d = 0; d < R; ++d) {
        float* rem = cluster.map_shared_rank(h1S, d);
        rem[b * H1P + j0] = v0;
        rem[b * H1P + j1] = v1;
      }
    }
  }
  cluster.sync();

  // ---- P2: h2[:, own 8]
  {
    const int b = t >> 3, jj = t & 7;
    if (b < B) {
      const float4* h4 = reinterpret_cast<const float4*>(h1S + b * H1P);
      const float4* w4 = reinterpret_cast<const float4*>(w2r + jj * H1P);
      float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
      for (int k = 0; k < H1 / 4; ++k) {
        const float4 h = h4[k], w = w4[k];
        a0 = fmaf(h.x, w.x, a0); a1 = fmaf(h.y, w.y, a1); a0 = fmaf(h.z, w.z, a0); a1 = fmaf(h.w, w.w, a1);
      }
      const int j = r * J2 + jj;
      float v = a0 + a1 + __ldg(a.b2 + j);
      v = v > 0.f ? v : 0.f;
#pragma unroll
      for (int d = 0; d < R; ++d) cluster.map_shared_rank(h2S, d)[b * H2P + j] = v;
    }
  }
  cluster.sync();

  // ---- P3: logits / loss (every CTA redundantly: 64 outputs), dW3 (CTA 0), dh2[:, own 8]
  if (t < B * C) {
    const int b = t / C, c = t - b * C;
    float a0 = __ldg(a.b3 + c), a1 = 0.f;
#pragma unroll 8
    for (int j = 0; j < H2; j += 2) {
      a0 = fmaf(h2S[b * H2P + j], w3[c * H2 + j], a0);
      a1 = fmaf(h2S[b * H2P + j + 1], w3[c * H2 + j + 1], a1);
    }
    lgS[b * CM + c] = a0 + a1;
  }
  __syncthreads();
  if (t < 32) {                                               // one lane per sample
    float l = 0.f, nc = 0.f;
    if (t < B) {
      float mx = -1e30f;
      int am = 0;
      for (int c = 0; c < C; ++c) if (lgS[t * CM + c] > mx) { mx = lgS[t * CM + c]; am = c; }
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += __expf(lgS[t * CM + c] - mx);
      if (a.depth == kHeadScore) {                           // logits only: no labels, loss or backward
        if (r == 0)
          for (int c = 0; c < C; ++c) a.logits[t * C + c] = lgS[t * CM + c];
      } else if (a.depth == kHeadSaliency) {                 // d logits[t, target] / d logits: one-hot
        const int yy = (int)a.y[t];
        const int tt = yy < 0 ? am : yy;
        for (int c = 0; c < C; ++c) {
          if (r == 0) a.logits[t * C + c] = lgS[t * CM + c];
          lgS[t * CM + c] = c == tt ? 1.f : 0.f;
        }
      } else {
        const int yy = (int)a.y[t];
        l = -(lgS[t * CM + yy] - mx - __logf(s));
        nc = am == yy ? 1.f : 0.f;
        const float invB = 1.f / B;
        for (int c = 0; c < C; ++c) {
          const float p = __expf(lgS[t * CM + c] - mx) / s;
          lgS[t * CM + c] = (p - (c == yy ? 1.f : 0.f)) * invB;   // dlogits
        }
      }
    }
    for (int off = 16; off; off >>= 1) {
      l += __shfl_xor_sync(0xffffffffu, l, off);
      nc += __shfl_xor_sync(0xffffffffu, nc, off);
    }
    if (t == 0 && r == 0 && a.depth < kHeadSaliency) {
      a.out[0] = l / B;
      a.out[1] = nc;
    }
  }
  __syncthreads();
  if (!a.depth || a.depth == kHeadScore) return;   // nobody writes into this CTA's shared memory after the P2 barrier
  const bool params = a.depth != kHeadSaliency;
  if (r == 0 && params) {
    for (int o = t; o < C * H2 + C; o += NT) {
      if (o < C * H2) {
        const int c = o / H2, j = o - c * H2;
        float acc = 0.f;
        for (int b = 0; b < B; ++b) acc = fmaf(lgS[b * CM + c], h2S[b * H2P + j], acc);
        a.gW3[o] = acc;
      } else {
        const int c = o - C * H2;
        float acc = 0.f;
        for (int b = 0; b < B; ++b) acc += lgS[b * CM + c];
        a.gb3[c] = acc;
      }
    }
  }
  if (a.depth == 4) return;      // as above: the dh2 all-gather below is the first remote write after P2
  {
    const int b = t >> 3, jj = t & 7;
    if (b < B) {
      const int j = r * J2 + jj;
      float acc = 0.f;
      for (int c = 0; c < C; ++c) acc = fmaf(lgS[b * CM + c], w3[c * H2 + j], acc);
      const float v = h2S[b * H2P + j] > 0.f ? acc : 0.f;
#pragma unroll
      for (int d = 0; d < R; ++d) cluster.map_shared_rank(dh2S, d)[b * H2P + j] = v;
    }
  }
  cluster.sync();

  // ---- P4: dW2 / db2 (own 8 rows), dh1[:, own 16]
  if (params) {
    const int i = t & (H1 - 1), jh = t >> 7;                   // 2 groups of 4 rows
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int b = 0; b < B; ++b) {
      const float h = h1S[b * H1P + i];
      const float4 d = *reinterpret_cast<const float4*>(dh2S + b * H2P + r * J2 + jh * 4);
      acc[0] = fmaf(d.x, h, acc[0]); acc[1] = fmaf(d.y, h, acc[1]);
      acc[2] = fmaf(d.z, h, acc[2]); acc[3] = fmaf(d.w, h, acc[3]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) a.gW2[(size_t)(r * J2 + jh * 4 + q) * H1 + i] = acc[q];
    if (t < J2) {
      float s = 0.f;
      for (int b = 0; b < B; ++b) s += dh2S[b * H2P + r * J2 + t];
      a.gb2[r * J2 + t] = s;
    }
  }
  if (a.depth == 3) return;      // the dh1 all-gather below is the first remote write after the P3 barrier
  {
    const int b = t >> 3, iq = t & 7;
    if (b < B) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
      for (int j = 0; j < H2; ++j) {
        const float d = dh2S[b * H2P + j];
        a0 = fmaf(d, w2c[j * J1 + iq], a0);
        a1 = fmaf(d, w2c[j * J1 + iq + 8], a1);
      }
      const int i0 = r * J1 + iq, i1 = i0 + 8;
      const float v0 = h1S[b * H1P + i0] > 0.f ? a0 : 0.f;
      const float v1 = h1S[b * H1P + i1] > 0.f ? a1 : 0.f;
#pragma unroll
      for (int d = 0; d < R; ++d) {
        float* rem = cluster.map_shared_rank(dh1S, d);
        rem[i0 * BM + b] = v0;
        rem[i1 * BM + b] = v1;
      }
    }
  }
  cluster.sync();

  // ---- P5: dW1 / db1 (own 16 rows), dfeat[:, own 64 features]
  if (params) {
    float acc[J1][2];
#pragma unroll
    for (int j = 0; j < J1; ++j) acc[j][0] = acc[j][1] = 0.f;
    for (int b = 0; b < B; ++b) {
      const float f0 = featS[b * FP + t], f1 = featS[b * FP + t + NT];
#pragma unroll
      for (int j = 0; j < J1; ++j) {
        const float d = dh1S[(r * J1 + j) * BM + b];
        acc[j][0] = fmaf(d, f0, acc[j][0]);
        acc[j][1] = fmaf(d, f1, acc[j][1]);
      }
    }
#pragma unroll
    for (int j = 0; j < J1; ++j) {
      a.gW1[(size_t)(r * J1 + j) * F + t] = acc[j][0];
      a.gW1[(size_t)(r * J1 + j) * F + t + NT] = acc[j][1];
    }
    if (t < J1) {
      float s = 0.f;
      for (int b = 0; b < B; ++b) s += dh1S[(r * J1 + t) * BM + b];
      a.gb1[r * J1 + t] = s;
    }
  }
  if (a.depth == 2) return;      // P5 reads and writes this CTA's shared memory only
  {
    const int kk = t & (KS - 1), bg = t >> 6;                   // 4 groups of 8 samples
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
#pragma unroll 4
    for (int j = 0; j < H1; ++j) {
      const float w = w1c[j * KS + kk];
      const float4 d0 = *reinterpret_cast<const float4*>(dh1S + j * BM + bg * 8);
      const float4 d1 = *reinterpret_cast<const float4*>(dh1S + j * BM + bg * 8 + 4);
      acc[0] = fmaf(d0.x, w, acc[0]); acc[1] = fmaf(d0.y, w, acc[1]);
      acc[2] = fmaf(d0.z, w, acc[2]); acc[3] = fmaf(d0.w, w, acc[3]);
      acc[4] = fmaf(d1.x, w, acc[4]); acc[5] = fmaf(d1.y, w, acc[5]);
      acc[6] = fmaf(d1.z, w, acc[6]); acc[7] = fmaf(d1.w, w, acc[7]);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int b = bg * 8 + q;
      if (b < B) a.dfeat[(size_t)b * F + r * KS + kk] = __float2bfloat16(acc[q]);
    }
  }
}

bool head_cluster_supported(int B, int F, int H1, int H2, int C) {
  return F == hc::F && H1 == hc::H1 && H2 == hc::H2 && B >= 1 && B <= hc::BM && C >= 1 && C <= hc::CM;
}

void head_cluster(const void* feat, const float* W1, const float* b1, const float* W2, const float* b2,
                  const float* W3, const float* b3, const int64_t* y, float* gW1, float* gb1, float* gW2, float* gb2,
                  float* gW3, float* gb3, void* dfeat, float* out, float* logits, int B, int C, int depth,
                  cudaStream_t st) {
  HeadClusterArgs a{reinterpret_cast<const __nv_bfloat16*>(feat), W1, b1, W2, b2, W3, b3, y, gW1, gb1, gW2, gb2, gW3, gb3,
                    reinterpret_cast<__nv_bfloat16*>(dfeat), out, logits, B, C, depth};
  cudaFuncSetAttribute(head_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, hc::SMEM_BYTES);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(hc::R);
  cfg.blockDim = dim3(hc::NT);
  cfg.dynamicSmemBytes = hc::SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = hc::R;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  cudaLaunchKernelEx(&cfg, head_cluster_kernel, a);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl
