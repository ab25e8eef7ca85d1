// Launchers of the NN kernels (csrc/nn/*.cu). Raw-pointer C++ API; see nn_bindings.cpp.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace hefl {
namespace nn {

// Fused Adam with Keras' legacy time-based decay (FLPyfhelin.py:140):
//   lr_t = lr * lr_scale / (1 + decay * (t-1)),  t = *step (already incremented)
// Updates p, m, v in place, zeroes g, optionally writes a bf16 shadow of p.
// FedProx: with an fp32 anchor (the round's global model) and mu != 0, the gradient is g + mu * (p - anchor).
void adam_step(float* p, float* g, float* m, float* v, void* shadow_bf16, int64_t n,
               const int64_t* step, const float* lr_scale, float lr, float decay, float beta1,
               float beta2, float eps, const float* anchor, float mu, cudaStream_t st);

// ---- tensor-core implicit-GEMM convolution (conv_tcgen05.cu) ----
// spack: the layer-1 input is packed by preprocess_u8 — s-packed when in_channels == 3 (weights [3][CO][16]),
// rs-packed when in_channels == 1 (weights [1][CO][16]); in_channels is not read without spack.
void conv_fwd_pool(const void* X, const void* Wf, const float* bias, void* out, uint8_t* argmax, int B, int H,
                   int W, int CK, int CO, int spack, int in_channels, cudaStream_t st);
bool conv_fwd_pool_pair_supported(int H, int W, int CK, int CO);
// compact: X is the [B*H*W, 4] RGB layer-1 input (R, G, B, 0; preprocess_u8 compact), Wf the [3 r][2 dx][32][16]
// weights (conv_weight_relayout compact0); CK = 16, CO = 32, W <= 256
void conv_fwd_pool_pair(const void* X, const void* Wf, const float* bias, void* out, uint8_t* argmax, int B, int H,
                        int W, int CK, int CO, int spack, int in_channels, int compact, cudaStream_t st);
void conv_set_debug(int mask);
void conv_dgrad(const void* dY, const void* Wd, void* dX, int B, int H, int W, int CK, int CO, cudaStream_t st);
// Split-K weight gradients write one partial per CTA into a workspace and add the partials to dW32 in a fixed order
// (fp32 atomics would make the sum, and so training, depend on timing). ws: conv_wgrad_ws_floats(...) floats.
int64_t conv_wgrad_ws_floats(int B, int H, int W, int CK, int Co);
void conv_wgrad(const void* X, const void* DY, float* dW32, float* ws, int B, int H, int W, int CK, int Co,
                cudaStream_t st);
// Both gradients of a CK = Co = 32 layer from one pass over dY: the same bits as conv_dgrad(dY, Wd, dX, .., 32, 32)
// and conv_wgrad(X, dY, dW32, .., 32, 32). ws: conv_dgrad_wgrad_ws_floats(...) floats.
bool conv_dgrad_wgrad_supported(int H, int W, int CK, int Co);
int64_t conv_dgrad_wgrad_ws_floats(int B, int H, int W);
void conv_dgrad_wgrad(const void* X, const void* dY, const void* Wd, void* dX, float* dW32, float* ws, int B, int H,
                      int W, int CK, int Co, cudaStream_t st);

// Dense head (Flatten -> Dense/ReLU -> Dense/ReLU -> Dense -> softmax-CE) forward + backward. depth: 0 forward and
// loss only, 1 every gradient and dfeat, 2 / 3 / 4 the gradients of the last 3 / 2 / 1 Dense layers and no dfeat.
// kHeadSaliency (Grad-CAM): y holds a target class per sample (-1: the arg-max of the logits, lowest index on ties),
// logits [B][C] are written, the backward is seeded with d logits[b, y_b] instead of the loss and yields dfeat only:
// no parameter gradient, no loss (gW* and out are not touched).
constexpr int kHeadSaliency = 5;
// kHeadScore (federated evaluation): the forward only; logits [B][C] are written, y is not read, and no loss, gradient
// or dfeat is written.
constexpr int kHeadScore = 6;
void head_forward_backward(const void* feat, const float* W1, const float* b1, const float* W2, const float* b2,
                           const float* W3, const float* b3, const int64_t* y, float* gW1, float* gb1, float* gW2,
                           float* gb2, float* gW3, float* gb3, void* dfeat, float* h1_buf, float* dh1_buf,
                           float* out, float* logits, int B, int F, int H1, int H2, int C, int depth, cudaStream_t st);
bool head_cluster_supported(int B, int F, int H1, int H2, int C);
void head_cluster(const void* feat, const float* W1, const float* b1, const float* W2, const float* b2,
                  const float* W3, const float* b3, const int64_t* y, float* gW1, float* gb1, float* gW2, float* gb2,
                  float* gW3, float* gb3, void* dfeat, float* out, float* logits, int B, int C, int depth,
                  cudaStream_t st);
// ---- Grad-CAM (gradcam.cu) ----
// X, G: bf16 [B*Hp*Hp][C] (a conv stage's output and the class score's gradient at it), C a multiple of 8 up to 128.
// out: fp32 [nvalid][S][S], the bilinear (half-pixel) upsampling of relu(sum_c mean_hw(G) X) divided by the maximum of
// the Hp x Hp map (0 where that maximum is 0). Scans >= nvalid are neither read nor written.
bool gradcam_supported(int Hp, int C, int S);
void gradcam(const void* X, const void* G, float* out, int Hp, int C, int S, int nvalid, cudaStream_t st);
// ---- layer-1 input gradient (input_grad.cu, DESIGN.md §12) ----
// g: bf16 [B*Hp*Hp][32], the gradient at layer 1's pooled output, Hp = (S - 2) / 2; amax: its codes (bits 0-1 arg-max
// position, bit 2 active unit); w: layer 1's bf16 weights [32][in_channels][3][3]. acc: fp32 [nvalid][S][S]
// [in_channels] += the full correlation of the conv-grid gradient (g at the arg-max of every active window, 0 elsewhere)
// with w, in_channels 1 or 3. Scans >= nvalid are neither read nor written.
void input_grad0(const void* g, const uint8_t* amax, const void* w, float* acc, int S, int Hp, int in_channels,
                 int nvalid, cudaStream_t st);
// ---- federated evaluation counts (score.cu, DESIGN.md §13) ----
// logits fp32 [B][C], labels int64 [B], *nvalid (device): rows >= nvalid are neither read nor written. probs fp32
// [B][C] = softmax(logits). counts int32 [C*C + C*C*nbins] += the confusion matrix conf[t][argmax] and the score
// histograms hist[t][c][min(nbins - 1, floor(p_c * nbins))]; *loss_sum (fp64) += the cross-entropy of the rows, summed
// in a fixed order by one thread. A label outside 0..C-1 sets *err to 1 and its row adds nothing.
constexpr int kScoreMaxClasses = 32;
void score_stats(const float* logits, const int64_t* labels, const int* nvalid, float* probs, int* counts,
                 double* loss_sum, int* err, int B, int C, int nbins, cudaStream_t st);
bool wgrad0_gather_supported(int W, int Wp, int CK, int Ci, int Co);
// layer-1 partials: [wgrad0_parts(B, Hp)][kWgrad0Part] floats of workspace
constexpr int kWgrad0Part = 28 * 32;
int wgrad0_parts(int B, int Hp);
void wgrad0_reduce(const float* ws, int parts, float* dW, cudaStream_t st);
void wgrad0_gather(const void* X, const void* g, const uint8_t* amax, float* dW, float* ws, int B, int H, int W, int Hp,
                   int Wp, cudaStream_t st);
// the same gradient as four masked GEMMs on the tensor cores (wgrad0_mma.cu); needs the packed layer-1 input
// (s-packed for in_channels == 3, rs-packed for in_channels == 1)
bool wgrad0_mma_supported(int W, int Wp, int CK, int Ci, int Co);
void wgrad0_mma(const void* X, const void* g, const uint8_t* amax, float* dW, float* ws, int B, int H, int W, int Hp,
                int Wp, int in_channels, cudaStream_t st);
// the same on the compact [B*H*W, 4] RGB input (preprocess_u8 compact)
void wgrad0_mma_compact(const void* X, const void* g, const uint8_t* amax, float* dW, float* ws, int B, int H, int W,
                        int Hp, int Wp, cudaStream_t st);
// ---- general tensor-core GEMMs for the ResNet convolutions (gemm_tcgen05.cu) ----
// C[rows_out, N] (bf16) = sum_{t < taps} A[m + shifts[t], K] . B[t*N + n, K]^T. padded != 0: A rows index a zero-padded
// [Bn][H+2][W+2] grid and only interior pixels are written (to the dense [Bn*H*W, N] output). fp8: A and B hold e4m3
// bytes and the product of the two device scalars scale_a * scale_b multiplies the result.
void gemm_taps(const void* A, const void* Bm, void* C, int64_t a_rows, int N, int K, int taps, const int* shifts, int padded,
               int Bn, int H, int W, bool fp8, const float* scale_a, const float* scale_b, cudaStream_t st);
// dW[taps][Co][Ci] (fp32, zeroed by the caller) += dY[rows, Co]^T . X[rows + shift(tap), Ci]; taps = 1, or 9 on a padded
// grid whose rows are Wp pixels long.
void wgrad_taps(const void* DY, const void* X, float* dW, int64_t rows, int Co, int Ci, int taps, int Wp, cudaStream_t st);
void gemm_mxfp8(const void* A, const void* Bm, const void* sfa, const void* sfb, void* C, int64_t M, int N, int K,
                cudaStream_t st);
void pad_nhwc(const void* x, void* xp, int B, int H, int W, int C, cudaStream_t st);          // bf16, zero border of 1
void conv_weight_prep(const float* w, void* wt, void* wd, int Co, int Ci, int kk, cudaStream_t st);
void conv_wgrad_unpack(const float* dw, float* g, int Co, int Ci, int kk, cudaStream_t st);
// ---- ResNet building blocks (resnet_kernels.cu) ----
void bn_forward(const void* x, const void* res, const float* gamma, const float* beta, float* run_mean, float* run_var,
                float* mean, float* invstd, float* sums, void* y, int64_t P, int C, float momentum, float eps, int relu,
                cudaStream_t st);
void bn_backward(const void* dy, const void* x, const void* y, const float* mean, const float* invstd,
                 const float* gamma, float* sums, void* dx, void* dres, int64_t P, int C, int relu, cudaStream_t st);
void avgpool_forward(const void* x, float* out, int B, int HW, int C, cudaStream_t st);
void avgpool_backward(const float* dout, void* dx, int B, int HW, int C, cudaStream_t st);
void fp8_quantize(const void* x, uint8_t* q, const float* scale, float* amax, int64_t n, cudaStream_t st);
// bf16 [R,K] -> e4m3 [R,K] + UE8M0 scale tiles [ceil(R/128)][K/128][512] (rows beyond R must be pre-set by the caller)
void mxfp8_quantize(const void* x, uint8_t* q, uint8_t* sf, int64_t R, int K, cudaStream_t st);
void fp8_scale_update(float* amax, float* scale, float* inv, float target, cudaStream_t st);
void umma_shift_probe(const void* A, const void* Bm, float* out, int CK, int shift_rows, cudaStream_t st);

// ---- data-movement kernels around the convolutions (nn_kernels.cu) ----
constexpr int kMaxConvLayers = 8;
struct ConvLayerTable {
  int n;
  int Ci[kMaxConvLayers], CK[kMaxConvLayers], Co[kMaxConvLayers];
  int64_t w_off[kMaxConvLayers], b_off[kMaxConvLayers];       // offsets into the flat fp32 parameter buffer
  int64_t wf_off[kMaxConvLayers], wd_off[kMaxConvLayers];     // offsets (elements) into the bf16 Wf / Wd buffers
  int64_t dw_off[kMaxConvLayers];                             // offsets (elements) into the fp32 dW32 buffer
};
// x: uint8 [B,H,W,C] with C = 3 or 1; compact (C = 3 only): X is [B*H*W, 4] (R, G, B, 0) instead of [B*H*W, 16]
void preprocess_u8(const uint8_t* x, const float* theta, void* X, int B, int H, int W, int C, uint64_t aug_seed,
                   const int64_t* step, int spack, int compact, cudaStream_t st);
void unpool_relu(const void* g, const uint8_t* amax, const void* ypool, void* dY, int B, int H, int W, int Hp,
                 int Wp, int Co, cudaStream_t st);
// compact0 (with spack0, RGB): layer 1 gets the weights of the compact input, [3 r][2 dx][Co][16], after its s-packed
// [3][Co][16] ones (both fit in the [9][Co][16] slot)
void conv_weight_relayout(const void* shadow, const ConvLayerTable& t, void* Wf, void* Wd, int l0, int l1,
                          int spack0, int compact0, cudaStream_t st);
void conv_grad_finalize(float* dW32, const ConvLayerTable& t, float* grad, int l0, int l1, cudaStream_t st);

}  // namespace nn
}  // namespace hefl
