// Federated evaluation counts (DESIGN.md §13): one client's confusion matrix, score histograms and cross-entropy sum
// from the logits of a batch, in one launch of one CTA.
//
// One thread per row (strided over the batch): the arg-max of the logits (lowest index on ties), p = softmax(logits)
// in fp32, written to probs; conf[y][argmax] and hist[y][c][bin(p_c)] are bumped with integer atomics, so the counts do
// not depend on the order the rows land in. Each thread sums the float64 cross-entropy of its rows in row order, and
// thread 0 adds the 256 partials in thread order into the client's loss sum: a fixed order, no float atomics, the same
// bits on every run. The valid row count is read from the device, so a captured graph can score a partial last batch;
// rows >= nvalid are neither read nor written. A label outside 0..C-1 raises the error flag (no trap) and its row adds
// nothing.
#include <cuda_runtime.h>

#include "../he/kernels.h"
#include "launch.cuh"
#include "nn.h"

namespace hefl {
namespace nn {

namespace sc {
constexpr int NT = 256;
}  // namespace sc

__global__ void __launch_bounds__(sc::NT)
score_stats_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, const int* __restrict__ nvalid,
                   float* __restrict__ probs, int* __restrict__ counts, double* __restrict__ loss_sum,
                   int* __restrict__ err, int B, int C, int nbins) {
  __shared__ double part[sc::NT];
  pdl_prologue();
  const int nv = min(max(*nvalid, 0), B);
  const int t = threadIdx.x;
  double acc = 0.0;
  for (int b = t; b < nv; b += sc::NT) {
    const float* l = logits + (size_t)b * C;
    float mx = l[0];
    int am = 0;
    for (int c = 1; c < C; ++c)
      if (l[c] > mx) { mx = l[c]; am = c; }
    float s = 0.f;
    double sd = 0.0;
    for (int c = 0; c < C; ++c) {
      s += expf(l[c] - mx);
      sd += exp((double)l[c] - (double)mx);
    }
    float* pr = probs + (size_t)b * C;
    for (int c = 0; c < C; ++c) pr[c] = expf(l[c] - mx) / s;
    const int64_t y = labels[b];
    if (y < 0 || y >= C) {
      atomicOr(err, 1);
      continue;
    }
    const int yy = (int)y;
    acc += (double)mx + log(sd) - (double)l[yy];
    atomicAdd(counts + yy * C + am, 1);
    int* h = counts + C * C + (size_t)yy * C * nbins;
    for (int c = 0; c < C; ++c) {
      const int bin = max(0, min(nbins - 1, (int)floorf(pr[c] * (float)nbins)));
      atomicAdd(h + c * nbins + bin, 1);
    }
  }
  part[t] = acc;
  __syncthreads();
  if (t == 0) {
    double s = 0.0;
    for (int i = 0; i < sc::NT; ++i) s += part[i];
    *loss_sum += s;
  }
}

void score_stats(const float* logits, const int64_t* labels, const int* nvalid, float* probs, int* counts,
                 double* loss_sum, int* err, int B, int C, int nbins, cudaStream_t st) {
  launch_pdl(score_stats_kernel, dim3(1), dim3(sc::NT), 0, st, logits, labels, nvalid, probs, counts, loss_sum, err, B,
             C, nbins);
  hefl::cuda::note_launch();
}

}  // namespace nn
}  // namespace hefl
