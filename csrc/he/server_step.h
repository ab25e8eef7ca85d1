// Arguments of the server-optimizer step fused into the CKKS decode (DESIGN.md §8), shared by the CUDA
// launcher (kernels.h) and its host twin (host_math.h).
#pragma once
#include <cstdint>

namespace hefl {

// Value g of a decoded batch is flat index g0 + g of the model: x_t / x_new / avg_* are indexed by it; m and v
// hold n_trainable entries; from n_trainable on the new model is the average itself (BatchNorm statistics) and
// no state is touched. avg_f32 / avg_f64 are optional copies of the decoded average.
struct ServerStep {
  const float* x_t = nullptr;
  float* x_new = nullptr;
  float* m = nullptr;
  float* v = nullptr;
  float* avg_f32 = nullptr;
  double* avg_f64 = nullptr;
  int64_t g0 = 0, n_trainable = 0;
  float lr = 0.f, beta1 = 0.f, beta2 = 0.f, tau = 0.f;
};

// opt codes of the fused step; 0 is the plain decode
enum ServerOpt : int { kFedAvg = 0, kFedAvgM = 1, kFedAdagrad = 2, kFedYogi = 3, kFedAdam = 4 };

}  // namespace hefl
