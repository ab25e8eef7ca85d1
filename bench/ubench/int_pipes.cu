// Integer-pipe microbenchmark for the NTT butterfly (sm_90a): issue rates of IMAD, IMAD.WIDE.U32,
// IMAD.HI.U32, IADD3, DFMA, mixes of them, __umul64hi and a complete Shoup butterfly, at 4/8/16
// warps per scheduler. Prints warp-instructions per cycle per SM. Build: see bench/ubench/build.sh.
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#define CHAINS 8
#define ITERS 4096

template <int MODE>
__global__ void k(uint64_t* out, uint32_t seed, uint64_t q, uint64_t w, uint64_t wp) {
  uint32_t a[CHAINS], b[CHAINS];
  uint64_t c[CHAINS];
  double d[CHAINS];
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) {
    a[i] = seed + threadIdx.x * 7 + i;
    b[i] = seed * 3 + i * 5 + 1;
    c[i] = ((uint64_t)a[i] << 20) + b[i];
    d[i] = (double)a[i];
  }
  const long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int i = 0; i < CHAINS; ++i) {
      if (MODE == 0) { a[i] = a[i] * b[i] + a[i]; }                                   // IMAD
      if (MODE == 1) { c[i] = (uint64_t)(uint32_t)c[i] * b[i] + c[i]; }               // IMAD.WIDE.U32
      if (MODE == 2) { a[i] = __umulhi(a[i], b[i]) + b[i]; }                          // IMAD.HI.U32
      if (MODE == 3) { a[i] = a[i] + b[i] + (a[i] >> 3); }                            // IADD3 (+SHF)
      if (MODE == 4) { c[i] = (uint64_t)(uint32_t)c[i] * b[i] + c[i]; a[i] = a[i] + b[i] + 12345u; }  // WIDE + IADD3
      if (MODE == 5) { c[i] = __umul64hi(c[i], w) + c[i]; }                           // mulhi64
      if (MODE == 6) { d[i] = fma(d[i], 1.0000001, 0.5); }                            // DFMA
      if (MODE == 7) { a[i] = a[i] * b[i] + a[i]; b[i] = b[i] + a[i] + 77u; }         // IMAD + IADD3
      if (MODE == 8) { c[i] = c[i] + w + (c[i] >> 7); }                               // 64-bit add chain (IADD3 + .X)
    }
    if (MODE == 9) {  // four complete Shoup butterflies (pairs of chains)
#pragma unroll
      for (int i = 0; i < CHAINS; i += 2) {
        const uint64_t X = c[i], Y = c[i + 1];
        const uint64_t qh = __umul64hi(Y, wp);
        const uint64_t Q = Y * w - qh * q;
        c[i] = X + Q;
        c[i + 1] = X + (2 * q - Q);
      }
    }
  }
  const long long t1 = clock64();
  uint64_t acc = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; ++i) acc += a[i] + b[i] + c[i] + (uint64_t)d[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0 && blockIdx.x == 0) out[gridDim.x * blockDim.x] = (uint64_t)(t1 - t0);
}

template <int MODE>
void run(const char* name, int per_iter, int threads) {
  uint64_t* out;
  int dev = 0, blocks = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&blocks, cudaDevAttrMultiProcessorCount, dev);   // one CTA per SM
  cudaMalloc(&out, (size_t)(blocks * threads + 1) * 8);
  k<MODE><<<blocks, threads>>>(out, 12345u, 18014398509404161ull, 123456789123ull, 987654321987654321ull);
  cudaDeviceSynchronize();
  k<MODE><<<blocks, threads>>>(out, 12345u, 18014398509404161ull, 123456789123ull, 987654321987654321ull);
  cudaDeviceSynchronize();
  uint64_t cyc;
  cudaMemcpy(&cyc, out + blocks * threads, 8, cudaMemcpyDeviceToHost);
  const double winst = (double)ITERS * per_iter * (threads / 32);
  printf("%-28s threads/SM %4d  %8.3f units/clk/SM   (%.2f clk per warp-unit per SMSP)\n", name, threads,
         winst / (double)cyc, (double)cyc * 4.0 / winst);
  cudaFree(out);
}

int main() {
  for (int threads : {512, 1024}) {
    run<0>("IMAD", CHAINS, threads);
    run<1>("IMAD.WIDE.U32", CHAINS, threads);
    run<2>("IMAD.HI.U32", CHAINS, threads);
    run<3>("IADD3+SHF (2 alu)", CHAINS, threads);
    run<4>("IMAD.WIDE + IADD3 pair", CHAINS, threads);
    run<5>("umul64hi + add64", CHAINS, threads);
    run<6>("DFMA", CHAINS, threads);
    run<7>("IMAD + IADD3 pair", CHAINS, threads);
    run<8>("add64 + shr64", CHAINS, threads);
    run<9>("Shoup butterfly", CHAINS / 2, threads);
  }
  return 0;
}
