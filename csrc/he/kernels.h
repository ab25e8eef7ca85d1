// Launchers of the sm_90a HE kernels (csrc/he/cuda/he_kernels.cu). Plain C++
// signatures with raw device pointers so the .cu files compile without the
// PyTorch headers (seconds, not minutes); csrc/bindings.cpp adapts tensors.
//
// Layouts: ciphertext batch [C][2][L][N] u64 in NTT form; plaintext/message
// [C][N]; tables [L][4][N]; consts [L][8] (see host_math.h).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "server_step.h"

namespace hefl {
namespace cuda {

void ntt(uint64_t* data, int64_t rows, int L, int logn, const uint64_t* tables,
         const uint64_t* consts, bool inverse, cudaStream_t st);
void pointwise(uint64_t* out, const uint64_t* a, const uint64_t* b, int64_t rows, int64_t brows,
               int L, int n, const uint64_t* consts, int op, cudaStream_t st);
void reduce_mod(uint64_t* data, int64_t rows, int L, int n, const uint64_t* consts,
                cudaStream_t st);
void ckks_encode(const float* vals_f32, const double* vals_f64, int64_t C, int64_t nvals_total,
                 int logn, double scale, const int32_t* rot_group, const double* ksi, int64_t* msg,
                 double* scratch, cudaStream_t st);
void ckks_decode_residues(const uint64_t* res, int64_t C, int k, int logn, uint64_t q0, uint64_t q1,
                          uint64_t q1_ratio_lo, uint64_t q1_ratio_hi, uint64_t q0_inv_q1,
                          double inv_scale, const int32_t* rot_group, const double* ksi,
                          float* out, int64_t nvals_total, double* scratch, cudaStream_t st);
void ckks_decode(const double* coeffs, int64_t C, int logn, double inv_scale,
                 const int32_t* rot_group, const double* ksi, float* out_f32, double* out_f64,
                 double* scratch, cudaStream_t st);

// Decode + server-optimizer step (server_step.h, DESIGN.md §8) in one launch; opt 1..4 (ServerOpt).
void ckks_decode_server_step(const uint64_t* res, int64_t C, int k, int logn, uint64_t q0, uint64_t q1,
                             uint64_t q1_ratio_lo, uint64_t q1_ratio_hi, uint64_t q0_inv_q1,
                             double inv_scale, const int32_t* rot_group, const double* ksi,
                             int64_t nvals, const ServerStep& sv, int opt, double* scratch, cudaStream_t st);
void coeff_encode(const float* vals, int64_t C, int64_t nvals_total, int n, double scale,
                  int64_t* msg, cudaStream_t st);
// accumulate: ct = (ct + Enc(m)) mod q word by word (the rank's clients summed without a buffer per client)
void encrypt(const int64_t* msg, const uint64_t* pk, uint64_t* ct, int64_t C, int L, int logn,
             const uint64_t* tables, const uint64_t* consts, const uint64_t* msg_scale,
             uint64_t seed, uint32_t ct_offset, bool accumulate, cudaStream_t st);
void decrypt(const uint64_t* ct, const uint64_t* sk, uint64_t* out, int64_t C, int Lct, int k,
             int logn, const uint64_t* tables, const uint64_t* consts, cudaStream_t st);
void crt_center(const uint64_t* res, int64_t C, int k, int n, uint64_t q0, uint64_t q1,
                uint64_t q1_ratio_lo, uint64_t q1_ratio_hi, uint64_t q0_inv_q1, double* out,
                cudaStream_t st);
void frac_encode(const double* vals, int64_t C, int n, int int_digits, int frac_digits,
                 int64_t* msg, cudaStream_t st);
void frac_decode(const int64_t* coeffs, int64_t C, int n, int int_digits, int frac_digits,
                 double* out, cudaStream_t st);
void bfv_scale_round(const uint64_t* x, int64_t C, int n, uint64_t q, uint64_t p, int64_t* out,
                     cudaStream_t st);
void digit_extract(const uint64_t* x, int64_t rows, int n, int shift, int bits, uint64_t* out,
                   cudaStream_t st);

// key generation on the device (same Philox streams as the host twin)
void keygen_sample(uint64_t* out, int E, int L, int n, const uint64_t* consts, uint64_t seed, uint32_t idx0, int mode,
                   cudaStream_t st);
void keygen_finish(const uint64_t* sk, uint64_t* pk, int E, int L, int n, const uint64_t* consts, uint64_t seed,
                   uint32_t idx0, cudaStream_t st);
void relin_message(uint64_t* evk, const uint64_t* s2, const int* limb_of, const uint64_t* w, int E, int L, int n,
                   const uint64_t* consts, cudaStream_t st);

// ---- second-generation persistent kernels (csrc/he/cuda/he_kernels2.cu) ----
// tw2: [L][2][N][2] interleaved (w, w') tables (forward, inverse); pkx: [2][L][N][2] (pk, pk');
// skx: [L][N][2] (s, s'); qbits: bit length of the largest prime. Each returns false (and
// launches nothing) when the parameters are outside the fast path: the caller falls back.
bool ntt2_supported(int logn, int L, int qbits);
// CTA budgets of the persistent kernels (0 = all SMs): lets encrypt / all-reduce / decrypt share the chip.
void set_cta_limits(int ntt, int enc, int dec);
bool ntt2(uint64_t* data, int64_t rows, int L, int logn, const uint64_t* tw2, const uint64_t* consts, int qbits,
          bool inverse, cudaStream_t st);
// At N = 16384 the ciphertext in flight keeps NTT(u) in a global row per CTA: `scratch` holds
// encrypt2_scratch_words(logn) words (0 below N = 16384) and belongs to this launch alone, so that
// encrypts on different streams cannot overwrite each other's rows.
int64_t encrypt2_scratch_words(int logn);
bool encrypt2(const int64_t* msg, const uint64_t* pkx, uint64_t* ct, int64_t C, int L, int logn, const uint64_t* tw2,
              const uint64_t* consts, const uint64_t* msg_scale, uint64_t seed, uint32_t ct_offset, int qbits,
              uint64_t* scratch, bool accumulate, cudaStream_t st);
bool decrypt2(const uint64_t* ct, const uint64_t* skx, uint64_t* out, int64_t C, int Lct, int k, int logn,
              const uint64_t* tw2, const uint64_t* consts, int Ltab, int qbits, cudaStream_t st);

// ---- fused evaluation kernels (csrc/he/cuda/he_eval2.cu); false = outside the fast path, nothing launched ----
// inv / inv_p: host arrays, q_last^-1 mod q_j and its Shoup companion for j < lvl - 1.
bool rescale2(const uint64_t* ct, uint64_t* out, int64_t C, int lvl, int logn, const uint64_t* tw2, const uint64_t* consts,
              const uint64_t* inv, const uint64_t* inv_p, int qbits, cudaStream_t st);
// acc [C][2][lvl][N] += sum_{i,k} NTT(digit_{i,k}(coef)) * evk[first[i] + k]; ndig / first: host arrays of lvl ints.
bool keyswitch2(const uint64_t* coef, const uint64_t* evk, uint64_t* acc, int64_t C, int lvl, int Ltab, int logn,
                int digit_bits, const int* ndig, const int* first, const uint64_t* tw2, const uint64_t* consts, int qbits,
                cudaStream_t st);
void ct_tensor(const uint64_t* A, const uint64_t* B, uint64_t* d01, uint64_t* d2, int64_t C, int lvl, int n,
               const uint64_t* consts, cudaStream_t st);

// rows [rows][n] (row r belongs to limb r % L) -> [rows][n][2] = (x, floor(x * 2^64 / q))
void shoup_pairs(const uint64_t* x, uint64_t* out, int64_t rows, int L, int n, const uint64_t* consts,
                 cudaStream_t st);

// Number of kernels launched by this library since process start (bench.py's gpu_launches).
uint64_t launch_count();
void note_launch(uint64_t n = 1);
// SM count of the current device (cached per device): grid caps of grid-stride kernels scale with it.
int device_sm_count();

}  // namespace cuda
}  // namespace hefl
