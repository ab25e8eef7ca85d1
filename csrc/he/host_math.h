// Host C++ runtime for the HE core: parameter generation (NTT-friendly primes,
// 2N-th roots, twiddle/Shoup/Barrett tables), and a CPU implementation of every
// HE kernel with the same signatures as the CUDA launchers in kernels.h. The CPU
// path is both the oracle for the GPU kernels and the backend of the CPU-only
// configuration (BASELINE.json configs[0]).
//
// Replaces Afseal::ContextGen / SEALContext reached from Pyfhel.contextGen
// (FLPyfhelin.py:332) — SURVEY.md §2.2 X1.a.
#pragma once
#include <cstdint>
#include <vector>

#include "server_step.h"

namespace hefl {
namespace host {

// tables layout: [L][4][N] = psi_br, psi_br_shoup, ipsi_br, ipsi_br_shoup
// consts layout: [L][8]    = q, ratio_lo, ratio_hi, ninv, ninv_shoup, psi, bits, 0
constexpr int kConstStride = 8;

bool is_prime(uint64_t n);
uint64_t pow_mod(uint64_t b, uint64_t e, uint64_t q);
uint64_t inv_mod(uint64_t a, uint64_t q);
// `count` primes q = 1 (mod 2N), q < 2^bits, descending from 2^bits, skipping
// any value present in `exclude`.
std::vector<uint64_t> gen_primes(int bits, int logn, int count,
                                 const std::vector<uint64_t>& exclude);
uint64_t find_psi(uint64_t q, int logn);
void build_tables(const uint64_t* moduli, int L, int logn, uint64_t* tables, uint64_t* consts);

// CKKS special-FFT tables: rot_group[N/2] (5^j mod 2N), ksi[2N+1][2] (cos, sin).
void build_fft_tables(int logn, int32_t* rot_group, double* ksi);

// ---- CPU kernels (same semantics as kernels.h) ----
void ntt(uint64_t* data, int64_t rows, int L, int logn, const uint64_t* tables,
         const uint64_t* consts, bool inverse);
void pointwise(uint64_t* out, const uint64_t* a, const uint64_t* b, int64_t rows, int64_t brows,
               int L, int n, const uint64_t* consts, int op);
void reduce_mod(uint64_t* data, int64_t rows, int L, int n, const uint64_t* consts);
void ckks_encode(const float* vals_f32, const double* vals_f64, int64_t C, int64_t nvals_total,
                 int logn, double scale, const int32_t* rot_group, const double* ksi, int64_t* msg);
void ckks_decode(const double* coeffs, int64_t C, int logn, double inv_scale,
                 const int32_t* rot_group, const double* ksi, float* out_f32, double* out_f64);
// Twin of cuda::ckks_decode_server_step on CRT-centred coefficients [C][N]: ckks_decode to fp64, then the
// server step of the first nvals values in the kernel's operation order (opt 1..4, server_step.h).
void ckks_decode_server_step(const double* coeffs, int64_t C, int logn, double inv_scale,
                             const int32_t* rot_group, const double* ksi, int64_t nvals,
                             const ServerStep& sv, int opt);
void coeff_encode(const float* vals, int64_t C, int64_t nvals_total, int n, double scale,
                  int64_t* msg);
void encrypt(const int64_t* msg, const uint64_t* pk, uint64_t* ct, int64_t C, int L, int logn,
             const uint64_t* tables, const uint64_t* consts, const uint64_t* msg_scale,
             uint64_t seed, uint32_t ct_offset, bool accumulate);
void decrypt(const uint64_t* ct, const uint64_t* sk, uint64_t* out, int64_t C, int Lct, int k,
             int logn, const uint64_t* tables, const uint64_t* consts);
void crt_center(const uint64_t* res, int64_t C, int k, int n, const uint64_t* consts, double* out);
void sample_secret(uint64_t* sk, int L, int logn, const uint64_t* tables, const uint64_t* consts,
                   uint64_t seed);
void gen_public(const uint64_t* sk, uint64_t* pk, int L, int logn, const uint64_t* tables,
                const uint64_t* consts, uint64_t seed, uint32_t idx);
// evk [E][2][L][n]: slot 0, limb limb_of[e] += w[e] * s2[limb_of[e]] (message term of a digit-decomposed evaluation key)
void relin_message(uint64_t* evk, const uint64_t* s2, const int* limb_of, const uint64_t* w, int64_t E, int L,
                   int64_t n, const uint64_t* consts);
void frac_encode(const double* vals, int64_t C, int n, int int_digits, int frac_digits,
                 int64_t* msg);
void frac_decode(const int64_t* coeffs, int64_t C, int n, int int_digits, int frac_digits,
                 double* out);
void bfv_scale_round(const uint64_t* x, int64_t C, int n, uint64_t q, uint64_t p, int64_t* out);
void digit_extract(const uint64_t* x, int64_t rows, int n, int shift, int bits, uint64_t* out);
// rows [rows][n] (row r belongs to limb r % L) -> [rows][n][2] = (x, floor(x * 2^64 / q))
void shoup_pairs(const uint64_t* x, uint64_t* out, int64_t rows, int L, int n, const uint64_t* consts);

}  // namespace host
}  // namespace hefl
