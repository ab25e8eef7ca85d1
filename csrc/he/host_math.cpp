// Host C++ runtime for the HE core. See host_math.h.
#include "host_math.h"

#include <algorithm>
#include <cmath>
#include <complex>
#include <cstring>
#include <stdexcept>

#include "modarith.h"
#include "philox.h"

namespace hefl {
namespace host {

using u128 = unsigned __int128;

uint64_t pow_mod(uint64_t b, uint64_t e, uint64_t q) {
  u128 r = 1, x = b % q;
  while (e) {
    if (e & 1) r = (r * x) % q;
    x = (x * x) % q;
    e >>= 1;
  }
  return (uint64_t)r;
}

uint64_t inv_mod(uint64_t a, uint64_t q) { return pow_mod(a, q - 2, q); }

bool is_prime(uint64_t n) {
  if (n < 2) return false;
  static const uint64_t small[] = {2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37};
  for (uint64_t p : small) {
    if (n % p == 0) return n == p;
  }
  uint64_t d = n - 1;
  int s = 0;
  while ((d & 1) == 0) { d >>= 1; ++s; }
  // Deterministic for n < 2^64 with these witnesses.
  for (uint64_t a : small) {
    uint64_t x = pow_mod(a, d, n);
    if (x == 1 || x == n - 1) continue;
    bool comp = true;
    for (int i = 1; i < s; ++i) {
      x = (uint64_t)(((u128)x * x) % n);
      if (x == n - 1) { comp = false; break; }
    }
    if (comp) return false;
  }
  return true;
}

std::vector<uint64_t> gen_primes(int bits, int logn, int count,
                                 const std::vector<uint64_t>& exclude) {
  if (bits < logn + 2 || bits > 61) throw std::invalid_argument("prime bit size out of range");
  std::vector<uint64_t> out;
  const uint64_t two_n = 1ull << (logn + 1);
  uint64_t cand = ((1ull << bits) - 1) / two_n * two_n + 1;
  while ((int)out.size() < count) {
    if (cand < (1ull << (bits - 1))) throw std::runtime_error("not enough NTT primes of this size");
    if (is_prime(cand) && std::find(exclude.begin(), exclude.end(), cand) == exclude.end() &&
        std::find(out.begin(), out.end(), cand) == out.end())
      out.push_back(cand);
    cand -= two_n;
  }
  return out;
}

uint64_t find_psi(uint64_t q, int logn) {
  // Minimal primitive 2N-th root of unity (SEAL convention) so tables are canonical.
  const uint64_t two_n = 1ull << (logn + 1);
  const uint64_t e = (q - 1) / two_n;
  uint64_t root = 0;
  for (uint64_t g = 2; g < q; ++g) {
    uint64_t c = pow_mod(g, e, q);
    if (pow_mod(c, two_n / 2, q) == q - 1) { root = c; break; }
  }
  if (!root) throw std::runtime_error("no primitive root");
  // minimal among all odd powers
  uint64_t best = root, cur = root;
  const uint64_t sq = (uint64_t)(((u128)root * root) % q);
  for (uint64_t i = 1; i < two_n / 2; ++i) {
    cur = (uint64_t)(((u128)cur * sq) % q);
    if (cur < best) best = cur;
  }
  return best;
}

static uint64_t shoup_of(uint64_t w, uint64_t q) { return (uint64_t)((((u128)w) << 64) / q); }

void build_tables(const uint64_t* moduli, int L, int logn, uint64_t* tables, uint64_t* consts) {
  const int64_t n = 1ll << logn;
  for (int l = 0; l < L; ++l) {
    const uint64_t q = moduli[l];
    const uint64_t psi = find_psi(q, logn);
    const uint64_t ipsi = inv_mod(psi, q);
    uint64_t* t = tables + (int64_t)l * 4 * n;
    uint64_t pw = 1, ipw = 1;
    for (int64_t i = 0; i < n; ++i) {
      const uint32_t r = bit_reverse((uint32_t)i, logn);
      t[0 * n + r] = pw;
      t[1 * n + r] = shoup_of(pw, q);
      t[2 * n + r] = ipw;
      t[3 * n + r] = shoup_of(ipw, q);
      pw = (uint64_t)(((u128)pw * psi) % q);
      ipw = (uint64_t)(((u128)ipw * ipsi) % q);
    }
    uint64_t* c = consts + (int64_t)l * kConstStride;
    // floor(2^128 / q)
    u128 hi_part = (~(u128)0) / q;  // floor((2^128 - 1)/q) == floor(2^128/q) since q is odd > 1
    c[0] = q;
    c[1] = (uint64_t)hi_part;
    c[2] = (uint64_t)(hi_part >> 64);
    const uint64_t ninv = inv_mod((uint64_t)n % q, q);
    c[3] = ninv;
    c[4] = shoup_of(ninv, q);
    c[5] = psi;
    int bits = 0;
    for (uint64_t v = q; v; v >>= 1) ++bits;
    c[6] = (uint64_t)bits;
    c[7] = 0;
  }
}

void build_fft_tables(int logn, int32_t* rot_group, double* ksi) {
  const int64_t n = 1ll << logn, m = 2 * n, nh = n / 2;
  int64_t five = 1;
  for (int64_t i = 0; i < nh; ++i) {
    rot_group[i] = (int32_t)five;
    five = (five * 5) % m;
  }
  const long double pi = 3.14159265358979323846264338327950288L;
  for (int64_t j = 0; j <= m; ++j) {
    long double ang = 2.0L * pi * (long double)j / (long double)m;
    ksi[2 * j] = (double)cosl(ang);
    ksi[2 * j + 1] = (double)sinl(ang);
  }
}

static inline Modulus load_mod(const uint64_t* consts, int l) {
  const uint64_t* c = consts + (int64_t)l * kConstStride;
  return Modulus{c[0], c[1], c[2]};
}

static void ntt_fwd_row(uint64_t* a, int logn, const uint64_t* w, const uint64_t* wp, uint64_t q) {
  const int64_t n = 1ll << logn;
  const uint64_t two_q = 2 * q;
  int64_t t = n;
  for (int64_t m = 1; m < n; m <<= 1) {
    t >>= 1;
    for (int64_t i = 0; i < m; ++i) {
      const uint64_t W = w[m + i], Wp = wp[m + i];
      const int64_t j1 = 2 * i * t;
      for (int64_t j = j1; j < j1 + t; ++j) {
        uint64_t X = a[j];
        if (X >= two_q) X -= two_q;
        const uint64_t Q = mul_shoup_lazy(a[j + t], W, Wp, q);
        a[j] = X + Q;
        a[j + t] = X - Q + two_q;
      }
    }
  }
  for (int64_t j = 0; j < n; ++j) {
    uint64_t x = a[j];
    if (x >= two_q) x -= two_q;
    if (x >= q) x -= q;
    a[j] = x;
  }
}

static void ntt_inv_row(uint64_t* a, int logn, const uint64_t* w, const uint64_t* wp, uint64_t q,
                        uint64_t ninv, uint64_t ninv_p) {
  const int64_t n = 1ll << logn;
  const uint64_t two_q = 2 * q;
  int64_t t = 1;
  for (int64_t m = n; m > 1; m >>= 1) {
    const int64_t h = m >> 1;
    int64_t j1 = 0;
    for (int64_t i = 0; i < h; ++i) {
      const uint64_t W = w[h + i], Wp = wp[h + i];
      for (int64_t j = j1; j < j1 + t; ++j) {
        const uint64_t U = a[j], V = a[j + t];
        uint64_t s = U + V;
        if (s >= two_q) s -= two_q;
        a[j] = s;
        a[j + t] = mul_shoup_lazy(U - V + two_q, W, Wp, q);
      }
      j1 += 2 * t;
    }
    t <<= 1;
  }
  for (int64_t j = 0; j < n; ++j) a[j] = mul_shoup(a[j], ninv, ninv_p, q);
}

void ntt(uint64_t* data, int64_t rows, int L, int logn, const uint64_t* tables,
         const uint64_t* consts, bool inverse) {
  const int64_t n = 1ll << logn;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < rows; ++r) {
    const int l = (int)(r % L);
    const uint64_t* t = tables + (int64_t)l * 4 * n;
    const uint64_t* c = consts + (int64_t)l * kConstStride;
    if (!inverse)
      ntt_fwd_row(data + r * n, logn, t, t + n, c[0]);
    else
      ntt_inv_row(data + r * n, logn, t + 2 * n, t + 3 * n, c[0], c[3], c[4]);
  }
}

void pointwise(uint64_t* out, const uint64_t* a, const uint64_t* b, int64_t rows, int64_t brows,
               int L, int n, const uint64_t* consts, int op) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < rows; ++r) {
    const int l = (int)(r % L);
    const Modulus m = load_mod(consts, l);
    const uint64_t* ar = a + r * n;
    const uint64_t* br = (op == 5 || op == 4 || b == nullptr) ? nullptr : b + (r % brows) * n;
    uint64_t* o = out + r * n;
    switch (op) {
      case 0: for (int i = 0; i < n; ++i) o[i] = add_mod(ar[i], br[i], m.q); break;
      case 1: for (int i = 0; i < n; ++i) o[i] = sub_mod(ar[i], br[i], m.q); break;
      case 2: for (int i = 0; i < n; ++i) o[i] = mul_mod(ar[i], br[i], m); break;
      case 3: for (int i = 0; i < n; ++i) o[i] = mad_mod(ar[i], br[i], o[i], m); break;
      case 4: for (int i = 0; i < n; ++i) o[i] = neg_mod(ar[i], m.q); break;
      case 5: { const uint64_t s = b[l]; for (int i = 0; i < n; ++i) o[i] = mul_mod(ar[i], s, m); } break;
      default: break;
    }
  }
}

void reduce_mod(uint64_t* data, int64_t rows, int L, int n, const uint64_t* consts) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < rows; ++r) {
    const Modulus m = load_mod(consts, (int)(r % L));
    uint64_t* d = data + r * n;
    for (int i = 0; i < n; ++i) d[i] = barrett_reduce_64(d[i], m);
  }
}

using cplx = std::complex<double>;

static void bit_reverse_perm(cplx* v, int64_t size) {
  for (int64_t i = 1, j = 0; i < size; ++i) {
    int64_t bit = size >> 1;
    for (; j >= bit; bit >>= 1) j -= bit;
    j += bit;
    if (i < j) std::swap(v[i], v[j]);
  }
}

// Inverse canonical embedding restricted to the 5^j orbit (HEAAN "fftSpecialInv").
static void fft_special_inv(cplx* v, int64_t size, int64_t m, const int32_t* rot, const double* ksi) {
  for (int64_t len = size; len >= 1; len >>= 1) {
    const int64_t lenh = len >> 1, lenq = len << 2, gap = m / lenq;
    for (int64_t i = 0; i < size; i += len) {
      for (int64_t j = 0; j < lenh; ++j) {
        const int64_t idx = (lenq - (rot[j] % lenq)) * gap;
        const cplx u = v[i + j] + v[i + j + lenh];
        cplx w = v[i + j] - v[i + j + lenh];
        w *= cplx(ksi[2 * idx], ksi[2 * idx + 1]);
        v[i + j] = u;
        v[i + j + lenh] = w;
      }
    }
  }
  bit_reverse_perm(v, size);
  const double inv = 1.0 / (double)size;
  for (int64_t i = 0; i < size; ++i) v[i] *= inv;
}

static void fft_special(cplx* v, int64_t size, int64_t m, const int32_t* rot, const double* ksi) {
  bit_reverse_perm(v, size);
  for (int64_t len = 2; len <= size; len <<= 1) {
    const int64_t lenh = len >> 1, lenq = len << 2, gap = m / lenq;
    for (int64_t i = 0; i < size; i += len) {
      for (int64_t j = 0; j < lenh; ++j) {
        const int64_t idx = (rot[j] % lenq) * gap;
        const cplx u = v[i + j];
        const cplx w = v[i + j + lenh] * cplx(ksi[2 * idx], ksi[2 * idx + 1]);
        v[i + j] = u + w;
        v[i + j + lenh] = u - w;
      }
    }
  }
}

void ckks_encode(const float* vals_f32, const double* vals_f64, int64_t C, int64_t nvals_total,
                 int logn, double scale, const int32_t* rot_group, const double* ksi, int64_t* msg) {
  const int64_t n = 1ll << logn, nh = n / 2, m = 2 * n;
#pragma omp parallel for schedule(static)
  for (int64_t c = 0; c < C; ++c) {
    std::vector<cplx> v(nh);
    for (int64_t i = 0; i < nh; ++i) {
      const int64_t g = c * nh + i;
      double x = 0.0;
      if (g < nvals_total) x = vals_f32 ? (double)vals_f32[g] : vals_f64[g];
      v[i] = cplx(x, 0.0);
    }
    fft_special_inv(v.data(), nh, m, rot_group, ksi);
    int64_t* o = msg + c * n;
    for (int64_t i = 0; i < nh; ++i) {
      o[i] = (int64_t)llrint(v[i].real() * scale);
      o[i + nh] = (int64_t)llrint(v[i].imag() * scale);
    }
  }
}

void ckks_decode(const double* coeffs, int64_t C, int logn, double inv_scale,
                 const int32_t* rot_group, const double* ksi, float* out_f32, double* out_f64) {
  const int64_t n = 1ll << logn, nh = n / 2, m = 2 * n;
#pragma omp parallel for schedule(static)
  for (int64_t c = 0; c < C; ++c) {
    std::vector<cplx> v(nh);
    const double* x = coeffs + c * n;
    for (int64_t i = 0; i < nh; ++i) v[i] = cplx(x[i] * inv_scale, x[i + nh] * inv_scale);
    fft_special(v.data(), nh, m, rot_group, ksi);
    for (int64_t i = 0; i < nh; ++i) {
      if (out_f32) out_f32[c * nh + i] = (float)v[i].real();
      if (out_f64) out_f64[c * nh + i] = v[i].real();
    }
  }
}

// fp32 step of one value, in the order of server_step_one (he_kernels.cu); fp-contract=off keeps g++ from fusing
// a multiply-add on targets that have FMA, where the kernel rounds every product and sum on its own.
__attribute__((optimize("fp-contract=off")))
static float server_step_one(double a, int64_t g, const ServerStep& s, int opt) {
  if (g >= s.n_trainable) return (float)a;
  const float x = s.x_t[g];
  const float d = (float)(a - (double)x);
  float m = s.m[g];
  if (opt == kFedAvgM) {
    m = s.beta1 * m + d;
    s.m[g] = m;
    return x + s.lr * m;
  }
  m = s.beta1 * m + (1.0f - s.beta1) * d;
  const float d2 = d * d;
  float v = s.v[g];
  if (opt == kFedAdagrad) {
    v = v + d2;
  } else if (opt == kFedYogi) {
    const float t = v - d2;
    const float sg = t > 0.0f ? 1.0f : (t < 0.0f ? -1.0f : 0.0f);
    v = v - ((1.0f - s.beta2) * d2) * sg;
  } else {
    v = s.beta2 * v + (1.0f - s.beta2) * d2;
  }
  s.m[g] = m;
  s.v[g] = v;
  return x + (s.lr * m) / (std::sqrt(v) + s.tau);
}

void ckks_decode_server_step(const double* coeffs, int64_t C, int logn, double inv_scale,
                             const int32_t* rot_group, const double* ksi, int64_t nvals,
                             const ServerStep& sv, int opt) {
  const int64_t nh = (1ll << logn) / 2;
  std::vector<double> avg((size_t)(C * nh));
  ckks_decode(coeffs, C, logn, inv_scale, rot_group, ksi, nullptr, avg.data());
#pragma omp parallel for schedule(static)
  for (int64_t g = 0; g < nvals; ++g) {
    const double a = avg[g];
    const int64_t gg = sv.g0 + g;
    if (sv.avg_f32) sv.avg_f32[gg] = (float)a;
    if (sv.avg_f64) sv.avg_f64[gg] = a;
    sv.x_new[gg] = server_step_one(a, gg, sv, opt);
  }
}

void coeff_encode(const float* vals, int64_t C, int64_t nvals_total, int n, double scale,
                  int64_t* msg) {
#pragma omp parallel for schedule(static)
  for (int64_t c = 0; c < C; ++c)
    for (int64_t i = 0; i < n; ++i) {
      const int64_t g = c * n + i;
      msg[g] = g < nvals_total ? (int64_t)llrint((double)vals[g] * scale) : 0;
    }
}

void encrypt(const int64_t* msg, const uint64_t* pk, uint64_t* ct, int64_t C, int L, int logn,
             const uint64_t* tables, const uint64_t* consts, const uint64_t* msg_scale,
             uint64_t seed, uint32_t ct_offset, bool accumulate) {
  const int64_t n = 1ll << logn;
#pragma omp parallel for schedule(static) collapse(2)
  for (int64_t c = 0; c < C; ++c) {
    for (int l = 0; l < L; ++l) {
      const Modulus m = load_mod(consts, l);
      const uint64_t* t = tables + (int64_t)l * 4 * n;
      std::vector<uint64_t> u(n), a(n), b(n);
      const uint64_t sc = msg_scale ? msg_scale[l] : 1;
      for (int64_t i = 0; i < n; ++i) {
        const EncNoise z = sample_enc_noise(seed, ct_offset + (uint32_t)c, (uint32_t)i);
        u[i] = lift_signed(z.u, m.q);
        uint64_t mm = msg ? reduce_signed(msg[c * n + i], m) : 0;
        if (sc != 1) mm = mul_mod(mm, sc, m);
        a[i] = add_mod(lift_signed(z.e0, m.q), mm, m.q);
        b[i] = lift_signed(z.e1, m.q);
      }
      ntt_fwd_row(u.data(), logn, t, t + n, m.q);
      ntt_fwd_row(a.data(), logn, t, t + n, m.q);
      ntt_fwd_row(b.data(), logn, t, t + n, m.q);
      uint64_t* c0 = ct + ((c * 2 + 0) * L + l) * n;
      uint64_t* c1 = ct + ((c * 2 + 1) * L + l) * n;
      const uint64_t* pk0 = pk + (int64_t)(0 * L + l) * n;
      const uint64_t* pk1 = pk + (int64_t)(1 * L + l) * n;
      for (int64_t i = 0; i < n; ++i) {
        c0[i] = mad_mod(u[i], pk0[i], accumulate ? add_mod(a[i], c0[i], m.q) : a[i], m);
        c1[i] = mad_mod(u[i], pk1[i], accumulate ? add_mod(b[i], c1[i], m.q) : b[i], m);
      }
    }
  }
}

void decrypt(const uint64_t* ct, const uint64_t* sk, uint64_t* out, int64_t C, int Lct, int k,
             int logn, const uint64_t* tables, const uint64_t* consts) {
  const int64_t n = 1ll << logn;
#pragma omp parallel for schedule(static) collapse(2)
  for (int64_t c = 0; c < C; ++c) {
    for (int l = 0; l < k; ++l) {
      const Modulus m = load_mod(consts, l);
      const uint64_t* t = tables + (int64_t)l * 4 * n;
      const uint64_t* cc = consts + (int64_t)l * kConstStride;
      const uint64_t* c0 = ct + ((c * 2 + 0) * Lct + l) * n;
      const uint64_t* c1 = ct + ((c * 2 + 1) * Lct + l) * n;
      const uint64_t* s = sk + (int64_t)l * n;
      uint64_t* o = out + (c * k + l) * n;
      for (int64_t i = 0; i < n; ++i) o[i] = mad_mod(c1[i], s[i], c0[i], m);
      ntt_inv_row(o, logn, t + 2 * n, t + 3 * n, m.q, cc[3], cc[4]);
    }
  }
}

void crt_center(const uint64_t* res, int64_t C, int k, int n, const uint64_t* consts, double* out) {
  if (k < 1 || k > 2) throw std::invalid_argument("crt_center supports 1 or 2 limbs");
  const uint64_t q0 = consts[0];
  if (k == 1) {
#pragma omp parallel for schedule(static)
    for (int64_t g = 0; g < C * n; ++g) {
      const uint64_t x = res[g];
      out[g] = x > q0 / 2 ? -(double)(q0 - x) : (double)x;
    }
    return;
  }
  const Modulus m1 = load_mod(consts, 1);
  const uint64_t q0_inv_q1 = inv_mod(q0 % m1.q, m1.q);
  const u128 Q = (u128)q0 * m1.q;
#pragma omp parallel for schedule(static)
  for (int64_t c = 0; c < C; ++c) {
    for (int64_t i = 0; i < n; ++i) {
      const uint64_t x0 = res[(c * 2 + 0) * n + i];
      const uint64_t x1 = res[(c * 2 + 1) * n + i];
      const uint64_t x0r = barrett_reduce_64(x0, m1);
      const uint64_t d = mul_mod(sub_mod(x1, x0r, m1.q), q0_inv_q1, m1);
      const u128 x = (u128)x0 + (u128)q0 * d;
      out[c * n + i] = x > Q / 2 ? -(double)(Q - x) : (double)x;
    }
  }
}

void sample_secret(uint64_t* sk, int L, int logn, const uint64_t* tables, const uint64_t* consts,
                   uint64_t seed) {
  const int64_t n = 1ll << logn;
  for (int l = 0; l < L; ++l) {
    const uint64_t q = consts[(int64_t)l * kConstStride];
    const uint64_t* t = tables + (int64_t)l * 4 * n;
    uint64_t* s = sk + (int64_t)l * n;
    for (int64_t i = 0; i < n; ++i) s[i] = lift_signed(sample_ternary(seed, STREAM_SK, (uint32_t)i), q);
    ntt_fwd_row(s, logn, t, t + n, q);
  }
}

void gen_public(const uint64_t* sk, uint64_t* pk, int L, int logn, const uint64_t* tables,
                const uint64_t* consts, uint64_t seed, uint32_t idx) {
  const int64_t n = 1ll << logn;
  for (int l = 0; l < L; ++l) {
    const Modulus m = load_mod(consts, l);
    const uint64_t* t = tables + (int64_t)l * 4 * n;
    std::vector<uint64_t> e(n);
    for (int64_t i = 0; i < n; ++i)
      e[i] = lift_signed(sample_cbd(seed, STREAM_PK_E, idx, (uint32_t)i), m.q);
    ntt_fwd_row(e.data(), logn, t, t + n, m.q);
    uint64_t* b = pk + (int64_t)(0 * L + l) * n;
    uint64_t* a = pk + (int64_t)(1 * L + l) * n;
    const uint64_t* s = sk + (int64_t)l * n;
    for (int64_t i = 0; i < n; ++i) {
      a[i] = sample_uniform(seed, idx, (uint32_t)l, (uint32_t)i, m);
      b[i] = neg_mod(mad_mod(a[i], s[i], e[i], m), m.q);
    }
  }
}

void relin_message(uint64_t* evk, const uint64_t* s2, const int* limb_of, const uint64_t* w, int64_t E, int L,
                   int64_t n, const uint64_t* consts) {
  for (int64_t e = 0; e < E; ++e) {
    const int l = limb_of[e];
    const Modulus m = load_mod(consts, l);
    uint64_t* b = evk + (e * 2 * L + l) * n;
    const uint64_t* s = s2 + (int64_t)l * n;
    for (int64_t i = 0; i < n; ++i) b[i] = add_mod(b[i], mul_mod(w[e], s[i], m), m.q);
  }
}

void frac_encode(const double* vals, int64_t C, int n, int int_digits, int frac_digits,
                 int64_t* msg) {
#pragma omp parallel for schedule(static)
  for (int64_t c = 0; c < C; ++c) {
    int64_t* o = msg + c * n;
    std::memset(o, 0, sizeof(int64_t) * n);
    double v = vals[c];
    const int sgn = v < 0 ? -1 : 1;
    v = std::fabs(v);
    double ip = std::floor(v);
    double fp = v - ip;
    for (int i = 0; i < int_digits && ip > 0; ++i) {
      const double half = std::floor(ip / 2.0);
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

void frac_decode(const int64_t* coeffs, int64_t C, int n, int int_digits, int frac_digits,
                 double* out) {
#pragma omp parallel for schedule(static)
  for (int64_t c = 0; c < C; ++c) {
    const int64_t* x = coeffs + c * n;
    double acc = 0.0, w = 1.0;
    for (int i = 0; i < int_digits; ++i) { acc += (double)x[i] * w; w *= 2.0; }
    w = 0.5;
    for (int i = 1; i <= frac_digits; ++i) { acc -= (double)x[n - i] * w; w *= 0.5; }
    out[c] = acc;
  }
}

void bfv_scale_round(const uint64_t* x, int64_t C, int n, uint64_t q, uint64_t p, int64_t* out) {
#pragma omp parallel for schedule(static)
  for (int64_t g = 0; g < C * (int64_t)n; ++g) {
    const u128 num = (u128)x[g] * p + q / 2;
    uint64_t mval = (uint64_t)(num / q) % p;
    out[g] = mval > p / 2 ? (int64_t)mval - (int64_t)p : (int64_t)mval;
  }
}

void digit_extract(const uint64_t* x, int64_t rows, int n, int shift, int bits, uint64_t* out) {
  const uint64_t mask = bits >= 64 ? ~0ull : ((1ull << bits) - 1);
#pragma omp parallel for schedule(static)
  for (int64_t g = 0; g < rows * (int64_t)n; ++g) out[g] = (x[g] >> shift) & mask;
}

void shoup_pairs(const uint64_t* x, uint64_t* out, int64_t rows, int L, int n, const uint64_t* consts) {
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < rows; ++r) {
    const uint64_t q = consts[(size_t)(r % L) * kConstStride];
    for (int i = 0; i < n; ++i) {
      const uint64_t v = x[r * n + i];
      out[(r * n + i) * 2] = v;
      out[(r * n + i) * 2 + 1] = (uint64_t)(((u128)v << 64) / q);
    }
  }
}

}  // namespace host
}  // namespace hefl
