// torch.ops.hefl.* bindings for the HE core. Each op dispatches on the device of its
// tensor arguments: CUDA tensors go to the sm_90a kernels (kernels.h), CPU tensors to the
// host implementation (host_math.h). u64 words travel as torch.int64 (same bits).
#include <ATen/cuda/CUDAContext.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "host_math.h"
#include "kernels.h"

namespace {

using at::Tensor;

inline uint64_t* u64(const Tensor& t) {
  TORCH_CHECK(t.scalar_type() == at::kLong, "expected int64 tensor");
  TORCH_CHECK(t.is_contiguous(), "expected contiguous tensor");
  return reinterpret_cast<uint64_t*>(t.data_ptr<int64_t>());
}
inline const uint64_t* u64o(const c10::optional<Tensor>& t) {
  return t.has_value() ? u64(*t) : nullptr;
}
inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
inline void same_device(const Tensor& a, const Tensor& b) {
  TORCH_CHECK(a.device() == b.device(), "tensors on different devices: ", a.device(), " vs ", b.device());
}

// ---- fast-path companions, built once per table / key tensor and cached ---------------------
// The persistent kernels (csrc/he/cuda/he_kernels2.cu) want (w, w') interleaved twiddle tables
// and keys stored next to their Shoup companions. Callers keep passing the plain tensors; the
// derived ones are cached here, keyed by the data pointer of the tensor they were derived from
// (the cache holds a reference, so the pointer cannot be recycled while the entry lives).
struct TableExt {
  Tensor src, tw2;
  int qbits = 64;
};
struct KeyExt {
  Tensor src, ext;
  uint32_t version = 0;
};

inline bool fast_path_enabled() {
  static const bool on = [] {
    const char* e = std::getenv("HEFL_HE_V1");
    return !(e && e[0] == '1');
  }();
  return on;
}

const TableExt& table_ext(const Tensor& tables, const Tensor& consts) {
  static std::mutex mu;
  static std::unordered_map<const void*, TableExt> cache;
  std::lock_guard<std::mutex> g(mu);
  auto it = cache.find(tables.data_ptr());
  if (it != cache.end() && it->second.src.sizes() == tables.sizes()) return it->second;
  if (cache.size() > 256) cache.clear();
  TableExt e;
  e.src = tables;
  const int64_t L = tables.size(0), n = tables.size(2);
  // [L][4][N] = (w, w', iw, iw') planes  ->  [L][2 dir][N][2]
  e.tw2 = tables.view({L, 2, 2, n}).permute({0, 1, 3, 2}).contiguous();
  Tensor q = consts.select(1, 0).cpu();
  int bits = 0;
  for (int64_t l = 0; l < L; ++l) {
    const uint64_t v = (uint64_t)q.data_ptr<int64_t>()[l];
    bits = std::max(bits, 64 - __builtin_clzll(v));
  }
  e.qbits = bits;
  return cache[tables.data_ptr()] = std::move(e);
}

// x [..., L, N] (rows cycle through the limbs) -> [..., L, N, 2] = (x, floor(x * 2^64 / q_limb))
Tensor with_shoup(const Tensor& x, const Tensor& consts, int64_t L) {
  const int64_t n = x.size(-1);
  const int64_t rows = x.numel() / n;
  auto shape = x.sizes().vec();
  shape.push_back(2);
  Tensor out = at::empty(shape, x.options());
  if (x.is_cuda())
    hefl::cuda::shoup_pairs(u64(x), u64(out), rows, (int)L, (int)n, u64(consts), cur_stream());
  else
    hefl::host::shoup_pairs(u64(x), u64(out), rows, (int)L, (int)n, u64(consts));
  return out;
}

const Tensor& key_ext(const Tensor& key, const Tensor& consts, int64_t L) {
  static std::mutex mu;
  static std::unordered_map<const void*, KeyExt> cache;
  std::lock_guard<std::mutex> g(mu);
  auto it = cache.find(key.data_ptr());
  if (it != cache.end() && it->second.version == key._version() && it->second.src.sizes() == key.sizes())
    return it->second.ext;
  if (cache.size() > 256) cache.clear();
  KeyExt e;
  e.src = key;
  e.version = key._version();
  e.ext = with_shoup(key, consts, L);
  return (cache[key.data_ptr()] = std::move(e)).ext;
}

Tensor shoup_pairs(const Tensor& x, const Tensor& consts, int64_t L) {
  same_device(x, consts);
  TORCH_CHECK(x.is_contiguous(), "expected contiguous tensor");
  return with_shoup(x, consts, L);
}

Tensor gen_primes(int64_t bits, int64_t logn, int64_t count, at::IntArrayRef exclude) {
  std::vector<uint64_t> ex(exclude.begin(), exclude.end());
  auto p = hefl::host::gen_primes((int)bits, (int)logn, (int)count, ex);
  Tensor out = at::empty({(int64_t)p.size()}, at::kLong);
  for (size_t i = 0; i < p.size(); ++i) out.data_ptr<int64_t>()[i] = (int64_t)p[i];
  return out;
}

std::tuple<Tensor, Tensor> build_tables(const Tensor& moduli, int64_t logn) {
  TORCH_CHECK(moduli.is_cpu(), "moduli must be a CPU tensor");
  const int64_t L = moduli.numel(), n = 1ll << logn;
  Tensor tables = at::empty({L, 4, n}, at::kLong);
  Tensor consts = at::empty({L, 8}, at::kLong);
  hefl::host::build_tables(u64(moduli), (int)L, (int)logn, u64(tables), u64(consts));
  return {tables, consts};
}

std::tuple<Tensor, Tensor> build_fft_tables(int64_t logn) {
  const int64_t n = 1ll << logn;
  Tensor rot = at::empty({n / 2}, at::kInt);
  Tensor ksi = at::empty({2 * n + 1, 2}, at::kDouble);
  hefl::host::build_fft_tables((int)logn, rot.data_ptr<int32_t>(), ksi.data_ptr<double>());
  return {rot, ksi};
}

void ntt_(Tensor data, const Tensor& tables, const Tensor& consts, int64_t L, int64_t logn,
          bool inverse) {
  same_device(data, tables);
  const int64_t n = 1ll << logn;
  TORCH_CHECK(data.size(-1) == n, "last dim must be N");
  const int64_t rows = data.numel() / n;
  if (data.is_cuda()) {
    if (fast_path_enabled() && tables.size(0) == L && rows % L == 0) {
      const TableExt& te = table_ext(tables, consts);
      if (hefl::cuda::ntt2(u64(data), rows, (int)L, (int)logn, u64(te.tw2), u64(consts), te.qbits, inverse, cur_stream()))
        return;
    }
    hefl::cuda::ntt(u64(data), rows, (int)L, (int)logn, u64(tables), u64(consts), inverse, cur_stream());
  } else
    hefl::host::ntt(u64(data), rows, (int)L, (int)logn, u64(tables), u64(consts), inverse);
}

void pointwise_(Tensor out, const Tensor& a, const c10::optional<Tensor>& b, int64_t L,
                const Tensor& consts, int64_t op) {
  same_device(out, a);
  same_device(out, consts);
  const int64_t n = a.size(-1);
  const int64_t rows = a.numel() / n;
  TORCH_CHECK(out.numel() == a.numel(), "out/a size mismatch");
  int64_t brows = 1;
  if (b.has_value()) {
    same_device(out, *b);
    if (op == 5) {
      TORCH_CHECK(b->numel() >= L, "scalar vector too short");
    } else {
      TORCH_CHECK(b->size(-1) == n, "b last dim mismatch");
      brows = b->numel() / n;
      TORCH_CHECK(rows % brows == 0, "b rows must divide a rows");
    }
  } else {
    TORCH_CHECK(op == 4, "b required");
  }
  if (out.is_cuda())
    hefl::cuda::pointwise(u64(out), u64(a), u64o(b), rows, brows, (int)L, (int)n, u64(consts), (int)op, cur_stream());
  else
    hefl::host::pointwise(u64(out), u64(a), u64o(b), rows, brows, (int)L, (int)n, u64(consts), (int)op);
}

void reduce_mod_(Tensor data, int64_t L, const Tensor& consts) {
  same_device(data, consts);
  const int64_t n = data.size(-1);
  const int64_t rows = data.numel() / n;
  if (data.is_cuda())
    hefl::cuda::reduce_mod(u64(data), rows, (int)L, (int)n, u64(consts), cur_stream());
  else
    hefl::host::reduce_mod(u64(data), rows, (int)L, (int)n, u64(consts));
}

Tensor ckks_encode(const Tensor& vals, int64_t C, int64_t logn, double scale, const Tensor& rot,
                   const Tensor& ksi) {
  same_device(vals, rot);
  TORCH_CHECK(vals.is_contiguous(), "vals must be contiguous");
  const int64_t n = 1ll << logn;
  const bool f32 = vals.scalar_type() == at::kFloat;
  TORCH_CHECK(f32 || vals.scalar_type() == at::kDouble, "vals must be float32 or float64");
  TORCH_CHECK(vals.numel() <= C * n / 2, "too many values for C ciphertexts");
  Tensor msg = at::empty({C, n}, vals.options().dtype(at::kLong));
  const float* pf = f32 ? vals.data_ptr<float>() : nullptr;
  const double* pd = f32 ? nullptr : vals.data_ptr<double>();
  if (vals.is_cuda()) {
    Tensor scratch;
    double* sp = nullptr;
    if (logn > 14) {
      scratch = at::empty({C, n / 2, 2}, vals.options().dtype(at::kDouble));
      sp = scratch.data_ptr<double>();
    }
    hefl::cuda::ckks_encode(pf, pd, C, vals.numel(), (int)logn, scale, rot.data_ptr<int32_t>(),
                            ksi.data_ptr<double>(), msg.data_ptr<int64_t>(), sp, cur_stream());
  } else {
    hefl::host::ckks_encode(pf, pd, C, vals.numel(), (int)logn, scale, rot.data_ptr<int32_t>(),
                            ksi.data_ptr<double>(), msg.data_ptr<int64_t>());
  }
  return msg;
}

Tensor coeff_encode(const Tensor& vals, int64_t C, int64_t n, double scale) {
  TORCH_CHECK(vals.scalar_type() == at::kFloat && vals.is_contiguous(), "vals must be contiguous float32");
  TORCH_CHECK(vals.numel() <= C * n, "too many values");
  Tensor msg = at::empty({C, n}, vals.options().dtype(at::kLong));
  if (vals.is_cuda())
    hefl::cuda::coeff_encode(vals.data_ptr<float>(), C, vals.numel(), (int)n, scale, msg.data_ptr<int64_t>(), cur_stream());
  else
    hefl::host::coeff_encode(vals.data_ptr<float>(), C, vals.numel(), (int)n, scale, msg.data_ptr<int64_t>());
  return msg;
}

Tensor crt_center(const Tensor& res, const Tensor& consts_cpu, int64_t q0_inv_q1) {
  TORCH_CHECK(res.dim() == 3, "res must be [C,k,N]");
  TORCH_CHECK(consts_cpu.is_cpu(), "consts_cpu must live on the CPU");
  const int64_t C = res.size(0), k = res.size(1), n = res.size(2);
  TORCH_CHECK(k == 1 || k == 2, "crt_center supports 1 or 2 limbs");
  Tensor out = at::empty({C, n}, res.options().dtype(at::kDouble));
  const uint64_t* cc = u64(consts_cpu);
  if (res.is_cuda()) {
    hefl::cuda::crt_center(u64(res), C, (int)k, (int)n, cc[0], k > 1 ? cc[8] : 1, k > 1 ? cc[9] : 0,
                           k > 1 ? cc[10] : 0, (uint64_t)q0_inv_q1, out.data_ptr<double>(), cur_stream());
  } else {
    hefl::host::crt_center(u64(res), C, (int)k, (int)n, cc, out.data_ptr<double>());
  }
  return out;
}

Tensor ckks_decode(const Tensor& coeffs, int64_t logn, double inv_scale, const Tensor& rot,
                   const Tensor& ksi, bool as_f64) {
  same_device(coeffs, rot);
  TORCH_CHECK(coeffs.scalar_type() == at::kDouble && coeffs.is_contiguous(), "coeffs must be contiguous float64");
  const int64_t n = 1ll << logn;
  const int64_t C = coeffs.numel() / n;
  Tensor out = at::empty({C, n / 2}, coeffs.options().dtype(as_f64 ? at::kDouble : at::kFloat));
  float* of = as_f64 ? nullptr : out.data_ptr<float>();
  double* od = as_f64 ? out.data_ptr<double>() : nullptr;
  if (coeffs.is_cuda()) {
    Tensor scratch;
    double* sp = nullptr;
    if (logn > 14) {
      scratch = at::empty({C, n / 2, 2}, coeffs.options());
      sp = scratch.data_ptr<double>();
    }
    hefl::cuda::ckks_decode(coeffs.data_ptr<double>(), C, (int)logn, inv_scale, rot.data_ptr<int32_t>(),
                            ksi.data_ptr<double>(), of, od, sp, cur_stream());
  } else {
    hefl::host::ckks_decode(coeffs.data_ptr<double>(), C, (int)logn, inv_scale, rot.data_ptr<int32_t>(),
                            ksi.data_ptr<double>(), of, od);
  }
  return out;
}

// Decrypted residues [C,k,N] -> flat float32 values [nvals] (CRT + /scale + special FFT fused on GPU).
Tensor ckks_decode_residues(const Tensor& res, const Tensor& consts_cpu, int64_t q0_inv_q1,
                            int64_t logn, double inv_scale, const Tensor& rot, const Tensor& ksi,
                            int64_t nvals) {
  TORCH_CHECK(res.dim() == 3, "res must be [C,k,N]");
  const int64_t C = res.size(0), k = res.size(1), n = res.size(2);
  TORCH_CHECK(n == (1ll << logn), "N mismatch");
  TORCH_CHECK(nvals <= C * n / 2, "nvals too large");
  if (res.is_cuda()) {
    const uint64_t* cc = u64(consts_cpu);
    Tensor out = at::empty({nvals}, res.options().dtype(at::kFloat));
    Tensor scratch;
    double* sp = nullptr;
    if (logn > 14) {
      scratch = at::empty({C, n / 2, 2}, res.options().dtype(at::kDouble));
      sp = scratch.data_ptr<double>();
    }
    hefl::cuda::ckks_decode_residues(u64(res), C, (int)k, (int)logn, cc[0], k > 1 ? cc[8] : 1,
                                     k > 1 ? cc[9] : 0, k > 1 ? cc[10] : 0, (uint64_t)q0_inv_q1,
                                     inv_scale, rot.data_ptr<int32_t>(), ksi.data_ptr<double>(),
                                     out.data_ptr<float>(), nvals, sp, cur_stream());
    return out;
  }
  Tensor coeffs = crt_center(res, consts_cpu, q0_inv_q1);
  Tensor full = ckks_decode(coeffs, logn, inv_scale, rot, ksi, false);
  return full.reshape({-1}).slice(0, 0, nvals).contiguous();
}

// Decrypted residues [C,k,N] of flat values g0 .. g0 + nvals - 1 -> one server-optimizer step (DESIGN.md §8):
// x_new = step(x_t, average), m and v updated in place for the indices below n_trainable. One launch on CUDA
// (ckks_decode_step_kernel<opt>); on CPU the host twin. avg_out (fp32 or fp64) also receives
// the decoded average.
void ckks_decode_server_step_(const Tensor& res, const Tensor& consts_cpu, int64_t q0_inv_q1, int64_t logn,
                              double inv_scale, const Tensor& rot, const Tensor& ksi, int64_t nvals, int64_t g0,
                              int64_t n_trainable, const Tensor& x_t, Tensor x_new, Tensor m, Tensor v, int64_t opt,
                              double lr, double beta1, double beta2, double tau,
                              const c10::optional<Tensor>& avg_out) {
  TORCH_CHECK(res.dim() == 3, "res must be [C,k,N]");
  const int64_t C = res.size(0), k = res.size(1), n = res.size(2);
  TORCH_CHECK(k == 1 || k == 2, "the decode supports 1 or 2 limbs");
  TORCH_CHECK(n == (1ll << logn), "N mismatch");
  TORCH_CHECK(consts_cpu.is_cpu(), "consts_cpu must live on the CPU");
  same_device(res, rot);
  same_device(res, ksi);
  TORCH_CHECK(opt >= hefl::kFedAvgM && opt <= hefl::kFedAdam, "opt must be 1 (fedavgm), 2 (fedadagrad), 3 (fedyogi) or 4 (fedadam), got ", opt);
  TORCH_CHECK(nvals >= 0 && nvals <= C * n / 2, "nvals too large");
  TORCH_CHECK(g0 >= 0 && n_trainable >= 0, "g0 and n_trainable must be >= 0");
  const int64_t end = g0 + nvals;
  const int64_t n_state = std::max<int64_t>(0, std::min(n_trainable, end));
  auto check_f32 = [&](const Tensor& t, const char* name, int64_t need) {
    same_device(res, t);
    TORCH_CHECK(t.scalar_type() == at::kFloat && t.is_contiguous(), name, " must be contiguous float32");
    TORCH_CHECK(t.numel() >= need, name, " has ", t.numel(), " elements, needs ", need);
  };
  check_f32(x_t, "x_t", end);
  check_f32(x_new, "x_new", end);
  check_f32(m, "m", n_state);
  check_f32(v, "v", n_state);
  hefl::ServerStep sv;
  sv.x_t = x_t.data_ptr<float>();
  sv.x_new = x_new.data_ptr<float>();
  sv.m = m.data_ptr<float>();
  sv.v = v.data_ptr<float>();
  if (avg_out.has_value()) {
    same_device(res, *avg_out);
    const bool f64 = avg_out->scalar_type() == at::kDouble;
    TORCH_CHECK((f64 || avg_out->scalar_type() == at::kFloat) && avg_out->is_contiguous(),
                "avg_out must be contiguous float32 or float64");
    TORCH_CHECK(avg_out->numel() >= end, "avg_out has ", avg_out->numel(), " elements, needs ", end);
    if (f64) sv.avg_f64 = avg_out->data_ptr<double>();
    else sv.avg_f32 = avg_out->data_ptr<float>();
  }
  sv.g0 = g0;
  sv.n_trainable = n_trainable;
  sv.lr = (float)lr;
  sv.beta1 = (float)beta1;
  sv.beta2 = (float)beta2;
  sv.tau = (float)tau;
  if (nvals == 0) return;
  if (res.is_cuda()) {
    const uint64_t* cc = u64(consts_cpu);
    Tensor scratch;
    double* sp = nullptr;
    if (logn > 14) {
      scratch = at::empty({C, n / 2, 2}, res.options().dtype(at::kDouble));
      sp = scratch.data_ptr<double>();
    }
    hefl::cuda::ckks_decode_server_step(u64(res), C, (int)k, (int)logn, cc[0], k > 1 ? cc[8] : 1,
                                        k > 1 ? cc[9] : 0, k > 1 ? cc[10] : 0, (uint64_t)q0_inv_q1, inv_scale,
                                        rot.data_ptr<int32_t>(), ksi.data_ptr<double>(), nvals, sv, (int)opt, sp,
                                        cur_stream());
    return;
  }
  Tensor coeffs = crt_center(res, consts_cpu, q0_inv_q1);
  hefl::host::ckks_decode_server_step(coeffs.data_ptr<double>(), C, (int)logn, inv_scale, rot.data_ptr<int32_t>(),
                                      ksi.data_ptr<double>(), nvals, sv, (int)opt);
}

void encrypt_out(const c10::optional<Tensor>& msg, const Tensor& pk, int64_t C, int64_t L, int64_t logn,
                 const Tensor& tables, const Tensor& consts, const c10::optional<Tensor>& msg_scale,
                 int64_t seed, int64_t ct_offset, Tensor ct, bool accumulate) {
  same_device(pk, tables);
  same_device(pk, ct);
  const int64_t n = 1ll << logn;
  TORCH_CHECK(pk.numel() == 2 * L * n, "pk must be [2,L,N]");
  TORCH_CHECK(ct.numel() >= C * 2 * L * n, "output buffer too small");
  TORCH_CHECK(!accumulate || ct.is_contiguous(), "accumulate reads the output buffer: it must be contiguous");
  const int64_t* mp = nullptr;
  if (msg.has_value()) {
    same_device(*msg, pk);
    TORCH_CHECK(msg->numel() == C * n && msg->is_contiguous(), "msg must be contiguous [C,N]");
    mp = msg->data_ptr<int64_t>();
  }
  if (pk.is_cuda()) {
    if (fast_path_enabled() && tables.size(0) == L) {
      const TableExt& te = table_ext(tables, consts);
      if (hefl::cuda::ntt2_supported((int)logn, (int)L, te.qbits) && logn <= 14) {
        const Tensor& pkx = key_ext(pk, consts, L);
        // per-launch scratch from the caching allocator on this stream (as ckks_encode's N = 32768 scratch)
        Tensor scratch;
        if (const int64_t words = hefl::cuda::encrypt2_scratch_words((int)logn)) scratch = at::empty({words}, pk.options());
        if (hefl::cuda::encrypt2(mp, u64(pkx), u64(ct), C, (int)L, (int)logn, u64(te.tw2), u64(consts),
                                 u64o(msg_scale), (uint64_t)seed, (uint32_t)ct_offset, te.qbits,
                                 scratch.defined() ? u64(scratch) : nullptr, accumulate, cur_stream()))
          return;
      }
    }
    hefl::cuda::encrypt(mp, u64(pk), u64(ct), C, (int)L, (int)logn, u64(tables), u64(consts),
                        u64o(msg_scale), (uint64_t)seed, (uint32_t)ct_offset, accumulate, cur_stream());
  } else
    hefl::host::encrypt(mp, u64(pk), u64(ct), C, (int)L, (int)logn, u64(tables), u64(consts),
                        u64o(msg_scale), (uint64_t)seed, (uint32_t)ct_offset, accumulate);
}

Tensor encrypt(const c10::optional<Tensor>& msg, const Tensor& pk, int64_t C, int64_t L, int64_t logn,
               const Tensor& tables, const Tensor& consts, const c10::optional<Tensor>& msg_scale,
               int64_t seed, int64_t ct_offset) {
  Tensor ct = at::empty({C, 2, L, 1ll << logn}, pk.options());
  encrypt_out(msg, pk, C, L, logn, tables, consts, msg_scale, seed, ct_offset, ct, false);
  return ct;
}

Tensor decrypt(const Tensor& ct, const Tensor& sk, int64_t k, int64_t logn, const Tensor& tables,
               const Tensor& consts) {
  same_device(ct, sk);
  TORCH_CHECK(ct.dim() == 4 && ct.size(1) == 2, "ct must be [C,2,L,N]");
  const int64_t C = ct.size(0), Lct = ct.size(2), n = ct.size(3);
  TORCH_CHECK(k >= 1 && k <= Lct, "bad k");
  Tensor out = at::empty({C, k, n}, ct.options());
  if (ct.is_cuda()) {
    if (fast_path_enabled()) {
      const TableExt& te = table_ext(tables, consts);
      const int64_t Ltab = tables.size(0);
      if (hefl::cuda::ntt2_supported((int)logn, (int)k, te.qbits) && sk.numel() == Ltab * n) {
        const Tensor& skx = key_ext(sk, consts, Ltab);
        if (hefl::cuda::decrypt2(u64(ct), u64(skx), u64(out), C, (int)Lct, (int)k, (int)logn, u64(te.tw2),
                                 u64(consts), (int)Ltab, te.qbits, cur_stream()))
          return out;
      }
    }
    hefl::cuda::decrypt(u64(ct), u64(sk), u64(out), C, (int)Lct, (int)k, (int)logn, u64(tables), u64(consts), cur_stream());
  } else
    hefl::host::decrypt(u64(ct), u64(sk), u64(out), C, (int)Lct, (int)k, (int)logn, u64(tables), u64(consts));
  return out;
}

// Key generation: host twin for CPU tables, device kernels (csrc/he/cuda/he_kernels.cu) for CUDA tables; the two are
// bit-identical for a given seed (tests/test_gpu_he.py).
Tensor keygen_secret(int64_t L, int64_t logn, const Tensor& tables, const Tensor& consts, int64_t seed) {
  same_device(tables, consts);
  Tensor sk = at::empty({L, 1ll << logn}, tables.options().dtype(at::kLong));
  if (tables.is_cuda()) {
    hefl::cuda::keygen_sample(u64(sk), 1, (int)L, 1 << logn, u64(consts), (uint64_t)seed, 0u, 0, cur_stream());
    ntt_(sk, tables, consts, L, logn, false);
  } else {
    hefl::host::sample_secret(u64(sk), (int)L, (int)logn, u64(tables), u64(consts), (uint64_t)seed);
  }
  return sk;
}

// E public-key-shaped pairs (-(a s + e), a) with stream indices idx0 .. idx0 + E - 1: [E, 2, L, N]
Tensor keygen_public_batch(const Tensor& sk, int64_t L, int64_t logn, const Tensor& tables, const Tensor& consts,
                           int64_t seed, int64_t idx0, int64_t E) {
  same_device(tables, consts);
  same_device(tables, sk);
  const int64_t n = 1ll << logn;
  TORCH_CHECK(sk.numel() == L * n && sk.is_contiguous() && E >= 1, "sk must be contiguous [L, N]");
  Tensor pk = at::zeros({E, 2, L, n}, tables.options().dtype(at::kLong));
  if (tables.is_cuda()) {
    hefl::cuda::keygen_sample(u64(pk), (int)E, (int)L, (int)n, u64(consts), (uint64_t)seed, (uint32_t)idx0, 1, cur_stream());
    ntt_(pk, tables, consts, L, logn, false);           // slot 1 is still zero: transformed along, then overwritten
    hefl::cuda::keygen_finish(u64(sk), u64(pk), (int)E, (int)L, (int)n, u64(consts), (uint64_t)seed, (uint32_t)idx0, cur_stream());
  } else {
    for (int64_t e = 0; e < E; ++e)
      hefl::host::gen_public(u64(sk), u64(pk) + e * 2 * L * n, (int)L, (int)logn, u64(tables), u64(consts), (uint64_t)seed,
                             (uint32_t)(idx0 + e));
  }
  return pk;
}

Tensor keygen_public(const Tensor& sk, int64_t L, int64_t logn, const Tensor& tables,
                     const Tensor& consts, int64_t seed, int64_t idx) {
  return keygen_public_batch(sk, L, logn, tables, consts, seed, idx, 1).squeeze(0);
}

// evk [E, 2, L, N]: slot 0, limb limb_of[e] += w[e] * s2[limb_of[e]] (message term of the digit-decomposed key)
void relin_message_(Tensor evk, const Tensor& s2, const Tensor& limb_of, const Tensor& w, int64_t L, const Tensor& consts) {
  same_device(evk, s2);
  same_device(evk, consts);
  const int64_t n = s2.size(-1), E = evk.size(0);
  TORCH_CHECK(evk.dim() == 4 && evk.size(1) == 2 && evk.size(2) == L && evk.size(3) == n && evk.is_contiguous() &&
              s2.numel() == L * n && s2.is_contiguous(), "evk must be [E,2,L,N], s2 [L,N]");
  TORCH_CHECK(limb_of.scalar_type() == at::kInt && w.scalar_type() == at::kLong && limb_of.numel() == E && w.numel() == E,
              "limb_of int32 [E], w int64 [E]");
  if (evk.is_cuda()) {
    same_device(evk, limb_of);
    same_device(evk, w);
    hefl::cuda::relin_message(u64(evk), u64(s2), limb_of.data_ptr<int>(), u64(w), (int)E, (int)L, (int)n, u64(consts), cur_stream());
  } else {
    const int* lo = limb_of.data_ptr<int>();
    for (int64_t e = 0; e < E; ++e) TORCH_CHECK(lo[e] >= 0 && lo[e] < L, "limb index");
    hefl::host::relin_message(u64(evk), u64(s2), lo, u64(w), E, (int)L, n, u64(consts));
  }
}

Tensor frac_encode(const Tensor& vals, int64_t n, int64_t int_digits, int64_t frac_digits) {
  TORCH_CHECK(vals.scalar_type() == at::kDouble && vals.is_contiguous(), "vals must be contiguous float64");
  const int64_t C = vals.numel();
  Tensor msg = at::empty({C, n}, vals.options().dtype(at::kLong));
  if (vals.is_cuda())
    hefl::cuda::frac_encode(vals.data_ptr<double>(), C, (int)n, (int)int_digits, (int)frac_digits, msg.data_ptr<int64_t>(), cur_stream());
  else
    hefl::host::frac_encode(vals.data_ptr<double>(), C, (int)n, (int)int_digits, (int)frac_digits, msg.data_ptr<int64_t>());
  return msg;
}

Tensor frac_decode(const Tensor& coeffs, int64_t int_digits, int64_t frac_digits) {
  TORCH_CHECK(coeffs.scalar_type() == at::kLong && coeffs.is_contiguous() && coeffs.dim() == 2, "coeffs must be contiguous int64 [C,N]");
  const int64_t C = coeffs.size(0), n = coeffs.size(1);
  Tensor out = at::empty({C}, coeffs.options().dtype(at::kDouble));
  if (coeffs.is_cuda())
    hefl::cuda::frac_decode(coeffs.data_ptr<int64_t>(), C, (int)n, (int)int_digits, (int)frac_digits, out.data_ptr<double>(), cur_stream());
  else
    hefl::host::frac_decode(coeffs.data_ptr<int64_t>(), C, (int)n, (int)int_digits, (int)frac_digits, out.data_ptr<double>());
  return out;
}

Tensor bfv_scale_round(const Tensor& x, int64_t q, int64_t p) {
  const int64_t n = x.size(-1);
  const int64_t C = x.numel() / n;
  Tensor out = at::empty_like(x);
  if (x.is_cuda())
    hefl::cuda::bfv_scale_round(u64(x), C, (int)n, (uint64_t)q, (uint64_t)p, out.data_ptr<int64_t>(), cur_stream());
  else
    hefl::host::bfv_scale_round(u64(x), C, (int)n, (uint64_t)q, (uint64_t)p, out.data_ptr<int64_t>());
  return out;
}

Tensor digit_extract(const Tensor& x, int64_t shift, int64_t bits) {
  const int64_t n = x.size(-1);
  const int64_t rows = x.numel() / n;
  Tensor out = at::empty_like(x);
  if (x.is_cuda())
    hefl::cuda::digit_extract(u64(x), rows, (int)n, (int)shift, (int)bits, u64(out), cur_stream());
  else
    hefl::host::digit_extract(u64(x), rows, (int)n, (int)shift, (int)bits, u64(out));
  return out;
}

// ct [C,2,lvl,N] -> round(ct / q_last) [C,2,lvl-1,N] in one launch. Returns an empty tensor when the fused kernel
// does not cover the parameters (CPU tensors, N >= 16384, primes >= 2^58): the caller runs the reference loop.
Tensor rescale_fused(const Tensor& ct, const Tensor& tables, const Tensor& consts, const Tensor& consts_cpu, int64_t logn) {
  TORCH_CHECK(ct.dim() == 4 && ct.size(1) == 2 && ct.is_contiguous(), "ct must be contiguous [C,2,lvl,N]");
  const int64_t C = ct.size(0), lvl = ct.size(2), n = ct.size(3);
  if (!ct.is_cuda() || !fast_path_enabled() || lvl < 2 || tables.size(0) < lvl) return Tensor();
  const TableExt& te = table_ext(tables, consts);
  const uint64_t* cc = u64(consts_cpu);
  const uint64_t ql = cc[(lvl - 1) * 8];
  std::vector<uint64_t> inv(lvl), invp(lvl);
  for (int64_t j = 0; j + 1 < lvl; ++j) {
    const uint64_t qj = cc[j * 8];
    inv[j] = hefl::host::inv_mod(ql % qj, qj);
    invp[j] = (uint64_t)(((unsigned __int128)inv[j] << 64) / qj);
  }
  Tensor out = at::empty({C, 2, lvl - 1, n}, ct.options());
  if (!hefl::cuda::rescale2(u64(ct), u64(out), C, (int)lvl, (int)logn, u64(te.tw2), u64(consts), inv.data(), invp.data(),
                            te.qbits, cur_stream()))
    return Tensor();
  return out;
}

// acc [C,2,lvl,N] (holding d0, d1) += key switch of d2 given in COEFFICIENT form [C,lvl,N]; evk [E,2,Ltab,N].
bool keyswitch_fused_(Tensor acc, const Tensor& coef, const Tensor& evk, at::IntArrayRef ndig, at::IntArrayRef first,
                      int64_t digit_bits, const Tensor& tables, const Tensor& consts, int64_t logn) {
  if (!acc.is_cuda() || !fast_path_enabled()) return false;
  TORCH_CHECK(acc.dim() == 4 && acc.is_contiguous() && coef.is_contiguous() && evk.is_contiguous(), "contiguous tensors expected");
  const int64_t C = acc.size(0), lvl = acc.size(2);
  TORCH_CHECK((int64_t)ndig.size() == lvl && (int64_t)first.size() == lvl, "one digit count per limb");
  const TableExt& te = table_ext(tables, consts);
  std::vector<int> nd(ndig.begin(), ndig.end()), fi(first.begin(), first.end());
  return hefl::cuda::keyswitch2(u64(coef), u64(evk), u64(acc), C, (int)lvl, (int)tables.size(0), (int)logn, (int)digit_bits,
                                nd.data(), fi.data(), u64(te.tw2), u64(consts), te.qbits, cur_stream());
}

// (a0 b0, a0 b1 + a1 b0) as a ciphertext-shaped tensor and a1 b1, element-wise (CUDA only).
std::tuple<Tensor, Tensor> ct_tensor(const Tensor& a, const Tensor& b, const Tensor& consts) {
  TORCH_CHECK(a.is_cuda() && a.dim() == 4 && a.sizes() == b.sizes() && a.is_contiguous() && b.is_contiguous(), "bad operands");
  const int64_t C = a.size(0), lvl = a.size(2), n = a.size(3);
  Tensor d01 = at::empty_like(a);
  Tensor d2 = at::empty({C, lvl, n}, a.options());
  hefl::cuda::ct_tensor(u64(a), u64(b), u64(d01), u64(d2), C, (int)lvl, (int)n, u64(consts), cur_stream());
  return {d01, d2};
}

int64_t launch_count() { return (int64_t)hefl::cuda::launch_count(); }
void set_he_cta_limits(int64_t ntt, int64_t enc, int64_t dec) { hefl::cuda::set_cta_limits((int)ntt, (int)enc, (int)dec); }

}  // namespace

TORCH_LIBRARY_FRAGMENT(hefl, m) {
  m.def("gen_primes(int bits, int logn, int count, int[] exclude) -> Tensor", &gen_primes);
  m.def("build_tables(Tensor moduli, int logn) -> (Tensor, Tensor)", &build_tables);
  m.def("build_fft_tables(int logn) -> (Tensor, Tensor)", &build_fft_tables);
  m.def("ntt_(Tensor(a!) data, Tensor tables, Tensor consts, int L, int logn, bool inverse) -> ()", &ntt_);
  m.def("pointwise_(Tensor(a!) out, Tensor a, Tensor? b, int L, Tensor consts, int op) -> ()", &pointwise_);
  m.def("reduce_mod_(Tensor(a!) data, int L, Tensor consts) -> ()", &reduce_mod_);
  m.def("ckks_encode(Tensor vals, int C, int logn, float scale, Tensor rot, Tensor ksi) -> Tensor", &ckks_encode);
  m.def("coeff_encode(Tensor vals, int C, int n, float scale) -> Tensor", &coeff_encode);
  m.def("crt_center(Tensor res, Tensor consts_cpu, int q0_inv_q1) -> Tensor", &crt_center);
  m.def("ckks_decode(Tensor coeffs, int logn, float inv_scale, Tensor rot, Tensor ksi, bool as_f64) -> Tensor", &ckks_decode);
  m.def("ckks_decode_residues(Tensor res, Tensor consts_cpu, int q0_inv_q1, int logn, float inv_scale, Tensor rot, Tensor ksi, int nvals) -> Tensor", &ckks_decode_residues);
  m.def("ckks_decode_server_step_(Tensor res, Tensor consts_cpu, int q0_inv_q1, int logn, float inv_scale, Tensor rot, Tensor ksi, int nvals, int g0, int n_trainable, Tensor x_t, Tensor(a!) x_new, Tensor(b!) m, Tensor(c!) v, int opt, float lr, float beta1, float beta2, float tau, Tensor(d!)? avg_out=None) -> ()", &ckks_decode_server_step_);
  m.def("encrypt(Tensor? msg, Tensor pk, int C, int L, int logn, Tensor tables, Tensor consts, Tensor? msg_scale, int seed, int ct_offset) -> Tensor", &encrypt);
  m.def("encrypt_out(Tensor? msg, Tensor pk, int C, int L, int logn, Tensor tables, Tensor consts, Tensor? msg_scale, int seed, int ct_offset, Tensor(a!) out, bool accumulate=False) -> ()", &encrypt_out);
  m.def("decrypt(Tensor ct, Tensor sk, int k, int logn, Tensor tables, Tensor consts) -> Tensor", &decrypt);
  m.def("keygen_secret(int L, int logn, Tensor tables, Tensor consts, int seed) -> Tensor", &keygen_secret);
  m.def("keygen_public(Tensor sk, int L, int logn, Tensor tables, Tensor consts, int seed, int idx) -> Tensor", &keygen_public);
  m.def("keygen_public_batch(Tensor sk, int L, int logn, Tensor tables, Tensor consts, int seed, int idx0, int E) -> Tensor", &keygen_public_batch);
  m.def("relin_message_(Tensor(a!) evk, Tensor s2, Tensor limb_of, Tensor w, int L, Tensor consts) -> ()", &relin_message_);
  m.def("frac_encode(Tensor vals, int n, int int_digits, int frac_digits) -> Tensor", &frac_encode);
  m.def("frac_decode(Tensor coeffs, int int_digits, int frac_digits) -> Tensor", &frac_decode);
  m.def("bfv_scale_round(Tensor x, int q, int p) -> Tensor", &bfv_scale_round);
  m.def("digit_extract(Tensor x, int shift, int bits) -> Tensor", &digit_extract);
  m.def("shoup_pairs(Tensor x, Tensor consts, int L) -> Tensor", &shoup_pairs);
  m.def("rescale_fused(Tensor ct, Tensor tables, Tensor consts, Tensor consts_cpu, int logn) -> Tensor", &rescale_fused);
  m.def("keyswitch_fused_(Tensor(a!) acc, Tensor coef, Tensor evk, int[] ndig, int[] first, int digit_bits, Tensor tables, Tensor consts, int logn) -> bool", &keyswitch_fused_);
  m.def("ct_tensor(Tensor a, Tensor b, Tensor consts) -> (Tensor, Tensor)", &ct_tensor);
  m.def("launch_count() -> int", &launch_count);
  m.def("set_he_cta_limits(int ntt, int enc, int dec) -> ()", &set_he_cta_limits);
}
