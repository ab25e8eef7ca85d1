// torch.ops.hefl.* bindings for the communication layer: the fused ciphertext all-reduce,
// a local K-way modular sum (loopback / file-drop aggregation), and a CUDA-IPC fallback for
// obtaining peer-mapped buffers when torch symmetric memory is unavailable.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <cstring>

#include "../he/modarith.h"
#include "../he/philox.h"
#include "comm.h"

namespace hefl {
namespace comm {
// CPU twin of pairwise_mask_kernel (gloo / loopback transports, tests).
void pairwise_mask_host(uint64_t* data, int64_t numel, int L, int logn, const MaskArgs& m) {
  const int64_t pairs = numel >> 1;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < pairs; ++i) {
    const int64_t e = i << 1;
    const int l = (int)((e >> logn) % L);
    const Modulus mod{m.q[l], m.ratio_lo[l], m.ratio_hi[l]};
    uint64_t x = data[e], y = data[e + 1];
    for (int j = 0; j < m.npeers; ++j) {
      const Philox4 r = philox4x32_10((uint32_t)i, (uint32_t)(i >> 32), m.round, 9u, (uint32_t)m.seed[j],
                                      (uint32_t)(m.seed[j] >> 32));
      const uint64_t a0 = barrett_reduce_64(((uint64_t)r.x << 32) | r.y, mod);
      const uint64_t a1 = barrett_reduce_64(((uint64_t)r.z << 32) | r.w, mod);
      if (m.sign[j] > 0) {
        x = add_mod(x, a0, mod.q);
        y = add_mod(y, a1, mod.q);
      } else {
        x = sub_mod(x, a0, mod.q);
        y = sub_mod(y, a1, mod.q);
      }
    }
    data[e] = x;
    data[e + 1] = y;
  }
}
}  // namespace comm
}  // namespace hefl

namespace {

using at::Tensor;

inline uint64_t* u64(const Tensor& t) {
  TORCH_CHECK(t.scalar_type() == at::kLong && t.is_contiguous(), "expected contiguous int64 tensor");
  return reinterpret_cast<uint64_t*>(t.data_ptr<int64_t>());
}

void allreduce_modq(at::IntArrayRef buf_ptrs, at::IntArrayRef sig_ptrs, int64_t mc_ptr,
                    const c10::optional<Tensor>& out, const Tensor& status, const Tensor& consts_cpu,
                    int64_t numel, int64_t L, int64_t logn, int64_t rank, int64_t world, int64_t algo,
                    int64_t blocks, int64_t threads, int64_t timeout_ms, int64_t no_owner,
                    const c10::optional<Tensor>& stats) {
  TORCH_CHECK(world >= 1 && world <= hefl::comm::kMaxWorld, "world size must be 1..8");
  TORCH_CHECK((int64_t)buf_ptrs.size() == world && (int64_t)sig_ptrs.size() == world, "need one pointer per rank");
  TORCH_CHECK(L >= 1 && L <= hefl::comm::kMaxLimbs, "too many limbs");
  TORCH_CHECK(numel % 4 == 0, "numel must be a multiple of 4 words");
  TORCH_CHECK(no_owner < world, "no_owner must be a rank or -1");
  TORCH_CHECK(!(no_owner >= 0 && (algo == 1 || world < 2)), "a key holder needs two_shot / multimem and >= 2 ranks");
  TORCH_CHECK(consts_cpu.is_cpu() && consts_cpu.size(0) >= L, "consts_cpu must be the CPU consts table");
  TORCH_CHECK(threads >= world && threads <= 512 && threads % 32 == 0, "bad thread count");
  hefl::comm::AllReduceArgs a;
  std::memset(&a, 0, sizeof(a));
  for (int i = 0; i < world; ++i) {
    a.bufs[i] = reinterpret_cast<uint64_t*>(buf_ptrs[i]);
    a.sigs[i] = reinterpret_cast<uint32_t*>(sig_ptrs[i]);
  }
  a.mc = reinterpret_cast<uint64_t*>(mc_ptr);
  if (algo == 2) TORCH_CHECK(mc_ptr != 0, "multimem algorithm needs a multicast pointer");
  if (algo == 1) {
    TORCH_CHECK(out.has_value() && out->is_cuda() && out->numel() >= numel, "one_shot needs an output buffer");
    a.out = u64(*out);
  }
  TORCH_CHECK(status.is_cuda() && status.scalar_type() == at::kInt, "status must be a CUDA int32 tensor");
  a.status = reinterpret_cast<uint32_t*>(status.data_ptr<int32_t>());
  const uint64_t* cc = reinterpret_cast<const uint64_t*>(consts_cpu.data_ptr<int64_t>());
  for (int l = 0; l < L; ++l) {
    a.q[l] = cc[l * 8];
    a.ratio_hi[l] = cc[l * 8 + 2];
  }
  a.numel = numel;
  a.timeout_ns = (uint64_t)timeout_ms * 1000000ull;
  a.rank = (int)rank;
  a.world = (int)world;
  a.L = (int)L;
  a.logn = (int)logn;
  a.no_owner = (int)no_owner;
  if (stats.has_value()) {
    TORCH_CHECK(stats->is_cuda() && stats->scalar_type() == at::kInt, "stats must be a CUDA int32 tensor");
    a.stats = reinterpret_cast<uint32_t*>(stats->data_ptr<int32_t>());
  }
  hefl::comm::allreduce_modq(a, (int)algo, (int)blocks, (int)threads,
                             at::cuda::getCurrentCUDAStream().stream());
}

// data (+)= sum_j sign_j * PRG(seed_j) mod q, in place (pairwise masks that cancel in the all-reduce).
void pairwise_mask_(Tensor data, at::IntArrayRef seeds, at::IntArrayRef signs, int64_t round, int64_t L,
                    int64_t logn, const Tensor& consts_cpu) {
  TORCH_CHECK(seeds.size() == signs.size() && seeds.size() <= (size_t)hefl::comm::kMaxWorld, "bad peer list");
  TORCH_CHECK(data.numel() % 2 == 0, "numel must be even");
  TORCH_CHECK(consts_cpu.is_cpu() && consts_cpu.size(0) >= L && L <= hefl::comm::kMaxLimbs, "bad consts");
  hefl::comm::MaskArgs m;
  std::memset(&m, 0, sizeof(m));
  m.npeers = (int)seeds.size();
  for (int j = 0; j < m.npeers; ++j) {
    m.seed[j] = (uint64_t)seeds[j];
    m.sign[j] = signs[j] >= 0 ? 1 : -1;
  }
  m.round = (uint32_t)round;
  const uint64_t* cc = reinterpret_cast<const uint64_t*>(consts_cpu.data_ptr<int64_t>());
  for (int l = 0; l < L; ++l) {
    m.q[l] = cc[l * 8];
    m.ratio_lo[l] = cc[l * 8 + 1];
    m.ratio_hi[l] = cc[l * 8 + 2];
  }
  if (data.is_cuda()) {
    hefl::comm::pairwise_mask(u64(data), data.numel(), (int)L, (int)logn, m, at::cuda::getCurrentCUDAStream().stream());
  } else {
    hefl::comm::pairwise_mask_host(u64(data), data.numel(), (int)L, (int)logn, m);
  }
}

void local_sum_modq(at::TensorList srcs, Tensor out, int64_t L, int64_t logn, const Tensor& consts) {
  const int K = (int)srcs.size();
  TORCH_CHECK(K >= 1, "need at least one source");
  const int64_t numel = out.numel();
  TORCH_CHECK(numel % 2 == 0, "numel must be even");
  for (const auto& s : srcs) {
    TORCH_CHECK(s.numel() == numel && s.device() == out.device(), "source shape/device mismatch");
  }
  if (out.is_cuda()) {
    std::vector<int64_t> ptrs(K);
    for (int k = 0; k < K; ++k) ptrs[k] = (int64_t)u64(srcs[k]);
    Tensor dptr = at::tensor(ptrs, at::kLong).to(out.device());
    hefl::comm::local_sum_modq(reinterpret_cast<const uint64_t* const*>(dptr.data_ptr<int64_t>()), K,
                               u64(out), numel, (int)logn, (int)L, u64(consts),
                               at::cuda::getCurrentCUDAStream().stream());
    return;
  }
  const uint64_t* cc = u64(consts);
  uint64_t* o = u64(out);
  const int64_t n = 1ll << logn;
  std::vector<const uint64_t*> sp(K);
  for (int k = 0; k < K; ++k) sp[k] = u64(srcs[k]);
#pragma omp parallel for schedule(static)
  for (int64_t e = 0; e < numel; ++e) {
    const int l = (int)((e / n) % L);
    const hefl::Modulus m{cc[l * 8], cc[l * 8 + 1], cc[l * 8 + 2]};
    uint64_t acc = 0;
    for (int k = 0; k < K; ++k) {
      acc += sp[k][e];
      if (k % 7 == 6) acc = hefl::barrett_reduce_64(acc, m);   // as the kernel: < q plus 7 addends < 2^64
    }
    o[e] = hefl::barrett_reduce_64(acc, m);
  }
}

// ---- CUDA IPC fallback -------------------------------------------------------------------

Tensor ipc_alloc(int64_t nbytes, int64_t device) {
  c10::cuda::CUDAGuard g((c10::DeviceIndex)device);
  void* p = nullptr;
  TORCH_CHECK(cudaMalloc(&p, (size_t)nbytes) == cudaSuccess, "cudaMalloc failed");
  cudaMemset(p, 0, (size_t)nbytes);
  auto opts = at::TensorOptions().dtype(at::kByte).device(at::kCUDA, (c10::DeviceIndex)device);
  return at::from_blob(p, {nbytes}, [](void* q) { cudaFree(q); }, opts);
}

Tensor ipc_get_handle(const Tensor& t) {
  cudaIpcMemHandle_t h;
  TORCH_CHECK(cudaIpcGetMemHandle(&h, t.data_ptr()) == cudaSuccess, "cudaIpcGetMemHandle failed");
  Tensor out = at::empty({(int64_t)sizeof(h)}, at::kByte);
  std::memcpy(out.data_ptr(), &h, sizeof(h));
  return out;
}

int64_t ipc_open_handle(const Tensor& handle, int64_t device) {
  c10::cuda::CUDAGuard g((c10::DeviceIndex)device);
  cudaIpcMemHandle_t h;
  TORCH_CHECK(handle.is_cpu() && handle.numel() == (int64_t)sizeof(h), "bad IPC handle");
  std::memcpy(&h, handle.data_ptr(), sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  TORCH_CHECK(e == cudaSuccess, "cudaIpcOpenMemHandle failed: ", cudaGetErrorString(e));
  return (int64_t)p;
}

void ipc_close_handle(int64_t ptr) { cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr)); }

int64_t enable_peer_access(int64_t device, int64_t peer) {
  c10::cuda::CUDAGuard g((c10::DeviceIndex)device);
  int can = 0;
  cudaDeviceCanAccessPeer(&can, (int)device, (int)peer);
  if (!can) return 0;
  cudaError_t e = cudaDeviceEnablePeerAccess((int)peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return 1; }
  return e == cudaSuccess ? 1 : 0;
}

Tensor tensor_from_ptr(int64_t ptr, int64_t numel, int64_t device) {
  auto opts = at::TensorOptions().dtype(at::kLong).device(at::kCUDA, (c10::DeviceIndex)device);
  return at::from_blob(reinterpret_cast<void*>(ptr), {numel}, [](void*) {}, opts);
}

}  // namespace

TORCH_LIBRARY_FRAGMENT(hefl, m) {
  m.def("allreduce_modq(int[] buf_ptrs, int[] sig_ptrs, int mc_ptr, Tensor? out, Tensor status, Tensor consts_cpu, int numel, int L, int logn, int rank, int world, int algo, int blocks, int threads, int timeout_ms, int no_owner=-1, Tensor? stats=None) -> ()", &allreduce_modq);
  m.def("pairwise_mask_(Tensor(a!) data, int[] seeds, int[] signs, int round, int L, int logn, Tensor consts_cpu) -> ()", &pairwise_mask_);
  m.def("local_sum_modq(Tensor[] srcs, Tensor(a!) out, int L, int logn, Tensor consts) -> ()", &local_sum_modq);
  m.def("ipc_alloc(int nbytes, int device) -> Tensor", &ipc_alloc);
  m.def("ipc_get_handle(Tensor t) -> Tensor", &ipc_get_handle);
  m.def("ipc_open_handle(Tensor handle, int device) -> int", &ipc_open_handle);
  m.def("ipc_close_handle(int ptr) -> ()", &ipc_close_handle);
  m.def("enable_peer_access(int device, int peer) -> int", &enable_peer_access);
  m.def("tensor_from_ptr(int ptr, int numel, int device) -> Tensor", &tensor_from_ptr);
}
