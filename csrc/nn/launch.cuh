// Programmatic dependent launch (PDL) for the training-step kernels. Every kernel of the step calls
// pdl_prologue() after its private set-up (barrier init, tensor-map prefetch) and
// before it touches global memory; launches go through launch_pdl(), which sets
// cudaLaunchAttributeProgrammaticStreamSerialization so the next kernel's CTAs become resident and run
// their set-up while the previous kernel drains. griddepcontrol.wait returns only when the previous
// grid has completed and its memory is visible, so data dependencies are unchanged (and transitive,
// because every kernel in the chain waits before it exits). Captured into the CUDA graph as
// programmatic edges.
#pragma once
#include <cuda_runtime.h>

namespace hefl {
namespace nn {

__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
  pdl_trigger();
  pdl_wait();
}
// Kernels that WRITE the parameters (Adam, weight re-layout) call only pdl_wait(): they never
// trigger their dependents early, so no later kernel can be resident before the new weights are complete.
// That is what allows the dense-head kernels to stage their weight tiles BEFORE griddepcontrol.wait (while
// the previous kernel is still running) — activations are only touched after the wait.

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace nn
}  // namespace hefl
