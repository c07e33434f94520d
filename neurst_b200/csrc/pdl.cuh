// Programmatic dependent launch (PDL): every kernel of the library is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization and starts with griddepcontrol.wait, so the launch latency and
// the prologue (barrier init, tensor-map prefetch, smem tables) of kernel N+1 overlap the tail of
// kernel N — the step is ~600 short dependent kernels, i.e. launch-latency sensitive.  Correctness rule: no global memory
// access before pdl_wait().  In a stream capture these launches become programmatic graph edges.
#pragma once
#include <cuda_runtime.h>
#include <utility>

namespace b200st {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

cudaError_t& pdl_launch_error();   // thread-local: first failed launch since the last check
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
  if (e != cudaSuccess && pdl_launch_error() == cudaSuccess) pdl_launch_error() = e;
}

}  // namespace b200st
