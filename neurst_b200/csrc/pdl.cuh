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

bool pdl_enabled();
// Counts one launched kernel (b200st_launch_count).
void count_launch();
// Clears CUDA's last error, sets the library's to "kernel launch failed: ..." and returns 1.
int launch_failed(cudaError_t e);

// Every kernel launch of the library goes through launch_ex: it counts the launch and returns 0, or returns 1 with the
// error set.  pdl: add the programmatic-serialization attribute.
template <typename... KArgs, typename... Args>
inline int launch_ex(bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
  if (e != cudaSuccess) return launch_failed(e);
  count_launch();
  return 0;
}

// A kernel that waits on its predecessor with pdl_wait (all but the few below); B200ST_NO_PDL drops the attribute.
template <typename... KArgs, typename... Args>
inline int launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  return launch_ex(pdl_enabled(), kern, grid, block, smem, stream, std::forward<Args>(args)...);
}
// A kernel without griddepcontrol.wait (the searches' init and extract kernels): it must not start under its predecessor.
template <typename... KArgs, typename... Args>
inline int launch_serial(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  return launch_ex(false, kern, grid, block, smem, stream, std::forward<Args>(args)...);
}

}  // namespace b200st
