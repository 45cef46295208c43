// Programmatic dependent launch (PDL): every kernel of the step is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, fires griddepcontrol.launch_dependents at its
// top and executes griddepcontrol.wait before its first access to global memory.  The next
// kernel's launch latency and prologue (barrier init, descriptor fetch) then overlap the
// tail of the current one; correctness is unchanged because `wait` returns only after the
// prerequisite grid has completed and its writes are visible.  NS2VC_PDL=0 disables it.
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>
#include <utility>

namespace ns2vc {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Diagnostics: [min entry, max exit] %globaltimer stamps of a whole grid (slot pre-set to {~0, 0}).
__device__ __forceinline__ unsigned long long gtime_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void span_begin(unsigned long long* s) { if (s && threadIdx.x == 0 && threadIdx.y == 0) atomicMin(s, gtime_ns()); }
__device__ __forceinline__ void span_end(unsigned long long* s) { if (s && threadIdx.x == 0 && threadIdx.y == 0) atomicMax(s + 1, gtime_ns()); }

inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("NS2VC_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
  return v == 1;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kc(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, dim3 cluster, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (pdl_enabled()) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster.x * cluster.y * cluster.z > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster.x; at[n].val.clusterDim.y = cluster.y; at[n].val.clusterDim.z = cluster.z;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  return launch_kc(kernel, grid, block, smem, st, dim3(1, 1, 1), std::forward<Args>(args)...);
}

}  // namespace ns2vc
