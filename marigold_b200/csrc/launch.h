// Kernel launch helper: every kernel of the library is launched with programmatic dependent launch
// (PDL) allowed, so the next kernel's launch latency and prologue (barrier init,
// tensor-map prefetch) overlap the tail of the previous one. Every kernel therefore executes
// pdl_launch_dependents() at its top and pdl_wait() before its first access to global memory that a
// predecessor may have written (common.cuh). Under stream capture the attribute becomes a programmatic
// dependency edge of the CUDA graph.
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>
#include <utility>

namespace mgb {

inline bool pdl_enabled() {
  static const bool on = getenv("MGB_NO_PDL") == nullptr;
  return on;
}

// Launches inside a PlainLaunchScope do NOT get the PDL attribute: the kernel starts only after every earlier kernel
// of the stream has completed. Needed where a kernel reads, BEFORE its griddepcontrol.wait, memory that an earlier
// kernel of the same stream writes: gemm_tc_kernel prefetches its first B ("weight") tiles ahead of the wait, which
// is only safe when B really is a static weight — not for the VAE attention GEMMs whose B operand is K / V^T.
inline int& plain_launch_depth() {
  static thread_local int depth = 0;
  return depth;
}
struct PlainLaunchScope {
  PlainLaunchScope() { ++plain_launch_depth(); }
  ~PlainLaunchScope() { --plain_launch_depth(); }
  PlainLaunchScope(const PlainLaunchScope&) = delete;
  PlainLaunchScope& operator=(const PlainLaunchScope&) = delete;
};

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                            Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  // not on the legacy default stream, not inside a PlainLaunchScope
  cfg.numAttrs = (pdl_enabled() && stream != nullptr && plain_launch_depth() == 0) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
}

}  // namespace mgb
