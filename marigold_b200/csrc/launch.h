// The one path every kernel of the library is launched through: launch_pdl / launch_plain issue the launch, turn a
// failure into MGB_ERR_CUDA with the kernel's name in the error text, and count the launch (mgb_launch_count).
//
// Programmatic dependent launch (PDL) lets the next kernel's launch latency and prologue (barrier init, tensor-map
// prefetch) overlap the tail of the previous one. A kernel launched with it executes pdl_launch_dependents() at its top
// and pdl_wait() before its first access to global memory that a predecessor may have written (common.cuh). Under
// stream capture the attribute becomes a programmatic dependency edge of the CUDA graph.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>
#include <utility>

#include "device.h"
#include "kernels.h"

namespace mgb {

inline std::atomic<long long> g_launches{0};
inline void count_launch(long long n) { g_launches += n; }
inline long long launch_count() { return g_launches.load(); }

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
inline int launch_kernel(const char* name, bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                         cudaStream_t stream, Args&&... args) {
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
  cfg.numAttrs = (pdl && pdl_enabled() && stream != nullptr && plain_launch_depth() == 0) ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
  const cudaError_t last = cudaGetLastError();   // also clears a failed launch's error
  if (e == cudaSuccess) e = last;
  if (e != cudaSuccess) {
    set_error("%s launch: %s", name, cudaGetErrorString(e));
    return MGB_ERR_CUDA;
  }
  count_launch(1);
  return MGB_OK;
}

// launch_pdl only for kernels that call pdl_wait(): for any other kernel the attribute is a race. launch_plain sets none.
template <typename... KArgs, typename... Args>
inline int launch_pdl(const char* name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                      cudaStream_t stream, Args&&... args) {
  return launch_kernel(name, true, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline int launch_plain(const char* name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                        cudaStream_t stream, Args&&... args) {
  return launch_kernel(name, false, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}

// Raises Kernel's dynamic shared-memory limit to `bytes` on the first call that succeeds; later calls do nothing.
template <auto Kernel>
inline int raise_smem_limit_once(const char* name, int bytes) {
  static bool done = false;
  if (!done) {
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
      set_error("%s smem limit: %s", name, cudaGetErrorString(e));
      return MGB_ERR_CUDA;
    }
    done = true;
  }
  return MGB_OK;
}

// Blocks for a grid-stride loop over n items: enough to cover n, at most 16 per SM, at least 1.
inline int grid_for(size_t n, int threads) {
  const size_t b = (n + threads - 1) / threads;
  const size_t cap = size_t(kNumSMs) * 16;
  return int(b < cap ? (b ? b : 1) : cap);
}

}  // namespace mgb
