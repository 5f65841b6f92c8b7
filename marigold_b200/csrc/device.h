// Owners of the library's device memory, pinned host memory, CUDA graph and capture stream. Each releases what it
// holds when it is destroyed, so an early return frees its temporaries and a handle is torn down by its destructor.
#pragma once
#include <atomic>
#include <memory>
#include <utility>

#include "kernels.h"

// Returns MGB_ERR_CUDA, with the failing call in the error text, when a CUDA runtime call fails.
#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      mgb::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));    \
      return MGB_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

// Returns the status of `expr` when it is not MGB_OK.
#define TRY(expr)                  \
  do {                             \
    int _rc = (expr);              \
    if (_rc != MGB_OK) return _rc; \
  } while (0)

namespace mgb {

// Bytes that every DevBuf and PinnedBuf together hold now (mgb_debug_live_device_bytes).
inline std::atomic<int64_t> g_live_bytes{0};

// One allocation, move-only. It converts to T* so that code written for the raw pointer it replaces reads it unchanged.
template <class T, cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
class Buf {
 public:
  Buf() = default;
  Buf(Buf&& o) noexcept { swap(o); }
  Buf& operator=(Buf&& o) noexcept { swap(o); return *this; }   // o frees what this held
  ~Buf() { reset(); }

  T* get() const { return static_cast<T*>(p_); }
  operator T*() const { return get(); }
  size_t bytes() const { return n_; }

  void reset() {
    if (p_) Free(p_);
    g_live_bytes -= int64_t(n_);
    p_ = nullptr;
    n_ = 0;
  }
  // At least `need` bytes. A smaller buffer is freed before the new one is allocated; if that allocation fails the
  // buffer is left empty and MGB_ERR_NOMEM is returned.
  int grow(size_t need) {
    if (need <= n_) return MGB_OK;
    reset();
    if (Alloc(&p_, need) != cudaSuccess) {
      p_ = nullptr;
      set_error("allocating %zu bytes failed", need);
      return MGB_ERR_NOMEM;
    }
    n_ = need;
    g_live_bytes += int64_t(need);
    return MGB_OK;
  }

 private:
  void swap(Buf& o) { std::swap(p_, o.p_); std::swap(n_, o.n_); }
  void* p_ = nullptr;
  size_t n_ = 0;
};
template <class T> using DevBuf = Buf<T, cudaMalloc, cudaFree>;
template <class T> using PinnedBuf = Buf<T, cudaMallocHost, cudaFreeHost>;

struct GraphExecDestroy { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
using GraphExec = std::unique_ptr<CUgraphExec_st, GraphExecDestroy>;   // cudaGraphExec_t is CUgraphExec_st*
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;            // cudaStream_t is CUstream_st*

}  // namespace mgb
