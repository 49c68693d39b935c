// Host-side helpers of the C ABI's CUDA units: an owned device buffer and the check of a CUDA call.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <string>

// Returns fail(TB200_ERR_CUDA, "<call>: <CUDA error>") from the enclosing function when the call fails; `fail` is the
// error channel of the unit that uses it.
#define CK(call)                                                                                      \
  do {                                                                                                \
    cudaError_t e_ = (call);                                                                          \
    if (e_ != cudaSuccess) return fail(TB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

namespace tb200 {

// A zero-filled device array of n elements of T, freed with its owner.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    std::swap(p, o.p);
    std::swap(n, o.n);
    return *this;
  }
  ~DevBuf() { release(); }
  // (Re)allocates count zeroed elements (at least one is allocated), freeing what the buffer held before.
  cudaError_t alloc(size_t count) {
    release();
    n = count;
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) e = cudaMemset(p, 0, bytes);
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
};

}  // namespace tb200
