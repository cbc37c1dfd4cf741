// cuda_owned.cuh -- owners of the CUDA memory, streams and events behind the C ABI, and the one path a failed CUDA
// call takes.  Every allocation, free, create and destroy call of the library is in this file: a buffer or handle is
// a member of the object that owns it and goes away with that object.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdio>
#include <utility>

#include "../../include/b200match.h"

// Returns from the enclosing function through b2m::fail: B2M_ENOMEM when the call ran out of memory, B2M_ECUDA
// otherwise, with the message "[<file>:<line>] CUDA error: <error string> (<expr>)".
#define B2M_CUDA_TRY(ctx, expr)                                                                               \
  do {                                                                                                        \
    const cudaError_t b2m_e_ = (expr);                                                                        \
    if (b2m_e_ != cudaSuccess) {                                                                              \
      char b2m_msg_[512];                                                                                     \
      snprintf(b2m_msg_, sizeof(b2m_msg_), "[%s:%d] CUDA error: %s (%s)", __FILE__, __LINE__,                 \
               cudaGetErrorString(b2m_e_), #expr);                                                            \
      return ::b2m::fail((ctx), b2m_e_ == cudaErrorMemoryAllocation ? B2M_ENOMEM : B2M_ECUDA, b2m_msg_);      \
    }                                                                                                         \
  } while (0)

namespace b2m {

// An array of T in device memory (Pinned = false) or in page-locked host memory (Pinned = true), freed with its owner.
template <class T, bool Pinned>
class CudaArray {
 public:
  CudaArray() = default;
  CudaArray(CudaArray&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  CudaArray& operator=(CudaArray&& o) noexcept {
    if (this != &o) {
      reset();
      p_ = std::exchange(o.p_, nullptr);
      n_ = std::exchange(o.n_, 0);
    }
    return *this;
  }
  ~CudaArray() { reset(); }

  // Room for n elements.  A block that holds n already is kept; otherwise the old block is freed first (the peak
  // stays one block) and max(n, 1) elements are allocated, so an empty array always gets a block.  On failure the
  // array is left empty.
  cudaError_t ensure(size_t n) {
    if (p_ && n <= n_) return cudaSuccess;
    reset();
    const size_t m = n > 0 ? n : 1;
    void* p = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&p, sizeof(T) * m) : cudaMalloc(&p, sizeof(T) * m);
    if (e != cudaSuccess) return e;
    p_ = static_cast<T*>(p);
    n_ = m;
    return cudaSuccess;
  }
  void reset() {
    if (p_) {
      if (Pinned) cudaFreeHost(p_);
      else cudaFree(p_);
    }
    p_ = nullptr;
    n_ = 0;
  }
  size_t capacity() const { return n_; }
  operator T*() const { return p_; }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};
template <class T>
using DeviceArray = CudaArray<T, false>;
template <class T>
using PinnedArray = CudaArray<T, true>;

inline cudaError_t create_handle(cudaStream_t* h, unsigned flags) { return cudaStreamCreateWithFlags(h, flags); }
inline cudaError_t create_handle(cudaEvent_t* h, unsigned flags) { return cudaEventCreateWithFlags(h, flags); }
inline void destroy_handle(cudaStream_t h) { cudaStreamDestroy(h); }
inline void destroy_handle(cudaEvent_t h) { cudaEventDestroy(h); }

// A cudaStream_t or cudaEvent_t, destroyed with its owner.
template <class H>
class CudaHandle {
 public:
  CudaHandle() = default;
  CudaHandle(CudaHandle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  CudaHandle& operator=(CudaHandle&& o) noexcept {
    if (this != &o) {
      reset();
      h_ = std::exchange(o.h_, nullptr);
    }
    return *this;
  }
  ~CudaHandle() { reset(); }

  cudaError_t create(unsigned flags) {
    reset();
    return create_handle(&h_, flags);
  }
  void reset() {
    if (h_) destroy_handle(h_);
    h_ = nullptr;
  }
  operator H() const { return h_; }

 private:
  H h_ = nullptr;
};
using Stream = CudaHandle<cudaStream_t>;
using Event = CudaHandle<cudaEvent_t>;

// Builds a group of owners all or nothing: `g` is emptied first (its old blocks are freed before any new one is
// allocated), `alloc(g)` fills it and returns a B2M code, and on failure `g` is emptied again.  So a group is either
// complete or empty, and any one of its members tells which.
template <class Group, class Alloc>
int alloc_group(Group& g, Alloc&& alloc) {
  g = Group{};
  const int rc = alloc(g);
  if (rc != B2M_OK) g = Group{};
  return rc;
}

}  // namespace b2m
