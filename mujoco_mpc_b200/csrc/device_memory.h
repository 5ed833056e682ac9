// device_memory.h - move-only owners of the engine's device arrays (cudaMalloc / cudaFree) and pinned host arrays
// (cudaMallocHost / cudaFreeHost).  An owner frees its array when it is destroyed or replaced, and converts to the raw
// pointer wherever one is expected (kernel arguments, copies, pointer arithmetic).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>

namespace mjpc_mem {

template <class T, bool Pinned>
class CudaArray {
 public:
  CudaArray() = default;
  CudaArray(const CudaArray&) = delete;
  CudaArray& operator=(const CudaArray&) = delete;
  CudaArray(CudaArray&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
  CudaArray& operator=(CudaArray&& o) noexcept {
    if (this != &o) { reset(); p_ = o.p_; o.p_ = nullptr; }
    return *this;
  }
  ~CudaArray() { reset(); }

  // A new array of n elements in this empty owner.  n = 0 still allocates one element: kernels receive non-null
  // pointers for empty arrays.  On failure the owner stays empty and the error is cleared from cudaGetLastError.  An
  // owner that holds an array is refused (cudaErrorInvalidValue): a launch in flight may still read it, so a live
  // array is only replaced by allocating into a new owner, synchronising the stream, and moving that owner in.
  cudaError_t alloc(size_t n) {
    if (p_) return cudaErrorInvalidValue;
    void* p = nullptr;
    const size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
    const cudaError_t e = Pinned ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    p_ = static_cast<T*>(p);
    return cudaSuccess;
  }
  void reset() {
    if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
    p_ = nullptr;
  }
  T* get() const { return p_; }
  operator T*() const { return p_; }

 private:
  T* p_ = nullptr;
};

template <class T>
using DeviceArray = CudaArray<T, false>;
template <class T>
using PinnedArray = CudaArray<T, true>;

}  // namespace mjpc_mem
