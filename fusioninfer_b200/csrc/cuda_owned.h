// cuda_owned.h — owners of the CUDA resources a handle holds: std::unique_ptr with the matching release call.
// Use sites read .get(); the kernel-facing views (IndexView, DevLru, PeerXchg, ...) stay plain structs filled from
// the owners.  The helpers leave the owner null when the CUDA call fails and return its error.
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <type_traits>

namespace fi {

struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  template <typename T>
  void operator()(T* p) const { cudaFreeHost(const_cast<std::remove_cv_t<T>*>(p)); }
};
struct CudaEventDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct CudaStreamDestroy {
  void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};

template <typename T>
using DevPtr = std::unique_ptr<T, CudaFree>;  // device memory (cudaMalloc)
template <typename T>
using PinnedPtr = std::unique_ptr<T, CudaFreeHost>;  // pinned host memory (cudaHostAlloc)
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, CudaEventDestroy>;
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, CudaStreamDestroy>;

// n elements of device memory, or of pinned host memory (flags: cudaHostAlloc's)
template <typename T>
cudaError_t cuda_alloc(DevPtr<T>& p, size_t n) {
  void* raw = nullptr;
  const cudaError_t e = cudaMalloc(&raw, n * sizeof(T));
  p.reset(e == cudaSuccess ? static_cast<T*>(raw) : nullptr);
  return e;
}
template <typename T>
cudaError_t cuda_alloc(PinnedPtr<T>& p, size_t n, unsigned flags = cudaHostAllocDefault) {
  void* raw = nullptr;
  const cudaError_t e = cudaHostAlloc(&raw, n * sizeof(T), flags);
  p.reset(e == cudaSuccess ? static_cast<T*>(raw) : nullptr);
  return e;
}

// an event (flags: cudaEventCreateWithFlags'), or a non-blocking stream
inline cudaError_t cuda_create(Event& ev, unsigned flags = cudaEventDisableTiming) {
  cudaEvent_t raw = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&raw, flags);
  ev.reset(e == cudaSuccess ? raw : nullptr);
  return e;
}
inline cudaError_t cuda_create(Stream& s) {
  cudaStream_t raw = nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&raw, cudaStreamNonBlocking);
  s.reset(e == cudaSuccess ? raw : nullptr);
  return e;
}

}  // namespace fi
