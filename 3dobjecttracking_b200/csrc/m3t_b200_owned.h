// m3t_b200_owned.h — owners of the host library's CUDA resources: device buffers, pinned host buffers, streams, events.
// The only place in the library that creates or releases one. Host code only.
#ifndef M3T_B200_OWNED_H_
#define M3T_B200_OWNED_H_

#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <utility>

namespace m3tb {

// Resources held across all contexts, and the fault injection of m3tb_debug_resources (> 0: the n-th creation from
// now on fails). Process-wide, so that contexts on different threads count correctly.
inline std::atomic<long long> g_live_resources{0};
inline std::atomic<long long> g_fail_after{0};

enum class ResourceKind { kDevice, kPinned, kStream, kEvent };

// Creates one resource; on failure *out is untouched.
inline cudaError_t CreateResource(ResourceKind kind, size_t bytes, void** out) {
  for (long long n = g_fail_after.load(); n > 0;)
    if (g_fail_after.compare_exchange_weak(n, n - 1)) {
      if (n == 1) return cudaErrorMemoryAllocation;
      break;
    }
  void* p = nullptr;
  cudaError_t e = cudaSuccess;
  switch (kind) {
    case ResourceKind::kDevice: e = cudaMalloc(&p, bytes); break;
    case ResourceKind::kPinned: e = cudaMallocHost(&p, bytes); break;
    case ResourceKind::kStream:
      e = cudaStreamCreateWithFlags(reinterpret_cast<cudaStream_t*>(&p), cudaStreamNonBlocking);
      break;
    case ResourceKind::kEvent:
      e = cudaEventCreateWithFlags(reinterpret_cast<cudaEvent_t*>(&p), cudaEventDisableTiming);
      break;
  }
  if (e != cudaSuccess) return e;
  if (p) ++g_live_resources;  // a zero-byte allocation holds nothing
  *out = p;
  return cudaSuccess;
}

// Synchronous release: the device-wide synchronisation of cudaFree is relied upon where a launch in flight may still
// read the object being replaced.
inline void ReleaseResource(ResourceKind kind, void* p) {
  if (!p) return;
  switch (kind) {
    case ResourceKind::kDevice: cudaFree(p); break;
    case ResourceKind::kPinned: cudaFreeHost(p); break;
    case ResourceKind::kStream: cudaStreamDestroy(static_cast<cudaStream_t>(p)); break;
    case ResourceKind::kEvent: cudaEventDestroy(static_cast<cudaEvent_t>(p)); break;
  }
  --g_live_resources;
}

// Move-only owner of one resource of `Kind` holding `n` elements of T (streams and events: T is the handle's pointee).
// It converts to the raw pointer / handle, which is how the kernel argument structs and device records view it.
template <typename T, ResourceKind Kind>
class Owned {
 public:
  Owned() = default;
  Owned(Owned&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  Owned& operator=(Owned&& o) noexcept {
    Owned tmp(std::move(o));
    std::swap(p_, tmp.p_);
    std::swap(n_, tmp.n_);
    return *this;
  }
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() { ReleaseResource(Kind, p_); }

  // Replaces the held object with a new one of n elements, releasing the old one only after the new one exists.
  // On failure the owner keeps what it held.
  cudaError_t create(size_t n = 1) {
    size_t bytes = 0;
    if constexpr (Kind == ResourceKind::kDevice || Kind == ResourceKind::kPinned) bytes = sizeof(T) * n;
    void* p = nullptr;
    const cudaError_t e = CreateResource(Kind, bytes, &p);
    if (e != cudaSuccess) return e;
    ReleaseResource(Kind, p_);
    p_ = p;
    n_ = n;
    return cudaSuccess;
  }

  T* get() const { return static_cast<T*>(p_); }
  operator T*() const { return get(); }
  size_t size() const { return n_; }

 private:
  void* p_ = nullptr;
  size_t n_ = 0;
};

template <typename T>
using DeviceBuffer = Owned<T, ResourceKind::kDevice>;
template <typename T>
using PinnedBuffer = Owned<T, ResourceKind::kPinned>;
using Stream = Owned<CUstream_st, ResourceKind::kStream>;
using Event = Owned<CUevent_st, ResourceKind::kEvent>;

}  // namespace m3tb

#endif  // M3T_B200_OWNED_H_
