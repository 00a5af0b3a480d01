// Owners of CUDA memory, events and streams: std::unique_ptr with the matching release call as its deleter.  Like
// any teardown, the deleters ignore errors.
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <type_traits>

namespace eb {

struct DeviceFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct HostFree {
  void operator()(void* p) const { cudaFreeHost(p); }
};
struct EventDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct StreamDestroy {
  void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};

template <class T>
using DevPtr = std::unique_ptr<T, DeviceFree>;  // cudaMalloc
template <class T>
using HostPtr = std::unique_ptr<T, HostFree>;  // cudaMallocHost (pinned)
using EventPtr = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;
using StreamPtr = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;

// allocate / create into an owner: on success p owns the new object (and releases what it held), on failure p is
// left as it was
template <class T>
cudaError_t dev_alloc(DevPtr<T>& p, size_t bytes) {
  void* raw = nullptr;
  const cudaError_t e = cudaMalloc(&raw, bytes);
  if (e == cudaSuccess) p.reset(static_cast<T*>(raw));
  return e;
}

template <class T>
cudaError_t host_alloc(HostPtr<T>& p, size_t bytes) {
  void* raw = nullptr;
  const cudaError_t e = cudaMallocHost(&raw, bytes);
  if (e == cudaSuccess) p.reset(static_cast<T*>(raw));
  return e;
}

inline cudaError_t event_create(EventPtr& p, unsigned flags = cudaEventDefault) {
  cudaEvent_t ev = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&ev, flags);
  if (e == cudaSuccess) p.reset(ev);
  return e;
}

inline cudaError_t stream_create(StreamPtr& p, unsigned flags) {
  cudaStream_t st = nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&st, flags);
  if (e == cudaSuccess) p.reset(st);
  return e;
}

}  // namespace eb
