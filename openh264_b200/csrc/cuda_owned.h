// cuda_owned.h — move-only owners of CUDA resources: a device buffer, a pinned host buffer, an event and a stream.  An owner
// releases its resource when it is destroyed or assigned another one.  Each allocation returns the CUDA status and changes
// nothing on failure.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace b2h264 {

template <class H, cudaError_t (*Release)(H)>
class CudaOwned {
 public:
  CudaOwned() = default;
  CudaOwned(CudaOwned&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  CudaOwned& operator=(CudaOwned&& o) noexcept {
    if (this != &o) { release(); h_ = o.h_; o.h_ = nullptr; }
    return *this;
  }
  ~CudaOwned() { release(); }

 protected:
  // h replaces the held handle when err is success.  Callers acquire h in a statement of its own: were the acquiring call an
  // argument of adopt, h could be read before that call writes it (argument evaluation order is unspecified)
  cudaError_t adopt(cudaError_t err, H h) {
    if (err == cudaSuccess) { release(); h_ = h; }
    return err;
  }
  void release() { if (h_) Release(h_); h_ = nullptr; }
  H h_ = nullptr;
};

template <class T>
struct DeviceBuf : CudaOwned<void*, cudaFree> {
  cudaError_t alloc(size_t bytes) {
    void* p = nullptr;
    const cudaError_t err = cudaMalloc(&p, bytes);
    return adopt(err, p);
  }
  T* get() const { return static_cast<T*>(h_); }
};

template <class T>
struct HostBuf : CudaOwned<void*, cudaFreeHost> {
  cudaError_t alloc(size_t bytes, unsigned flags = cudaHostAllocDefault) {
    void* p = nullptr;
    const cudaError_t err = cudaHostAlloc(&p, bytes, flags);
    return adopt(err, p);
  }
  T* get() const { return static_cast<T*>(h_); }
};

struct Event : CudaOwned<cudaEvent_t, cudaEventDestroy> {
  cudaError_t create(unsigned flags = cudaEventDefault) {
    cudaEvent_t ev = nullptr;
    const cudaError_t err = cudaEventCreateWithFlags(&ev, flags);
    return adopt(err, ev);
  }
  cudaEvent_t get() const { return h_; }
};

struct Stream : CudaOwned<cudaStream_t, cudaStreamDestroy> {
  cudaError_t create(unsigned flags, int priority = 0) {
    cudaStream_t s = nullptr;
    const cudaError_t err = cudaStreamCreateWithPriority(&s, flags, priority);
    return adopt(err, s);
  }
  cudaStream_t get() const { return h_; }
};

}  // namespace b2h264
