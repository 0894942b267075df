// Owners of the CUDA resources the engine and the vocabulary-tree database hold across calls, and the status macro both use.
// Each owner releases what it holds in its destructor, so a half-built object or a failed call leaks nothing.
// Stream-ordered memory (cudaMallocAsync / cudaFreeAsync) is not owned here: its lifetime follows stream order, not scope.
#pragma once
#include "../../include/b200match.h"

#include <cuda_runtime.h>

#include <string>
#include <utility>

namespace b200m { int set_error(int code, const std::string& msg); }   // engine.cu: thread-local message behind b200m_last_error()

#define CK(call)                                                                                                      \
  do {                                                                                                                \
    cudaError_t e_ = (call);                                                                                          \
    if (e_ != cudaSuccess) return b200m::set_error(B200M_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

namespace b200m {

// A grow-only block of device (cudaMalloc) or pinned host (cudaMallocHost) memory, used as T* (as<U>() for another element type).
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Release)(void*), class T = void>
class Buffer {
 public:
  Buffer() = default;
  Buffer(Buffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)) {}
  Buffer& operator=(Buffer&& o) noexcept { std::swap(p_, o.p_); std::swap(cap_, o.cap_); return *this; }
  ~Buffer() { if (p_) Release(p_); }

  // At least `bytes` bytes; the contents are not kept.  A larger request frees the old block first (cudaFree synchronises the
  // device, so nothing enqueued still reads it) and allocates bytes + bytes / 4.  On failure the buffer is empty.
  int reserve(size_t bytes) {
    if (bytes <= cap_) return B200M_OK;
    void* old = std::exchange(p_, nullptr);
    cap_ = 0;
    if (old) CK(Release(old));
    void* p = nullptr;
    CK(Alloc(&p, bytes + bytes / 4));
    p_ = p; cap_ = bytes + bytes / 4;
    return B200M_OK;
  }
  size_t capacity() const { return cap_; }
  operator T*() const { return static_cast<T*>(p_); }
  template <class U> U* as() const { return static_cast<U*>(p_); }

 private:
  void* p_ = nullptr;
  size_t cap_ = 0;
};
template <class T = void> using DeviceBuffer = Buffer<cudaMalloc, cudaFree, T>;
template <class T = void> using PinnedBuffer = Buffer<cudaMallocHost, cudaFreeHost, T>;

class Event {
 public:
  Event() = default;
  Event(Event&& o) noexcept : e_(std::exchange(o.e_, nullptr)) {}
  Event& operator=(Event&& o) noexcept { std::swap(e_, o.e_); return *this; }
  ~Event() { if (e_) cudaEventDestroy(e_); }
  int create(unsigned flags = cudaEventDefault) {      // no-op once created
    if (e_) return B200M_OK;
    cudaEvent_t e = nullptr;
    CK(cudaEventCreateWithFlags(&e, flags));
    e_ = e;
    return B200M_OK;
  }
  operator cudaEvent_t() const { return e_; }

 private:
  cudaEvent_t e_ = nullptr;
};

// A non-blocking stream of its own, or one the caller lent (never destroyed here).
class Stream {
 public:
  Stream() = default;
  Stream(Stream&& o) noexcept : s_(std::exchange(o.s_, nullptr)), own_(std::exchange(o.own_, false)) {}
  Stream& operator=(Stream&& o) noexcept { std::swap(s_, o.s_); std::swap(own_, o.own_); return *this; }
  ~Stream() { if (own_) cudaStreamDestroy(s_); }
  int create() {
    cudaStream_t s = nullptr;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    s_ = s; own_ = true;
    return B200M_OK;
  }
  void borrow(cudaStream_t s) { s_ = s; }
  operator cudaStream_t() const { return s_; }

 private:
  cudaStream_t s_ = nullptr;
  bool own_ = false;
};

}  // namespace b200m
