// One owner for every device (cudaMalloc) and pinned host (cudaMallocHost) array of the library.  Host code only: a plain
// host compiler builds it.
//
// A growth that fails leaves the buffer empty (null, capacity 0) and clears the error from cudaGetLastError, so no capacity
// outlives the array it describes and a later launch check does not report the allocation.  Arrays that grow together
// reset each other when one of them fails, so any one of them tells the group's capacity.
#ifndef LS_BUFFER_CUH_
#define LS_BUFFER_CUH_

#include <cstddef>

#include <cuda_runtime.h>

namespace ls {

template <class T, bool kPinned = false>
class Buffer {
 public:
  Buffer() = default;
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;
  Buffer(Buffer&& o) noexcept : p_(o.p_), cap_(o.cap_) {
    o.p_ = nullptr;
    o.cap_ = 0;
  }
  Buffer& operator=(Buffer&& o) noexcept {
    if (this != &o) {
      reset();
      p_ = o.p_;
      cap_ = o.cap_;
      o.p_ = nullptr;
      o.cap_ = 0;
    }
    return *this;
  }
  ~Buffer() { reset(); }

  T* get() const { return p_; }
  size_t capacity() const { return cap_; }  // elements

  // Nothing when need <= capacity().  Otherwise frees the old allocation and allocates cap (>= need, at least 1) elements.
  // On failure the buffer is empty, and the error is returned and cleared from cudaGetLastError.
  cudaError_t reserve(size_t need, size_t cap) {
    if (need <= cap_) return cudaSuccess;
    reset();
    if (cap < need) cap = need;
    if (cap < 1) cap = 1;
    void* q = nullptr;
    const cudaError_t e = kPinned ? cudaMallocHost(&q, cap * sizeof(T)) : cudaMalloc(&q, cap * sizeof(T));
    if (e != cudaSuccess) {
      cudaGetLastError();
      return e;
    }
    p_ = static_cast<T*>(q);
    cap_ = cap;
    return cudaSuccess;
  }

  void reset() {
    if (p_) {
      if (kPinned) cudaFreeHost(p_);
      else cudaFree(p_);
    }
    p_ = nullptr;
    cap_ = 0;
  }

 private:
  T* p_ = nullptr;
  size_t cap_ = 0;
};

template <class T>
using PinnedBuffer = Buffer<T, true>;

}  // namespace ls

#endif  // LS_BUFFER_CUH_
