/*
 * mm_devbuf.h -- an owning device array, for host code (internal to libmashmap_b200.so).
 *
 * mm_devbuf<T> is move-only and frees its array when it goes out of scope. Allocations go to the current device.
 * After any failed reserve the array is empty (nullptr, capacity 0) and the runtime's pending error has been read and
 * cleared, so a caller that reports the returned error and comes back later finds a consistent buffer: a capacity never
 * stands for memory that is not there.
 */
#ifndef MM_DEVBUF_H
#define MM_DEVBUF_H

#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

template <typename T>
class mm_devbuf {
 public:
  mm_devbuf() = default;
  mm_devbuf(const mm_devbuf &) = delete;
  mm_devbuf &operator=(const mm_devbuf &) = delete;
  mm_devbuf(mm_devbuf &&o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)) {}
  mm_devbuf &operator=(mm_devbuf &&o) noexcept
  {
    if (this != &o) {
      reset();
      p_ = std::exchange(o.p_, nullptr);
      cap_ = std::exchange(o.cap_, 0);
    }
    return *this;
  }
  ~mm_devbuf() { reset(); }

  T *get() const { return p_; }
  uint64_t capacity() const { return cap_; } /* elements */
  explicit operator bool() const { return p_ != nullptr; }

  void reset()
  {
    if (p_) cudaFree(p_);
    p_ = nullptr;
    cap_ = 0;
  }

  /* room for n elements; growing drops the contents */
  cudaError_t reserve(uint64_t n)
  {
    if (n <= cap_) return cudaSuccess;
    reset();
    return alloc(n, p_, cap_);
  }

  /* room for n elements; growing keeps [0, used), copied on `st`, which is synchronised before the old array goes */
  cudaError_t reserve_keep(uint64_t n, uint64_t used, cudaStream_t st)
  {
    if (n <= cap_) return cudaSuccess;
    T *q = nullptr;
    uint64_t q_cap = 0;
    cudaError_t e = alloc(n, q, q_cap);
    if (e == cudaSuccess && used) e = cudaMemcpyAsync(q, p_, used * sizeof(T), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    reset();
    if (e != cudaSuccess) {
      if (q) cudaFree(q);
      cudaGetLastError();
      return e;
    }
    p_ = q;
    cap_ = q_cap;
    return cudaSuccess;
  }

 private:
  static cudaError_t alloc(uint64_t n, T *&p, uint64_t &cap)
  {
    const cudaError_t e = cudaMalloc((void **)&p, n * sizeof(T));
    if (e != cudaSuccess) {
      p = nullptr;
      cap = 0;
      cudaGetLastError(); /* a failed allocation stays pending otherwise, and the next launch check would report it */
      return e;
    }
    cap = n;
    return cudaSuccess;
  }

  T *p_ = nullptr;
  uint64_t cap_ = 0;
};

#endif
