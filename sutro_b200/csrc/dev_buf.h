// sutro_b200 — device allocations owned by host objects.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "common.cuh"

namespace sb {

// device allocation that frees itself on every return path
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;  // bytes asked for by the last alloc()

  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  // (re)allocates `bytes` (at least one); the previous allocation and its contents are gone
  int alloc(size_t bytes) {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    void* q = nullptr;
    SB_CUDA_CHECK(cudaMalloc(&q, bytes ? bytes : 1));
    p = q;
    cap = bytes;
    return 0;
  }
  // grow-only: reallocates only when `bytes` exceeds the allocation held (never when both are 0)
  int reserve(size_t bytes) { return bytes <= cap ? 0 : alloc(bytes); }
  template <class T>
  T* as() const {
    return static_cast<T*>(p);
  }
};

// a DevBuf of `T` elements that stands in for a T*
template <class T>
struct DevArray : DevBuf {
  int alloc(size_t n) { return DevBuf::alloc(n * sizeof(T)); }
  int reserve(size_t n) { return DevBuf::reserve(n * sizeof(T)); }
  T* get() const { return as<T>(); }
  operator T*() const { return get(); }
};

}  // namespace sb
