// chromap_b200 — owners of the CUDA resources the library's host code holds (api.cu, the index build): device memory, and
// streams, events and page-locked host memory.  Move-only; the destructor releases, and reset() releases early where that
// bounds peak device memory.  Also the error return of a failing runtime call into a plain string.  Host code only.
#pragma once
#include <cuda_runtime.h>

#include <cstdio>
#include <string>
#include <type_traits>
#include <utility>

#include "../../include/chromap_b200.h"

// Device memory.  alloc(bytes) releases what the owner holds before it allocates exactly `bytes`, so a regrow never holds both.
template <class T = void>
struct DevMem {
  T *p = nullptr;
  size_t cap = 0;  // bytes
  DevMem() = default;
  DevMem(DevMem &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevMem &operator=(DevMem &&o) noexcept {
    if (this != &o) { reset(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); }
    return *this;
  }
  ~DevMem() { reset(); }
  void reset() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  cudaError_t alloc(size_t bytes) {
    reset();
    const cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes; else p = nullptr;
    return e;
  }
  operator T *() const { return p; }
};

// A stream, an event or a page-locked host buffer.  alloc(arg) makes a non-blocking stream, an event with flags `arg`, or
// `arg` bytes of page-locked host memory.
template <class H, cudaError_t (*Release)(H)>
struct CudaHandle {
  H h = nullptr;
  CudaHandle() = default;
  CudaHandle(CudaHandle &&o) noexcept : h(std::exchange(o.h, nullptr)) {}
  CudaHandle &operator=(CudaHandle &&o) noexcept {
    if (this != &o) { reset(); h = std::exchange(o.h, nullptr); }
    return *this;
  }
  ~CudaHandle() { reset(); }
  void reset() { if (h) Release(h); h = nullptr; }
  cudaError_t alloc(size_t arg = 0) {
    reset();
    cudaError_t e;
    if constexpr (std::is_same_v<H, cudaStream_t>) e = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking);
    else if constexpr (std::is_same_v<H, cudaEvent_t>) e = cudaEventCreateWithFlags(&h, (unsigned)arg);
    else e = cudaMallocHost(&h, arg);
    if (e != cudaSuccess) h = nullptr;
    return e;
  }
  operator H() const { return h; }
};
using Stream = CudaHandle<cudaStream_t, cudaStreamDestroy>;
using Event = CudaHandle<cudaEvent_t, cudaEventDestroy>;
using PinnedMem = CudaHandle<void *, cudaFreeHost>;

// A failing runtime call returns CMX_ERR_CUDA and leaves its place and message in the std::string `err` of the caller: a
// lane's own (lanes run on their own host threads and must not write the context's), or the index build's.
#define CUE(call)                                                                                  \
  do {                                                                                             \
    const cudaError_t e_ = (call);                                                                 \
    if (e_ != cudaSuccess) {                                                                       \
      char b_[512];                                                                                \
      snprintf(b_, sizeof(b_), "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
      err = b_;                                                                                    \
      return CMX_ERR_CUDA;                                                                         \
    }                                                                                              \
  } while (0)
