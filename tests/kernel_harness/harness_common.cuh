// Test harness plumbing shared by its translation units (harness.cu, arith.cu): error codes, the per-call device
// allocation scope, and the wrapper that turns exceptions into return codes.
// Return codes: 0 ok, -1 a launcher threw (std::runtime_error), -2 a CUDA error, -3 a publication slot did not carry
// the message's tag, -4 bad arguments.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "../../lasso_b200/csrc/kernels.cuh"
#include "../../lasso_b200/csrc/msm.cuh"

namespace kh {

struct HarnessError {
  int code;
};

inline void ck(cudaError_t e) {
  if (e != cudaSuccess) {
    fprintf(stderr, "kernel harness: CUDA error %s\n", cudaGetErrorString(e));
    throw HarnessError{-2};
  }
}

// every device allocation of one call; freed when the call returns, whatever happens
struct Scope {
  std::vector<void*> dev, host;
  cudaStream_t st = nullptr;
  Scope() { ck(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); }
  ~Scope() {
    if (st) cudaStreamSynchronize(st);
    for (void* p : dev) cudaFree(p);
    for (void* p : host) cudaFreeHost(p);
    if (st) cudaStreamDestroy(st);
  }
  template <class T>
  T* alloc(size_t count) {
    void* p = nullptr;
    ck(cudaMalloc(&p, count * sizeof(T) + 16));
    dev.push_back(p);
    ck(cudaMemsetAsync(p, 0, count * sizeof(T) + 16, st));
    return (T*)p;
  }
  template <class T>
  T* up(const void* h, size_t count) {
    T* d = alloc<T>(count);
    if (count) ck(cudaMemcpyAsync(d, h, count * sizeof(T), cudaMemcpyHostToDevice, st));
    return d;
  }
  template <class T>
  void down(void* h, const T* d, size_t count) {
    if (count) ck(cudaMemcpyAsync(h, d, count * sizeof(T), cudaMemcpyDeviceToHost, st));
  }
  // an array of device pointers to n arrays of `len` elements each, filled from host[k * len ..]
  lb::fr_t* const* ptr_array(const uint64_t* host, int n, size_t len, std::vector<lb::fr_t*>& ptrs) {
    ptrs.resize(n);
    for (int k = 0; k < n; k++) ptrs[k] = up<lb::fr_t>(host + (size_t)k * len * 4, len);
    return up<lb::fr_t*>(ptrs.data(), n);
  }
  void sync() {
    ck(cudaStreamSynchronize(st));
    ck(cudaGetLastError());
  }
};

inline bool g_inited = false;
inline void init() {
  if (g_inited) return;
  lb::poly_init_device();
  lb::msm_init_device();
  g_inited = true;
}

template <class F>
int guarded(F f) {
  try {
    init();
    f();
    return 0;
  } catch (const HarnessError& e) {
    return e.code;
  } catch (const std::runtime_error& e) {
    fprintf(stderr, "kernel harness: %s\n", e.what());
    return -1;
  }
}

}  // namespace kh
