// Test harness plumbing shared by its translation units (harness.cu, harness_comb.cu, harness_msm.cu, arith.cu,
// harness_fr.cu): error codes, the per-call device allocation scope, the publication region of the launchers that
// publish, the generator tables, and the wrapper that turns exceptions into return codes.
// Return codes: 0 ok, -1 a launcher threw (std::runtime_error), -2 a CUDA error, -3 a publication slot did not carry
// the message's tag, -4 bad arguments, -5 a repeated launch published different values (harness_comb.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
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

// one publication region in mapped pinned host memory (as the prover's Ctx); messages carry tag 1 unless set_tag
struct Pub {
  unsigned long long* h = nullptr;
  lb::PubDst dst = {};
  explicit Pub(Scope& s) {
    const size_t bytes = (size_t)lb::kPubElems * lb::kPubSlotWords * 8;
    ck(cudaHostAlloc((void**)&h, bytes, cudaHostAllocMapped));
    s.host.push_back(h);
    memset(h, 0, bytes);
    unsigned long long* d = nullptr;
    ck(cudaHostGetDevicePointer((void**)&d, h, 0));
    dst.dst[0] = d;
    dst.ndst = 1;
    dst.tag = 1;
  }
  // the next launch publishes with this tag (a Finalize copied before the call keeps the old one)
  void set_tag(uint32_t tag) { dst.tag = tag; }
  // elements [v0, v0 + count) -> out (4 x u64 each); every word must carry the current tag
  void decode(int v0, int count, uint64_t* out) const {
    for (int v = v0; v < v0 + count; v++) {
      unsigned long long w[5];
      for (int k = 0; k < 5; k++) {
        const unsigned long long word = h[(size_t)v * lb::kPubSlotWords + k];
        if (lb::pub_tag_of(word) != dst.tag) throw HarnessError{-3};
        w[k] = word & lb::kPubValueMask;
      }
      uint32_t x[8];
      lb::pub_decode(w, x);
      memcpy(out + 4 * (size_t)(v - v0), x, 32);
    }
  }
  // elements [v0, v0 + count) must not have been written
  void expect_empty(int v0, int count) const {
    for (size_t i = (size_t)v0 * lb::kPubSlotWords; i < (size_t)(v0 + count) * lb::kPubSlotWords; i++)
      if (h[i] != 0) throw HarnessError{-3};
  }
};

// window + digit-multiples tables of a generator set (kh_tables_create, harness.cu; kh_tables_build, harness_setup.cu).
// The device arrays belong to the process's primary context, so every harness library loaded into the process can use
// them.  T has npts points per window; M covers the first nd of them (nd == npts unless built by kh_tables_build);
// K16[k] = the centring constant of 2^k local columns, for every 2^k <= ncols16 (kh_tables_build only).
struct KhTables {
  size_t npts = 0, ncols16 = 0;
  lb::pt_niels *T = nullptr, *M = nullptr, *M16 = nullptr;
  size_t nd = 0, nk16 = 0;
  lb::pt_ext* K16 = nullptr;
};

inline lb::Finalize make_fin(Scope& s, const Pub& p, size_t partial_elems) {
  lb::Finalize f;
  f.partial = s.alloc<lb::fr_t>(partial_elems);
  f.counter = s.alloc<unsigned>(1);
  f.pub = p.dst;
  return f;
}

inline lb::fr_t fr_of(const uint64_t* x) {
  lb::fr_t r;
  memcpy(r.v, x, 32);
  return r;
}

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
