// Device side of the arithmetic harness: one kernel per operation of arith_ops.cuh, and the launcher KH_ARITH_LAUNCH
// that arith.cu calls.  Included by arith_default.cu and arith_msm.cu, which differ only in the fq_mul attributes
// they choose before including it: the same source compiled the two ways the library compiles it.
#pragma once
#ifndef KH_ARITH_LAUNCH
#error "define KH_ARITH_LAUNCH (the launcher's name) before including arith_kernels.cuh"
#endif
#include <stdexcept>

#include "../../lasso_b200/csrc/quad.cuh"
#include "arith_ops.cuh"

namespace {

using namespace arith;

template <int OP>
__global__ void __launch_bounds__(128) arith_thread_kernel(size_t n, const uint32_t* a, const uint32_t* b, const uint64_t* k,
                                                           uint32_t* out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    apply(OP, a + 32 * i, b + 32 * i, k[i], out + 32 * i);
}

// lane 4e + role holds coordinate `role` of element e (X, Y, Z, T), as the callers of quad.cuh hold a point.  The
// grid is whole warps and every lane runs the same path: lanes past the end repeat the last element and store nothing.
template <int OP>
__global__ void __launch_bounds__(128) arith_quad_kernel(size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  const size_t e = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const int lane = threadIdx.x & 31, role = lane & 3;
  const size_t ei = e < n ? e : n - 1;
  const fq_t mine = ldq(a + 32 * ei, role);
  fq_t r;
  if (OP == OP_quad_add) {
    r = lb::quad_add(0xffffffffu, lane, mine, reinterpret_cast<const fq_t*>(b + 32 * ei));  // X2, Y2, Z2, T2
  } else if (OP == OP_quad_madd) {
    // b = niels (y+x, y-x, 2dxy); lanes 0 / 1 / 3 take y-x / y+x / 2dxy (a positive digit), lane 2 nothing
    const int src = role == 0 ? 1 : role == 1 ? 0 : 2;
    r = lb::quad_madd(0xffffffffu, lane, mine, ldq(b + 32 * ei, src));
  } else {
    r = lb::quad_dbl(0xffffffffu, lane, mine);
  }
  if (e < n) stq(out + 32 * e, role, r);
}

}  // namespace

// a, b, out: device arrays of n elements of 32 u32; k: n u64
void KH_ARITH_LAUNCH(int op, size_t n, const uint32_t* a, const uint32_t* b, const uint64_t* k, uint32_t* out,
                     cudaStream_t st) {
  size_t blocks = (n + 127) / 128;
  if (blocks > 4096) blocks = 4096;
  const unsigned quad_blocks = (unsigned)((4 * n + 127) / 128);
  switch (op) {
#define KH_ARITH_THREAD_CASE(name) \
  case OP_##name: lb::launch(arith_thread_kernel<OP_##name>, (unsigned)blocks, 128, 0, st, n, a, b, k, out); break;
    KH_ARITH_THREAD_OPS(KH_ARITH_THREAD_CASE)
#undef KH_ARITH_THREAD_CASE
#define KH_ARITH_QUAD_CASE(name) \
  case OP_##name: lb::launch(arith_quad_kernel<OP_##name>, quad_blocks, 128, 0, st, n, a, b, out); break;
    KH_ARITH_QUAD_OPS(KH_ARITH_QUAD_CASE)
#undef KH_ARITH_QUAD_CASE
    default: throw std::runtime_error("kh_arith: unknown operation");
  }
}
