// The arithmetic harness with fq_mul's default attributes: inlined, arguments by reference (as msm_final.cu,
// poly_kernels.cu and the Bulletproofs kernels compile it).
#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

void kh_arith_launch_default(int op, size_t n, const uint32_t* a, const uint32_t* b, const uint64_t* k, uint32_t* out,
                             cudaStream_t st);
#define KH_ARITH_LAUNCH kh_arith_launch_default
#include "arith_kernels.cuh"
