// The arithmetic harness with the fq_mul attributes of msm_kernels.cu and msm_large.cu: an out-of-line function that
// takes its arguments by value.
#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

void kh_arith_launch_msm(int op, size_t n, const uint32_t* a, const uint32_t* b, const uint64_t* k, uint32_t* out,
                         cudaStream_t st);
#define LB_FQ_MUL_ATTR static __host__ __device__ __noinline__
#define LB_FQ_MUL_BYVALUE
#define KH_ARITH_LAUNCH kh_arith_launch_msm
#include "arith_kernels.cuh"
