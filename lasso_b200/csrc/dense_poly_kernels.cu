// lasso_b200 — ingest of a caller's dense polynomial (DensePolynomial::new, poly/dense_mlpoly.rs:62-71).
// Two passes over the evaluations: the copy into the library's buffer with the canonical-residue check and the widest
// value's bit width, and — for integer-valued polynomials (every value below 2^32) — a u32 mirror that lets the
// commitment and the opening run over the 16-bit digit tables and the IMAD dot products (poly_kernels.cu bound_u32).
#include "kernels.cuh"

namespace lb {

static constexpr int kIngestThreads = 256;

// Rows may be only 8-byte aligned (a strided view of an int64 tensor), so the limbs are read as four 64-bit loads.
// The widest value is reduced over the warp, then over the CTA, and one atomic per CTA publishes it.
__global__ void __launch_bounds__(kIngestThreads)
    poly_ingest_kernel(const uint64_t* src, size_t row_stride, size_t n, fr_t* dst, unsigned* flags) {
  __shared__ unsigned s_bits[kIngestThreads / 32];
  unsigned mb = 0, bad = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint64_t* p = src + i * row_stride;
    fr_t x;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const uint64_t w = p[k];
      x.v[2 * k] = (uint32_t)w;
      x.v[2 * k + 1] = (uint32_t)(w >> 32);
    }
    // x < l  <=>  subtracting l once changes nothing (for x >= l it always does)
    if (!fr_eq(fr_reduce_once(x.v), x)) {
      bad = 1;
    } else {
      const fr_t c = fr_to_canonical(x);
      unsigned b = 0;
#pragma unroll
      for (int l = 0; l < 8; l++)
        if (c.v[l]) b = 32 * l + (32 - __clz(c.v[l]));
      mb = b > mb ? b : mb;
    }
    st_fr(dst + i, x);
  }
  mb = __reduce_max_sync(0xffffffffu, mb);
  bad = __reduce_or_sync(0xffffffffu, bad);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_bits[warp] = mb;
    if (bad) atomicOr(flags, 1u);
  }
  __syncthreads();
  if (warp == 0) {
    unsigned v = lane < (int)(blockDim.x >> 5) ? s_bits[lane] : 0u;
    v = __reduce_max_sync(0xffffffffu, v);
    if (lane == 0 && v) atomicMax(flags + 1, v);
  }
}
void launch_poly_ingest(const uint64_t* src, size_t row_stride, size_t n, fr_t* dst, unsigned* flags, cudaStream_t st) {
  size_t b = (n + kIngestThreads - 1) / kIngestThreads;
  if (b > (size_t)kNumSMs * 8) b = (size_t)kNumSMs * 8;
  if (b == 0) return;
  launch(poly_ingest_kernel, (unsigned)b, kIngestThreads, 0, st, src, row_stride, n, dst, flags);
}

__global__ void __launch_bounds__(kIngestThreads) poly_mirror_u32_kernel(const fr_t* in, size_t n, uint32_t* out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = fr_to_canonical(ld_fr(in + i)).v[0];
}
void launch_poly_mirror_u32(const fr_t* in, size_t n, uint32_t* out, cudaStream_t st) {
  size_t b = (n + kIngestThreads - 1) / kIngestThreads;
  if (b > (size_t)kNumSMs * 8) b = (size_t)kNumSMs * 8;
  if (b == 0) return;
  launch(poly_mirror_u32_kernel, (unsigned)b, kIngestThreads, 0, st, in, n, out);
}

}  // namespace lb
