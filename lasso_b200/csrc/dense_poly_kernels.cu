// lasso_b200 — ingest of a caller's dense polynomial (DensePolynomial::new, poly/dense_mlpoly.rs:62-71).
// Two passes over the evaluations: the copy into the library's buffer with the canonical-residue check and the widest
// value's bit width, and — for integer-valued polynomials (every value below 2^32) — a u32 mirror that lets the
// commitment and the opening run over the 16-bit digit tables and the IMAD dot products (poly_kernels.cu bound_u32).
// Then the binds of up to 8 variables per pass over a caller's polynomial (DESIGN §3.14).
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

// ---- binds of several variables in one pass (DESIGN §3.14)
// The 2^t weights eq(pt, b), pt.r[0] on the most significant bit of b, times pt.scale, built by the CTA into shared
// memory.  t <= kBindPassVars, so the table is at most 256 elements (8 KiB).
__device__ __forceinline__ void bind_weights(const BindPass& pt, fr_t* w) {
  const int nw = 1 << pt.t;
  for (int b = threadIdx.x; b < nw; b += blockDim.x) {
    fr_t x = pt.scale;
    for (int j = 0; j < pt.t; j++) x = fr_mul(x, (b >> (pt.t - 1 - j)) & 1 ? pt.r[j] : pt.omr[j]);
    w[b] = x;
  }
  __syncthreads();
}
// out[i] = sum_b w[b] P[b m + i], i < m: the top t variables bound at once.  A CTA covers 256 / S consecutive outputs,
// and the S = 2^lg_s threads of an output each take 2^t / S of its terms (S > 1 only when m alone would leave the GPU
// idle: m = 2^12 at 2^20 and t = 8), adding their sums in shared memory.  The threads of one slice take consecutive
// outputs, so a warp's loads are runs of 256 B to 1 KiB (32 B to 128 B from the u32 mirror).  The integer form sums
// its products (Montgomery weight x integer) as one 320-bit integer (< 2^253 * 2^32 * 2^8) and reduces once.
template <bool U32>
__global__ void __launch_bounds__(kIngestThreads)
    bind_top_multi_kernel(const void* in, size_t m, int lg_s, BindPass pt, fr_t* out) {
  __shared__ fr_t w[1 << kBindPassVars];
  __shared__ fr_t part[kIngestThreads];
  bind_weights(pt, w);
  const int per = kIngestThreads >> lg_s, s = threadIdx.x / per, il = threadIdx.x - s * per;
  const int nb = (1 << pt.t) >> lg_s, b0 = s * nb;
  const size_t blocks = (m + per - 1) / per;
  for (size_t c = blockIdx.x; c < blocks; c += gridDim.x) {  // uniform over the CTA: __syncthreads below
    const size_t i = c * per + il;
    fr_t acc = fr_zero();
    if (i < m) {
      if (U32) {
        const uint32_t* P = static_cast<const uint32_t*>(in) + i;
        wide_t wa;
        wide_zero(wa);
        for (int b = b0; b < b0 + nb; b++) wide_mad(wa, w[b], __ldcs(P + (size_t)b * m));
        acc = wide_reduce(wa);
      } else {
        const fr_t* P = static_cast<const fr_t*>(in) + i;
        for (int b = b0; b < b0 + nb; b++) acc = fr_add(acc, fr_mul(w[b], ld_fr_stream(P + (size_t)b * m)));
      }
    }
    if (lg_s == 0) {
      if (i < m) st_fr(out + i, acc);
      continue;
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    if (s == 0 && i < m) {
      for (int k = 1; k < (1 << lg_s); k++) acc = fr_add(acc, part[k * per + il]);
      st_fr(out + i, acc);
    }
    __syncthreads();
  }
}
void launch_bind_top_multi(const fr_t* in_fr, const uint32_t* in_u32, size_t n, const BindPass& pt, fr_t* out,
                           cudaStream_t st) {
  const size_t m = n >> pt.t;
  int lg_s = 0;  // threads per output: until about 2^17 threads (the resident threads of the 132 SMs) are busy
  while (lg_s < 5 && lg_s < pt.t && (m << lg_s) < ((size_t)1 << 17)) lg_s++;
  const size_t per = (size_t)kIngestThreads >> lg_s;
  size_t b = (m + per - 1) / per;
  if (b > (size_t)kNumSMs * 8) b = (size_t)kNumSMs * 8;
  if (b == 0) return;
  if (in_u32)
    launch(bind_top_multi_kernel<true>, (unsigned)b, kIngestThreads, 0, st, static_cast<const void*>(in_u32), m, lg_s, pt, out);
  else
    launch(bind_top_multi_kernel<false>, (unsigned)b, kIngestThreads, 0, st, static_cast<const void*>(in_fr), m, lg_s, pt, out);
}

// out[i] = sum_b w[b] P[i 2^t + b]: the bottom t variables bound at once, with pt.r[0] on the most significant of them
// (the caller reverses its challenges).  Thread = input element, so every load of a warp is 1 KiB contiguous; the
// products of one group of 2^t consecutive elements are then added by a butterfly over the lanes (t <= 5), and for
// t > 5 by the warps' sums in shared memory.  A chunk is the CTA's 256 consecutive elements.
__global__ void __launch_bounds__(kIngestThreads) bind_bot_multi_kernel(const fr_t* P, size_t n, BindPass pt, fr_t* out) {
  __shared__ fr_t w[1 << kBindPassVars];
  __shared__ fr_t s_warp[kIngestThreads / 32];
  bind_weights(pt, w);
  const int t = pt.t, lane_bits = t < 5 ? t : 5, mask = (1 << t) - 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t chunks = (n + kIngestThreads - 1) / kIngestThreads;
  for (size_t c = blockIdx.x; c < chunks; c += gridDim.x) {  // uniform over the CTA: __syncthreads below
    const size_t e = c * kIngestThreads + threadIdx.x;
    fr_t x = e < n ? fr_mul(w[e & mask], ld_fr_stream(P + e)) : fr_zero();
    for (int d = 1; d < (1 << lane_bits); d <<= 1) {
      fr_t o;
#pragma unroll
      for (int l = 0; l < 8; l++) o.v[l] = __shfl_xor_sync(0xffffffffu, x.v[l], d);
      x = fr_add(x, o);
    }
    if (t <= 5) {
      if (e < n && (e & mask) == 0) st_fr(out + (e >> t), x);
      continue;
    }
    if (lane == 0) s_warp[warp] = x;
    __syncthreads();
    const int wpg = 1 << (t - 5);  // warps per group: 2, 4 or 8
    if ((int)threadIdx.x < (kIngestThreads / 32) / wpg) {
      const size_t e0 = c * kIngestThreads + (size_t)threadIdx.x * wpg * 32;
      fr_t s = s_warp[threadIdx.x * wpg];
      for (int k = 1; k < wpg; k++) s = fr_add(s, s_warp[threadIdx.x * wpg + k]);
      if (e0 < n) st_fr(out + (e0 >> t), s);
    }
    __syncthreads();
  }
}
void launch_bind_bot_multi(const fr_t* in, size_t n, const BindPass& pt, fr_t* out, cudaStream_t st) {
  size_t b = (n + kIngestThreads - 1) / kIngestThreads;
  if (b > (size_t)kNumSMs * 8) b = (size_t)kNumSMs * 8;
  if (b == 0) return;
  launch(bind_bot_multi_kernel, (unsigned)b, kIngestThreads, 0, st, in, n, pt, out);
}

// The partial sums of a sharded bottom bind of k < lg G variables: rank g holds element x = i G + g of every group,
// whose bound index is j = x >> k and whose weight is `weight` (the same for every element of the rank).  out[j] for
// every j < m: weight * P[(j - (g >> k)) / (G >> k)] where j = g >> k mod G >> k, else zero.
__global__ void __launch_bounds__(kIngestThreads)
    bind_bot_spread_kernel(const fr_t* P, size_t m, size_t period, size_t phase, fr_t weight, fr_t* out) {
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (size_t)gridDim.x * blockDim.x) {
    const size_t q = j / period;
    st_fr(out + j, j - q * period == phase ? fr_mul(weight, ld_fr(P + q)) : fr_zero());
  }
}
void launch_bind_bot_spread(const fr_t* in, size_t m, size_t period, size_t phase, const fr_t& weight, fr_t* out,
                            cudaStream_t st) {
  size_t b = (m + kIngestThreads - 1) / kIngestThreads;
  if (b > (size_t)kNumSMs * 8) b = (size_t)kNumSMs * 8;
  if (b == 0) return;
  launch(bind_bot_spread_kernel, (unsigned)b, kIngestThreads, 0, st, in, m, period, phase, weight, out);
}

}  // namespace lb
