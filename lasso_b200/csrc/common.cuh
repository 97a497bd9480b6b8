// lasso_b200 — shared device helpers: 32-byte global loads/stores of field elements,
// warp-shuffle + shared-memory reductions of Fr partial sums, error checking, the kernel launch helper.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <utility>

#include "ed25519.cuh"
#include "pub_codec.hpp"

namespace lb {

#define LB_CUDA_CHECK(x)                                                                              \
  do {                                                                                                \
    cudaError_t e_ = (x);                                                                             \
    if (e_ != cudaSuccess)                                                                            \
      throw std::runtime_error(std::string("CUDA error ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + \
                               std::to_string(__LINE__));                                             \
  } while (0)

static constexpr int kNumSMs = 132;  // H100 SXM

// kernels launched by this library in this process (lasso_launch_count, bench.py's gpu_launches); only launch() adds
// to it, so copies, memsets and NCCL's own kernels are not counted
inline std::atomic<unsigned long long> g_launches{0};

#if defined(__CUDACC__)
// Every kernel launch of the library goes through here.  A bad configuration (shared memory opt-in missing on this
// device, grid too large) fails synchronously and must not go unnoticed; a launch that was enqueued is counted.
template <typename... Params, typename... Args>
void launch(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
  LB_CUDA_CHECK(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
}

// One 32-byte element per thread as two 128-bit accesses (the widest global access sm_90 has). The first
// instruction of a warp touches every 32-byte sector the warp needs; the second is expected to hit those sectors in
// L1, so DRAM should still see each element once (not profiled; the bind kernel's measured bandwidth, DESIGN.md §7,
// is consistent with it).
__device__ __forceinline__ void ld_u32x8(uint32_t (&v)[8], const void* p) {
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p));
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
               : "l"((const char*)p + 16));
}
__device__ __forceinline__ void st_u32x8(void* p, const uint32_t (&v)[8]) {
  asm volatile("st.global.v4.u32 [%4], {%0,%1,%2,%3};" ::"r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]), "l"(p) : "memory");
  asm volatile("st.global.v4.u32 [%4], {%0,%1,%2,%3};" ::"r"(v[4]), "r"(v[5]), "r"(v[6]), "r"(v[7]),
               "l"((char*)p + 16)
               : "memory");
}
__device__ __forceinline__ fr_t ld_fr(const fr_t* p) {
  fr_t r;
  ld_u32x8(r.v, p);
  return r;
}
// streaming variant for data read exactly once per kernel: first in line for eviction from L1, rather than not
// allocated there, so that the second half of the element can still hit
__device__ __forceinline__ fr_t ld_fr_stream(const fr_t* p) {
  fr_t r;
  asm volatile("ld.global.L1::evict_first.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3])
               : "l"(p));
  asm volatile("ld.global.L1::evict_first.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
               : "l"((const char*)p + 16));
  return r;
}
__device__ __forceinline__ void st_fr(fr_t* p, const fr_t& r) { st_u32x8(p, r.v); }
__device__ __forceinline__ fq_t ld_fq(const fq_t* p) {
  fq_t r;
  ld_u32x8(r.v, p);
  return r;
}
__device__ __forceinline__ void st_fq(fq_t* p, const fq_t& r) { st_u32x8(p, r.v); }

__device__ __forceinline__ fr_t shfl_down_fr(const fr_t& a, int delta) {
  fr_t r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = __shfl_down_sync(0xffffffffu, a.v[i], delta);
  return r;
}
// sum over the warp, result valid in lane 0
__device__ __forceinline__ fr_t warp_sum_fr(fr_t a) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) a = fr_add(a, shfl_down_fr(a, d));
  return a;
}
// Sum NV values per thread over the block.  `scratch` needs NV * (blockDim.x/32) elements.
// Result valid in thread 0.
template <int NV>
__device__ __forceinline__ void block_sum_fr(fr_t (&v)[NV], fr_t* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; k++) {
    v[k] = warp_sum_fr(v[k]);
    if (lane == 0) scratch[k * nwarps + warp] = v[k];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NV; k++) {
      fr_t x = lane < nwarps ? scratch[k * nwarps + lane] : fr_zero();
      v[k] = warp_sum_fr(x);
    }
  }
  __syncthreads();
}

// A sum of products (Montgomery field element) x (32-bit integer) carried as a plain 320-bit integer and reduced once
// (poly_kernels.cu K7, dense_poly_kernels.cu): an element stored as a*R mod l times z sums to the Montgomery form of
// sum a z.
struct wide_t {
  uint32_t v[10];
};
__device__ __forceinline__ void wide_zero(wide_t& a) {
#pragma unroll
  for (int l = 0; l < 10; l++) a.v[l] = 0;
}
__device__ __forceinline__ void wide_mad(wide_t& acc, const fr_t& a, uint32_t z) {  // acc += a * z
  uint64_t carry = 0;
#pragma unroll
  for (int l = 0; l < 8; l++) {
    const uint64_t t = (uint64_t)a.v[l] * z + acc.v[l] + carry;
    acc.v[l] = (uint32_t)t;
    carry = t >> 32;
  }
  const uint64_t t = (uint64_t)acc.v[8] + carry;
  acc.v[8] = (uint32_t)t;
  acc.v[9] += (uint32_t)(t >> 32);
}
// X mod l for X < 2^320, as a field element: X = X_lo + 2^256 * X_hi;  X_lo mod l through two Montgomery products
// (x -> x*R -> x), X_hi * 2^256 mod l = the Montgomery form of the 64-bit integer X_hi
__device__ __forceinline__ fr_t wide_reduce(const wide_t& a) {
  fr_t lo;
#pragma unroll
  for (int l = 0; l < 8; l++) lo.v[l] = a.v[l];
  const fr_t lo_mod = fr_to_canonical(fr_from_raw_int(lo));
  return fr_add(lo_mod, fr_from_u64((uint64_t)a.v[8] | ((uint64_t)a.v[9] << 32)));
}
// ---- single-launch reduction + publication of a round message ---------------------------------------------
// Every CTA stores its partial sums, takes a ticket, and the LAST CTA to finish adds the partials of all
// values and writes the results straight into mapped pinned host memory the host is spinning on.  One kernel per sumcheck round instead of eval + reduce + copy: the rounds of the
// grand-product ladder are pure launch/sync latency.
//
// Publication needs no flag and no system-scope fence (each costs microseconds per round) and makes NO
// assumption about the atomicity of wide stores: a published value x < 2^255 (an Fr residue or a canonical
// Fq coordinate) travels as FIVE 64-bit words, word k = bits [51k, 51k+51) of x in its low 51 bits and a
// 13-bit message tag in its high bits.  Aligned 64-bit stores are single-copy atomic in the PTX memory model,
// so every word identifies the message it belongs to on its own: the host polls each of the five words for the
// tag of the message it waits for, reassembles x, and zeroes the slot (a cleared word can never satisfy a later
// wait).  Order between words or elements is irrelevant; a word of an older message is simply not accepted.
// One proof sharded over G GPUs uses the same mechanism as its per-round exchange: every process maps every
// other process's receive buffer (a shared pinned host segment, comm.cu) and each GPU stores its partial sums
// into all G of them — the G replicated host transcripts add the G residues, no collective, no extra launch.
static constexpr int kPubSlotWords = 8;       // 64 B per element slot (5 words used): never straddles a line
static constexpr int kPubMaxReaders = 8;      // one node
static constexpr int kPubRegions = 4;         // rings of regions per writer (prover.cuh pub_begin)
static constexpr int kPubElems = 512;         // elements per region (largest message: 8 * alpha tree tops)
static constexpr uint32_t kPubTagMod = 8191;  // tags 1..8191 (13 bits, 0 = empty)
struct PubDst {
  unsigned long long* dst[kPubMaxReaders];  // device pointers: (this writer, region) inside reader p's buffer
  int ndst;
  uint32_t tag;
  // host-side bookkeeping of the wait (ignored by kernels)
  int region, all;
};
// x = 8 x u32 little-endian, x < 2^255
__device__ __forceinline__ void pub_store(const PubDst& p, int v, const uint32_t x[8]) {
  unsigned long long w[5];
  pub_encode(x, p.tag, w);
#pragma unroll 1
  for (int d = 0; d < p.ndst; d++) {
    unsigned long long* s = p.dst[d] + (size_t)v * kPubSlotWords;
    asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(s), "l"(w[0]), "l"(w[1]) : "memory");
    asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(s + 2), "l"(w[2]), "l"(w[3]) : "memory");
    asm volatile("st.global.u64 [%0], %1;" ::"l"(s + 4), "l"(w[4]) : "memory");
  }
}
struct Finalize {
  fr_t* partial;      // scratch: [nvals][blocks_per_val]
  unsigned* counter;  // device ticket counter: 0 on entry, reset to 0 by the last CTA
  PubDst pub;         // publication of the nvals results to mapped host memory
};
__device__ __forceinline__ fr_t ld_fr_cg(const fr_t* p) {  // bypass L1: written by other CTAs of this launch
  fr_t r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]) : "l"(p));
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
               : "l"((const char*)p + 16));
  return r;
}
// result v of a round: tagged host copy
__device__ __forceinline__ void finalize_publish(const Finalize& f, int v, const fr_t& val) { pub_store(f.pub, v, val.v); }
// the LAST CTA of a launch (all threads): add the partials of every value and publish
__device__ __forceinline__ void finalize_last_stage(const Finalize& f, int blocks_per_val, int nvals_total) {
  __threadfence();
  // groups of gsz = 2^k >= min(32, blocks_per_val) lanes add the partials of one value each
  int gsz = 1;
  while (gsz < blocks_per_val && gsz < 32) gsz <<= 1;
  const int lane_g = threadIdx.x & (gsz - 1), ngroups = blockDim.x / gsz;
  for (int base = 0; base < nvals_total; base += ngroups) {  // uniform trip count: full-warp shuffles inside
    const int v = base + threadIdx.x / gsz;
    const bool ok = v < nvals_total;
    fr_t acc = fr_zero();
    if (ok)
      for (int i = lane_g; i < blocks_per_val; i += gsz) acc = fr_add(acc, ld_fr_cg(f.partial + (size_t)v * blocks_per_val + i));
    for (int d = gsz >> 1; d > 0; d >>= 1) {
      fr_t o;
#pragma unroll
      for (int l = 0; l < 8; l++) o.v[l] = __shfl_down_sync(0xffffffffu, acc.v[l], d, gsz);
      acc = fr_add(acc, o);
    }
    if (ok && lane_g == 0) finalize_publish(f, v, acc);
  }
  if (threadIdx.x == 0) *f.counter = 0;
}
// vals[0..NV) are valid in thread 0 of the CTA; they belong to value indices v0 .. v0+NV, partial slot bidx.
template <int NV>
__device__ __forceinline__ void finalize_block(const Finalize& f, const fr_t (&vals)[NV], int v0, int bidx,
                                               int blocks_per_val, int nvals_total, int total_blocks) {
  __shared__ int s_last;
  if (total_blocks == 1) {  // single CTA: nothing to combine
    if (threadIdx.x == 0) {
#pragma unroll
      for (int t = 0; t < NV; t++) finalize_publish(f, v0 + t, vals[t]);
    }
    return;
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int t = 0; t < NV; t++) f.partial[(size_t)(v0 + t) * blocks_per_val + bidx] = vals[t];
    __threadfence();
    unsigned ticket = atomicAdd(f.counter, 1u);
    s_last = (ticket == (unsigned)total_blocks - 1u);
  }
  __syncthreads();
  if (!s_last) return;
  finalize_last_stage(f, blocks_per_val, nvals_total);
}

#endif

}  // namespace lb
