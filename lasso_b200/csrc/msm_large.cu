// lasso_b200 — K6 for ONE large variable-base MSM (BASELINE config 5: 2^16 .. 2^26 terms): the Pippenger bucket
// method of src/msm/mod.rs:91-164 (msm_bigint_wnaf: signed c-bit digits, one bucket set per window, running-sum
// bucket reduction, c doublings between windows) laid out for a GPU.  The row-batched kernels of msm_kernels.cu are
// built for thousands of short rows over shared generators (fixed c = 8, buckets in shared memory); a single MSM of
// millions of terms wants the reference's large window (c = 13..17: ~16 bucket additions per term instead of 32)
// and buckets in HBM:
//   1. msm_prep_kernel     scalar -> canonical integer (into_bigint, msm/mod.rs:23-25), base -> affine-niels (96 B)
//   2. msm_hist_kernel     signed digits by the offset trick (digit_w = c-bit field of s + sum_w 2^(c-1) 2^(cw), minus
//                          2^(c-1): no carry chain, msm/mod.rs:277-316 yields the same digits), histogram of
//                          (window, |digit|) with RED atomics
//   3. msm_scan_*_kernel   exclusive scan (tiles, tile sums, apply) -> bucket offsets; a bucket with more than S entries
//                          (skewed scalars) is split into units of <= S entries so that no thread walks a long chain
//   4. msm_scatter_kernel  counting-sort scatter of (term | sign) by (window, bucket), one window at a time so that
//                          the window's slice of the list stays in L2
//   5. msm_accum_kernel    one THREAD per unit: a chain of mixed additions over its entries (7 Fq mul each), the
//                          next entry's 96 B in flight during the current addition;
//      msm_unit_combine    the units of a split bucket are added by one warp per bucket (none for uniform scalars)
//   6. msm_wsum_kernel     bucket reduction sum_b b * B_b: the running sum / weighted sum of msm/mod.rs:139-145 over
//                          groups of 16, applied recursively (2^16 buckets -> 4096 -> 256 -> 16 -> 1 groups), so the
//                          longest dependent chain is 32 additions per level instead of 2^17;
//      msm_psum_kernel     plain sums of every level's weighted parts
//   7. msm_final_kernel    per window W = A_0 + 16 (A_1 + 16 (...)), then the window combination sum_w 2^(c w) W_w
//                          (msm/mod.rs:150-163: c doublings per window, ~250 dependent doublings) by Horner on one QUAD
//                          of lanes (quad.cuh), then normalisation.
// Integer-ALU bound: reported as mixed additions/s.
// Same group element as msm_bigint_wnaf for every input; outputs are compared after affine normalisation.
#if defined(__CUDACC__)
#define LB_FQ_MUL_ATTR static __host__ __device__ __noinline__
#define LB_FQ_MUL_BYVALUE
#endif
#include "kernels.cuh"
#include "msm.cuh"

namespace lb {

namespace {

__device__ __forceinline__ pt_niels ldn(const pt_niels* p) {
  pt_niels n;
  n.yplusx = ld_fq(&p->yplusx);
  n.yminusx = ld_fq(&p->yminusx);
  n.t2d = ld_fq(&p->t2d);
  return n;
}
__device__ __forceinline__ void stn(pt_niels* p, const pt_niels& n) {
  st_fq(&p->yplusx, n.yplusx);
  st_fq(&p->yminusx, n.yminusx);
  st_fq(&p->t2d, n.t2d);
}
__device__ __forceinline__ pt_ext ldp(const pt_ext* p) {
  pt_ext r;
  r.X = ld_fq(&p->X);
  r.Y = ld_fq(&p->Y);
  r.Z = ld_fq(&p->Z);
  r.T = ld_fq(&p->T);
  return r;
}
__device__ __forceinline__ void stp(pt_ext* p, const pt_ext& r) {
  st_fq(&p->X, r.X);
  st_fq(&p->Y, r.Y);
  st_fq(&p->Z, r.Z);
  st_fq(&p->T, r.T);
}

// biased scalar s + sum_{w < nw} 2^(c-1) * 2^(c w) as 9 x u32 (c * nw <= 272 bits); digit w = its c-bit field w
// minus 2^(c-1), in [-2^(c-1), 2^(c-1))
struct Biased {
  uint32_t b[9];
  __device__ __forceinline__ Biased(const uint32_t s[8], const uint32_t off[9]) {
    uint32_t carry = 0;
#pragma unroll
    for (int l = 0; l < 9; l++) {
      const uint64_t t = (uint64_t)(l < 8 ? s[l] : 0u) + off[l] + carry;
      b[l] = (uint32_t)t;
      carry = (uint32_t)(t >> 32);
    }
  }
  __device__ __forceinline__ int digit(int w, int c) const {
    const int bit = w * c, limb = bit >> 5, sh = bit & 31;
    uint64_t two = 0;
#pragma unroll
    for (int l = 0; l < 9; l++) {  // b[limb] | b[limb+1] << 32 without dynamic register indexing
      if (l == limb) two |= b[l];
      if (l == limb + 1) two |= (uint64_t)b[l] << 32;
    }
    return (int)((two >> sh) & ((1u << c) - 1u)) - (1 << (c - 1));
  }
};
struct BiasOff {
  uint32_t v[9];
};

}  // namespace

// ---------------------------------------------------------------------------------------------- 1. prep
__global__ void __launch_bounds__(256)
    msm_prep_kernel(const fq_t* bases_ark, const fr_t* scalars_mont, size_t n, size_t n_pool, pt_niels* niels, fr_t* canon,
                    unsigned* max_bits) {
  unsigned mb = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t j = n_pool ? i % n_pool : i;  // bench inputs: a pool of distinct points tiled to n terms
    stn(niels + i, niels_from_ark_affine(ld_fq(bases_ark + 2 * j), ld_fq(bases_ark + 2 * j + 1)));
    const fr_t c = fr_to_canonical(ld_fr(scalars_mont + i));
    st_fr(canon + i, c);
    unsigned b = 0;
#pragma unroll
    for (int l = 0; l < 8; l++)
      if (c.v[l]) b = 32 * l + (32 - __clz(c.v[l]));
    mb = b > mb ? b : mb;
  }
  mb = __reduce_max_sync(0xffffffffu, mb);
  if ((threadIdx.x & 31) == 0 && mb) atomicMax(max_bits, mb);
}

// ---------------------------------------------------------------------------------------------- 2. histogram
__global__ void __launch_bounds__(256)
    msm_hist_kernel(const fr_t* canon, size_t n, int c, int nw, uint32_t NB1, BiasOff off, uint32_t* cnt) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t s = ld_fr(canon + i);
    const Biased bs(s.v, off.v);
    for (int w = 0; w < nw; w++) {
      const int d = bs.digit(w, c);
      if (d) atomicAdd(cnt + (size_t)w * NB1 + (uint32_t)(d < 0 ? -d : d), 1u);
    }
  }
}

// ---------------------------------------------------------------------------------------------- 3. scan
// off[i] = sum_{j < i} cnt[j], uoff[i] = sum_{j < i} units(cnt[j]) with units(x) = ceil(x / S).  Three small kernels:
// tiles of 4096 counters scanned by one CTA each (coalesced), the tile sums scanned by one CTA, the tile offsets added.
// totals[0] = number of entries, totals[1] = number of units, totals[2] = number of multi-unit buckets (filled later).
static constexpr uint32_t kScanTile = 4096;
__global__ void __launch_bounds__(1024)
    msm_scan_tiles_kernel(const uint32_t* cnt, uint32_t total, uint32_t S, uint32_t* off, uint32_t* uoff, uint2* tile_sums) {
  __shared__ uint32_t w1[32], w2[32];
  const uint32_t t = threadIdx.x, base = blockIdx.x * kScanTile + t * 4;
  uint32_t x[4], a = 0, b = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    x[k] = base + k < total ? cnt[base + k] : 0u;
    a += x[k];
    b += (x[k] + S - 1) / S;
  }
  // inclusive scan of (a, b) over the 1024 threads: warp shuffles, then the 32 warp totals
  uint32_t ia = a, ib = b;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, d), tb = __shfl_up_sync(0xffffffffu, ib, d);
    if ((t & 31) >= (uint32_t)d) {
      ia += ta;
      ib += tb;
    }
  }
  if ((t & 31) == 31) {
    w1[t >> 5] = ia;
    w2[t >> 5] = ib;
  }
  __syncthreads();
  if (t < 32) {
    uint32_t va = w1[t], vb = w2[t];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t ta = __shfl_up_sync(0xffffffffu, va, d), tb = __shfl_up_sync(0xffffffffu, vb, d);
      if (t >= (uint32_t)d) {
        va += ta;
        vb += tb;
      }
    }
    w1[t] = va;
    w2[t] = vb;
  }
  __syncthreads();
  const uint32_t wa = (t >> 5) ? w1[(t >> 5) - 1] : 0u, wb = (t >> 5) ? w2[(t >> 5) - 1] : 0u;
  uint32_t r1 = wa + ia - a, r2 = wb + ib - b;  // exclusive prefix inside the tile
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (base + k < total) {
      off[base + k] = r1;
      uoff[base + k] = r2;
    }
    r1 += x[k];
    r2 += (x[k] + S - 1) / S;
  }
  if (t == 1023) tile_sums[blockIdx.x] = make_uint2(w1[31], w2[31]);
}
__global__ void __launch_bounds__(1024)
    msm_scan_sums_kernel(uint2* tile_sums, uint32_t ntiles, uint32_t total, uint32_t* off, uint32_t* uoff, uint32_t* totals) {
  __shared__ uint32_t s1[1024], s2[1024];
  const uint32_t t = threadIdx.x;
  uint32_t carry1 = 0, carry2 = 0;
  for (uint32_t base = 0; base < ntiles; base += 1024) {  // ntiles <= 1024 in practice: one pass
    const uint2 v = base + t < ntiles ? tile_sums[base + t] : make_uint2(0u, 0u);
    s1[t] = v.x;
    s2[t] = v.y;
    __syncthreads();
    for (uint32_t d = 1; d < 1024; d <<= 1) {
      uint32_t x1 = 0, x2 = 0;
      if (t >= d) {
        x1 = s1[t - d];
        x2 = s2[t - d];
      }
      __syncthreads();
      s1[t] += x1;
      s2[t] += x2;
      __syncthreads();
    }
    if (base + t < ntiles) tile_sums[base + t] = make_uint2(carry1 + s1[t] - v.x, carry2 + s2[t] - v.y);  // exclusive
    carry1 += s1[1023];
    carry2 += s2[1023];
    __syncthreads();
  }
  if (t == 0) {
    off[total] = carry1;
    uoff[total] = carry2;
    totals[0] = carry1;
    totals[1] = carry2;
  }
}
__global__ void __launch_bounds__(1024)
    msm_scan_apply_kernel(const uint2* tile_sums, uint32_t total, uint32_t* off, uint32_t* uoff) {
  const uint2 o = tile_sums[blockIdx.x];
  const uint32_t base = blockIdx.x * kScanTile + threadIdx.x * 4;
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (base + k < total) {
      off[base + k] += o.x;
      uoff[base + k] += o.y;
    }
}
// unit -> bucket map; buckets split into several units are also listed (multi, totals[2]) for the combine kernel
__global__ void __launch_bounds__(256)
    msm_unit_map_kernel(const uint32_t* uoff, uint32_t total, uint32_t* unit_bucket, uint32_t* multi, uint32_t* totals) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const uint32_t u0 = uoff[i], u1 = uoff[i + 1];
  for (uint32_t u = u0; u < u1; u++) unit_bucket[u] = i;
  if (u1 - u0 > 1) multi[atomicAdd(totals + 2, 1u)] = i;
}

// ---------------------------------------------------------------------------------------------- 4. scatter
// blockIdx.y = window: the CTAs of one window run together, its slice of `entries` (n x 4 B) stays in L2
__global__ void __launch_bounds__(256)
    msm_scatter_kernel(const fr_t* canon, size_t n, int c, uint32_t NB1, BiasOff off, const uint32_t* boff, uint32_t* fill,
                       uint32_t* entries) {
  const int w = blockIdx.y;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t s = ld_fr(canon + i);
    const Biased bs(s.v, off.v);
    const int d = bs.digit(w, c);
    if (d) {
      const size_t bi = (size_t)w * NB1 + (uint32_t)(d < 0 ? -d : d);
      const uint32_t pos = boff[bi] + atomicAdd(fill + bi, 1u);
      entries[pos] = (uint32_t)i | (d < 0 ? 0x80000000u : 0u);
    }
  }
}

// ---------------------------------------------------------------------------------------------- 5. accumulate
__global__ void __launch_bounds__(128)
    msm_accum_kernel(const pt_niels* niels, const uint32_t* entries, const uint32_t* cnt, const uint32_t* boff,
                     const uint32_t* uoff, const uint32_t* unit_bucket, const uint32_t* totals, uint32_t S, pt_ext* unit_sum) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= totals[1]) return;
  const uint32_t bi = unit_bucket[u], k = u - uoff[bi];
  const uint32_t lo = boff[bi] + k * S, end = boff[bi] + cnt[bi], hi = min(end, lo + S);
  pt_ext acc = pt_identity();
  uint32_t e = entries[lo];
  pt_niels nn = ldn(niels + (e & 0x7fffffffu));
  for (uint32_t p = lo; p < hi; p++) {
    const uint32_t ecur = e;
    const pt_niels ncur = nn;
    if (p + 1 < hi) {
      e = entries[p + 1];
      nn = ldn(niels + (e & 0x7fffffffu));
    }
    acc = pt_madd(acc, (ecur & 0x80000000u) ? niels_neg(ncur) : ncur);
  }
  stp(unit_sum + u, acc);
}

// ---------------------------------------------------------------------------------------------- 6. bucket reduction
// A bucket that was split into several units (skewed scalars: e.g. the top window of 20-bit scalars has a handful of
// non-empty buckets holding all n terms) is combined here, one WARP per listed bucket: lanes stride over the units,
// then a shuffle tree; the sum replaces the bucket's first unit.  Uniform scalars: the list is empty.
__global__ void __launch_bounds__(256)
    msm_unit_combine_kernel(pt_ext* unit_sum, const uint32_t* uoff, const uint32_t* multi, const uint32_t* totals) {
  const uint32_t nmulti = totals[2];
  const int lane = threadIdx.x & 31;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < nmulti; m += nwarps) {
    const uint32_t bi = multi[m];
    const uint32_t u0 = uoff[bi], u1 = uoff[bi + 1];
    pt_ext acc = pt_identity();
    bool any = false;
    for (uint32_t u = u0 + lane; u < u1; u += 32) {
      const pt_ext p = ldp(unit_sum + u);
      acc = any ? pt_add(acc, p) : p;
      any = true;
    }
#pragma unroll 1
    for (int d = 16; d >= 1; d >>= 1) {
      pt_ext o;
#pragma unroll
      for (int l = 0; l < 8; l++) {
        o.X.v[l] = __shfl_down_sync(0xffffffffu, acc.X.v[l], d);
        o.Y.v[l] = __shfl_down_sync(0xffffffffu, acc.Y.v[l], d);
        o.Z.v[l] = __shfl_down_sync(0xffffffffu, acc.Z.v[l], d);
        o.T.v[l] = __shfl_down_sync(0xffffffffu, acc.T.v[l], d);
      }
      acc = pt_add(acc, o);
    }
    if (lane == 0) stp(unit_sum + u0, acc);
  }
}
// B_b of (window w, bucket b): its first unit (the whole bucket after msm_unit_combine_kernel)
__device__ __forceinline__ bool bucket_sum(const pt_ext* unit_sum, const uint32_t* uoff, size_t bi, pt_ext& out) {
  const uint32_t u0 = uoff[bi], u1 = uoff[bi + 1];
  if (u0 == u1) return false;
  out = ldp(unit_sum + u0);
  return true;
}
// sum_b b * B_b per window by the reference's running sums (msm/mod.rs:139-145), applied recursively so that no
// thread walks more than L items:
//   level 0: thread (w, t) walks the buckets t*L+1 .. t*L+L: run = sum B, acc = sum j * B_{tL+j}
//            => W = sum_t acc_t + L * Y_1,  Y_1 = sum_t t * run_t                      (a weighted sum again, 0-based)
//   level k: thread (w, u) walks the items u*L .. u*L+L-1 of level k-1's `run`: the same with 0-based weights
//   ... until one item is left:  W = A_0 + L_0 (A_1 + L_1 (A_2 + ...)),  A_k = the plain sum of level k's `acc`.
__global__ void __launch_bounds__(128)
    msm_wsum_kernel(const pt_ext* unit_sum, const uint32_t* uoff, uint32_t NB1, const pt_ext* in_run, int level, int nw,
                    uint32_t n_in, uint32_t L, pt_ext* out_run, pt_ext* out_acc) {
  const uint32_t n_out = n_in / L, id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (uint32_t)nw * n_out) return;
  const uint32_t w = id / n_out, t = id - w * n_out;
  pt_ext run = pt_identity(), acc = pt_identity();
  bool any = false;
  for (uint32_t jj = L; jj >= 1; jj--) {
    const uint32_t j = jj - 1;  // item t*L + j, weight j + 1 at level 0 (buckets are 1-based), j above
    pt_ext B;
    bool have;
    if (level == 0) {
      have = bucket_sum(unit_sum, uoff, (size_t)w * NB1 + (size_t)t * L + j + 1, B);
    } else {
      B = ldp(in_run + (size_t)w * n_in + (size_t)t * L + j);
      have = true;
    }
    if (have) {
      run = any ? pt_add(run, B) : B;
      any = true;
    }
    if (any && (level == 0 || j > 0)) acc = pt_add(acc, run);
  }
  stp(out_run + id, run);
  stp(out_acc + id, acc);
}
// shared-memory point storage (SoA): element (coord c, limb l) of point idx at base[(c*8 + l) * n + idx]
__device__ __forceinline__ void sm_st(uint32_t* base, int n, int idx, const pt_ext& p) {
#pragma unroll
  for (int l = 0; l < 8; l++) {
    base[(0 * 8 + l) * n + idx] = p.X.v[l];
    base[(1 * 8 + l) * n + idx] = p.Y.v[l];
    base[(2 * 8 + l) * n + idx] = p.Z.v[l];
    base[(3 * 8 + l) * n + idx] = p.T.v[l];
  }
}
__device__ __forceinline__ pt_ext sm_ld(const uint32_t* base, int n, int idx) {
  pt_ext p;
#pragma unroll
  for (int l = 0; l < 8; l++) {
    p.X.v[l] = base[(0 * 8 + l) * n + idx];
    p.Y.v[l] = base[(1 * 8 + l) * n + idx];
    p.Z.v[l] = base[(2 * 8 + l) * n + idx];
    p.T.v[l] = base[(3 * 8 + l) * n + idx];
  }
  return p;
}
// A[w][k] = the plain sum of level k's acc[w][0 .. n_k): CTA (w, k), 256 threads + shared-memory tree
struct MsmLevels {
  const pt_ext* acc[8];
  uint32_t n[8];
};
__global__ void __launch_bounds__(256) msm_psum_kernel(MsmLevels lv, int nlev, pt_ext* A) {
  __shared__ uint32_t buf[32 * 256];
  const int w = blockIdx.x, k = blockIdx.y, tid = threadIdx.x;
  const pt_ext* src = lv.acc[k] + (size_t)w * lv.n[k];
  pt_ext acc = pt_identity();
  bool any = false;
  for (uint32_t i = tid; i < lv.n[k]; i += 256) {
    const pt_ext p = ldp(src + i);
    acc = any ? pt_add(acc, p) : p;
    any = true;
  }
  sm_st(buf, 256, tid, acc);
  __syncthreads();
  for (int d = 128; d >= 1; d >>= 1) {
    if (tid < d) {
      acc = pt_add(acc, sm_ld(buf, 256, tid + d));
      sm_st(buf, 256, tid, acc);
    }
    __syncthreads();
  }
  if (tid == 0) stp(A + (size_t)w * nlev + k, acc);
}
// ---------------------------------------------------------------------------------------------- 7. final
// msm_final.cu (its own translation unit: a single warp walks ~250 dependent doublings there, and wants the field
// multiplication inlined instead of the out-of-line calls that keep the big kernels of this file small)
// ---------------------------------------------------------------------------------------------- naive cross-check
// An independent evaluation of the same sum for the parity tests at sizes the CPU oracle cannot reach: every term
// by plain double-and-add over the bits of its canonical scalar (no digits, no buckets, no tables), then a tree sum.
__global__ void __launch_bounds__(128)
    msm_naive_terms_kernel(const fq_t* bases_ark, const fr_t* scalars_mont, size_t n, size_t n_pool, pt_ext* partial) {
  __shared__ uint32_t buf[32 * 128];
  pt_ext acc = pt_identity();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t j = n_pool ? i % n_pool : i;
    const pt_niels b = niels_from_ark_affine(ld_fq(bases_ark + 2 * j), ld_fq(bases_ark + 2 * j + 1));
    const fr_t s = fr_to_canonical(ld_fr(scalars_mont + i));
    pt_ext t = pt_identity();
    int top = -1;
    for (int l = 7; l >= 0 && top < 0; l--)
      if (s.v[l]) top = 32 * l + 31 - __clz(s.v[l]);
    for (int bit = top; bit >= 0; bit--) {
      t = pt_dbl(t);
      if ((s.v[bit >> 5] >> (bit & 31)) & 1u) t = pt_madd(t, b);
    }
    acc = pt_add(acc, t);
  }
  sm_st(buf, 128, threadIdx.x, acc);
  __syncthreads();
  for (int d = 64; d >= 1; d >>= 1) {
    if ((int)threadIdx.x < d) {
      acc = pt_add(acc, sm_ld(buf, 128, threadIdx.x + d));
      sm_st(buf, 128, threadIdx.x, acc);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) stp(partial + blockIdx.x, acc);
}
__global__ void __launch_bounds__(128) msm_naive_sum_kernel(const pt_ext* partial, int count, fq_t* out_ext) {
  __shared__ uint32_t buf[32 * 128];
  pt_ext acc = pt_identity();
  for (int i = threadIdx.x; i < count; i += blockDim.x) acc = pt_add(acc, ldp(partial + i));
  sm_st(buf, 128, threadIdx.x, acc);
  __syncthreads();
  for (int d = 64; d >= 1; d >>= 1) {
    if ((int)threadIdx.x < d) {
      acc = pt_add(acc, sm_ld(buf, 128, threadIdx.x + d));
      sm_st(buf, 128, threadIdx.x, acc);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    fq_t x, y;
    pt_to_affine_canonical(acc, x, y);
    out_ext[0] = fq_to_ark(x);
    out_ext[1] = fq_to_ark(y);
    out_ext[2] = fq_to_ark(fq_mul(x, y));
    out_ext[3] = fq_to_ark(fq_one());
  }
}
void launch_msm_naive(const fq_t* bases_ark, const fr_t* scalars_mont, size_t n, size_t n_pool, pt_ext* partial /* kNumSMs * 8 */,
                      fq_t* out_ext, cudaStream_t st) {
  const int blocks = kNumSMs * 8;
  launch(msm_naive_terms_kernel, blocks, 128, 0, st, bases_ark, scalars_mont, n, n_pool, partial);
  launch(msm_naive_sum_kernel, 1, 128, 0, st, partial, blocks, out_ext);
}

// ---------------------------------------------------------------------------------------------- host side
int msm_large_window_bits(size_t n) {
  // the reference's rule is c = floor(log2(n) * 0.69) + 2 (msm/mod.rs:112-116, 322-325): 13 at 2^16, 17 at 2^22, 19 at 2^26;
  // here the bucket reduction's serial chains cap it at 17
  int lg = 0;
  while (((size_t)1 << (lg + 1)) <= n) lg++;
  int c = (int)(lg * 0.69) + 2;
  if (c < 8) c = 8;
  if (c > 17) c = 17;
  return c;
}
MsmLargePlan msm_large_plan(size_t n, unsigned max_bits, int c_force) {
  MsmLargePlan p;
  p.n = n;
  p.nbits = max_bits < 1 ? 1 : (int)max_bits;
  if (c_force != 0 && (c_force < 2 || c_force > 20)) throw std::runtime_error("msm_large: forced window width outside 2..20");
  p.c = c_force ? c_force : msm_large_window_bits(n);
  if (p.c > p.nbits + 1) p.c = p.nbits + 1 < 2 ? 2 : p.nbits + 1;  // small scalars: one window holds them
  p.nw = (p.nbits + 2 + p.c - 1) / p.c;                             // c nw >= nbits + 2  =>  s + bias < 2^(c nw)
  if (p.nw > 32) throw std::runtime_error("msm_large: more than 32 windows");
  if (p.c * p.nw > 9 * 32 - 1) throw std::runtime_error("msm_large: biased scalar wider than 9 limbs");
  p.NB = 1u << (p.c - 1);
  p.NB1 = p.NB + 1;
  // reduction levels: groups of (up to) 16 items until one is left
  p.nlev = 0;
  p.level_pts = 0;
  for (uint32_t items = p.NB; items > 1;) {
    const uint32_t L = items >= 16 ? 16 : items;
    if (p.nlev >= 8) throw std::runtime_error("msm_large: too many reduction levels");
    p.lev_L[p.nlev] = L;
    p.lev_n[p.nlev] = items / L;
    p.level_pts += items / L;
    items /= L;
    p.nlev++;
  }
  const size_t avg = (n + p.NB - 1) / p.NB;
  p.S = (uint32_t)std::max<size_t>(64, 4 * avg);
  p.total = (uint32_t)p.nw * p.NB1;
  p.max_entries = n * (size_t)p.nw;
  if (p.max_entries >= ((size_t)1 << 32) || n >= ((size_t)1 << 31)) throw std::runtime_error("msm_large: too many terms");
  p.max_units = (size_t)p.total + p.max_entries / p.S + 1;
  return p;
}
size_t msm_large_scratch_bytes(const MsmLargePlan& p) {
  size_t b = 0;
  b += 5 * (((size_t)p.total + 1) * 4 + 256);  // cnt, fill, off, uoff, multi
  b += ((size_t)p.total / kScanTile + 2) * 8 + 256 + 64;  // tile sums, totals
  b += p.max_entries * 4 + 256;                // entries
  b += p.max_units * 4 + 256;                  // unit_bucket
  b += p.max_units * sizeof(pt_ext) + 256;     // unit_sum
  b += 2 * (size_t)p.nw * p.level_pts * sizeof(pt_ext) + 512;  // run / acc of every level
  b += (size_t)p.nw * 8 * sizeof(pt_ext) + 256;                // A
  return b + 4096;
}
void msm_large_init_device() {}
void launch_msm_large_prep(const fq_t* bases_ark, const fr_t* scalars_mont, size_t n, size_t n_pool, pt_niels* niels,
                           fr_t* canon, unsigned* d_max_bits, cudaStream_t st) {
  size_t b = (n + 255) / 256;
  if (b > (size_t)kNumSMs * 8) b = kNumSMs * 8;
  launch(msm_prep_kernel, (unsigned)b, 256, 0, st, bases_ark, scalars_mont, n, n_pool, niels, canon, d_max_bits);
}
// scratch: msm_large_scratch_bytes(plan) bytes.  Outputs (either may be null): out_ext = (x, y, t, z = 1) arkworks
// limbs; out_raw = un-normalised (X, Y, Z, T) internal limbs (for the cross-GPU gather-then-add).
void launch_msm_large(const MsmLargePlan& p, const pt_niels* niels, const fr_t* canon, void* scratch, fq_t* out_ext,
                      uint32_t* out_raw, cudaStream_t st) {
  uint8_t* s = (uint8_t*)scratch;
  auto take = [&](size_t bytes) {
    uint8_t* r = s;
    s += (bytes + 255) & ~(size_t)255;
    return r;
  };
  const uint32_t ntiles = (p.total + kScanTile - 1) / kScanTile;
  uint32_t* cnt = (uint32_t*)take(((size_t)p.total + 1) * 4);
  uint32_t* fill = (uint32_t*)take(((size_t)p.total + 1) * 4);
  uint32_t* off = (uint32_t*)take(((size_t)p.total + 1) * 4);
  uint32_t* uoff = (uint32_t*)take(((size_t)p.total + 1) * 4);
  uint32_t* multi = (uint32_t*)take(((size_t)p.total + 1) * 4);
  uint2* tile_sums = (uint2*)take(((size_t)ntiles + 1) * 8);
  uint32_t* totals = (uint32_t*)take(16);
  uint32_t* entries = (uint32_t*)take(p.max_entries * 4);
  uint32_t* unit_bucket = (uint32_t*)take(p.max_units * 4);
  pt_ext* unit_sum = (pt_ext*)take(p.max_units * sizeof(pt_ext));
  pt_ext* lev_run = (pt_ext*)take((size_t)p.nw * p.level_pts * sizeof(pt_ext));
  pt_ext* lev_acc = (pt_ext*)take((size_t)p.nw * p.level_pts * sizeof(pt_ext));
  pt_ext* A = (pt_ext*)take((size_t)p.nw * 8 * sizeof(pt_ext));
  BiasOff bo;  // sum_{w < nw} 2^(c-1) * 2^(c w)
  for (int l = 0; l < 9; l++) bo.v[l] = 0;
  for (int w = 0; w < p.nw; w++) {
    const int bit = w * p.c + p.c - 1;
    bo.v[bit >> 5] |= 1u << (bit & 31);
  }
  LB_CUDA_CHECK(cudaMemsetAsync(cnt, 0, ((size_t)p.total + 1) * 4, st));
  LB_CUDA_CHECK(cudaMemsetAsync(fill, 0, ((size_t)p.total + 1) * 4, st));
  LB_CUDA_CHECK(cudaMemsetAsync(totals, 0, 16, st));
  size_t b = (p.n + 255) / 256;
  if (b > (size_t)kNumSMs * 8) b = kNumSMs * 8;
  launch(msm_hist_kernel, (unsigned)b, 256, 0, st, canon, p.n, p.c, p.nw, p.NB1, bo, cnt);
  launch(msm_scan_tiles_kernel, ntiles, 1024, 0, st, cnt, p.total, p.S, off, uoff, tile_sums);
  launch(msm_scan_sums_kernel, 1, 1024, 0, st, tile_sums, ntiles, p.total, off, uoff, totals);
  launch(msm_scan_apply_kernel, ntiles, 1024, 0, st, tile_sums, p.total, off, uoff);
  launch(msm_unit_map_kernel, (p.total + 255) / 256, 256, 0, st, uoff, p.total, unit_bucket, multi, totals);
  {
    size_t bx = (p.n + 255) / 256;
    if (bx > (size_t)kNumSMs * 4) bx = kNumSMs * 4;
    dim3 grid((unsigned)bx, (unsigned)p.nw);
    launch(msm_scatter_kernel, grid, 256, 0, st, canon, p.n, p.c, p.NB1, bo, off, fill, entries);
  }
  launch(msm_accum_kernel, (unsigned)((p.max_units + 127) / 128), 128, 0, st, niels, entries, cnt, off, uoff,
         unit_bucket, totals, p.S, unit_sum);
  launch(msm_unit_combine_kernel, kNumSMs * 4, 256, 0, st, unit_sum, uoff, multi, totals);
  // bucket reduction, level by level
  MsmLevels lv;
  struct {
    int v[8];
  } lg;
  size_t pts_off = 0;
  const pt_ext* prev_run = nullptr;
  uint32_t items = p.NB;
  for (int k = 0; k < p.nlev; k++) {
    const uint32_t L = p.lev_L[k], n_out = p.lev_n[k];
    pt_ext* run_k = lev_run + (size_t)p.nw * pts_off;
    pt_ext* acc_k = lev_acc + (size_t)p.nw * pts_off;
    launch(msm_wsum_kernel, (unsigned)(((size_t)p.nw * n_out + 127) / 128), 128, 0, st, unit_sum, uoff, p.NB1,
           prev_run, k, p.nw, items, L, run_k, acc_k);
    lv.acc[k] = acc_k;
    lv.n[k] = n_out;
    lg.v[k] = 0;
    while ((1u << lg.v[k]) < L) lg.v[k]++;
    prev_run = run_k;
    pts_off += n_out;
    items = n_out;
  }
  for (int k = p.nlev; k < 8; k++) {
    lv.acc[k] = nullptr;
    lv.n[k] = 0;
    lg.v[k] = 0;
  }
  {
    dim3 grid((unsigned)p.nw, (unsigned)p.nlev);
    launch(msm_psum_kernel, grid, 256, 0, st, lv, p.nlev, A);
  }
  launch_msm_final(A, p.nlev, lg.v, p.nw, p.c, out_ext, out_raw, st);
}

}  // namespace lb
