// lasso_b200 — K6: Pippenger bucket MSM over curve25519 on sm_90a, row-batched with shared
// bases.  Replaces src/msm/mod.rs:91-164 (msm_bigint_wnaf) and its callers
// src/poly/commitments.rs:84-93 (batch_commit) / src/poly/dense_mlpoly.rs:109-128 (commit_inner:
// L_size independent row MSMs over the same R_size generators).
//
// Shape of the work (SURVEY §7 "MSM shape"): thousands of independent rows of 2^9..2^14 terms over
// the SAME generators, mostly tiny scalars — not one giant MSM.  So:
//   * fixed window c = 8 with signed digits d in [-128, 127] via the offset trick
//     (s + 0x80..80, then byte w minus 128): digits are independent per window, no carry chain;
//   * the generators are expanded once into a table T[w][j] = 2^(8w) G_j in affine-niels form
//     (96 B/point), so every window of a row lands in ONE bucket set and no doublings are needed;
//   * one CTA per (row, column-chunk), ALL windows: counting sort of the chunk's (column, window)
//     digits in shared memory, then every thread adds an equal-sized contiguous slice of the sorted
//     list (robust against skewed digits, e.g. 0/1-valued LT tables), split buckets are stitched by
//     a segmented log-step reduction, and the weighted bucket sum  sum_b b*B_b  is a suffix scan +
//     tree reduction over the 128 buckets — once per CTA, not once per window;
//   * a finish kernel adds the per-chunk partials of a row, normalises (one Fq inversion per row)
//     and emits arkworks-layout points + compressed bytes.
// For bases without a precomputed table (variable-base lasso_msm) the same kernels run with the
// single window-0 table, one CTA per (window, row, chunk), and the finish kernel does the 8-doubling
// Horner combination instead.
// Integer-ALU bound (7 Fq muls per bucket add), not HBM bound: reported as point-adds/s.
#if defined(__CUDACC__)
#define LB_FQ_MUL_ATTR static __host__ __device__ __noinline__
#define LB_FQ_MUL_BYVALUE
#endif
#include "kernels.cuh"
#include "msm.cuh"
#include "quad.cuh"

namespace lb {

static constexpr int MSM_T = 128;        // threads per CTA = number of buckets
static constexpr int MSM_NB = 128;       // buckets 1..128 (|d|)
static constexpr int MSM_CHUNK = 8192;   // max columns per CTA

// ---------------------------------------------------------------- shared-memory point storage (SoA)
// element (coord c, limb l) of point idx lives at base[(c*8 + l) * n + idx] -> conflict-free
__device__ __forceinline__ void sm_store_pt(uint32_t* base, int n, int idx, const pt_ext& p) {
#pragma unroll
  for (int l = 0; l < 8; l++) {
    base[(0 * 8 + l) * n + idx] = p.X.v[l];
    base[(1 * 8 + l) * n + idx] = p.Y.v[l];
    base[(2 * 8 + l) * n + idx] = p.Z.v[l];
    base[(3 * 8 + l) * n + idx] = p.T.v[l];
  }
}
__device__ __forceinline__ pt_ext sm_load_pt(const uint32_t* base, int n, int idx) {
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
__device__ __forceinline__ pt_niels ld_niels(const pt_niels* p) {
  pt_niels n;
  n.yplusx = ld_fq(&p->yplusx);
  n.yminusx = ld_fq(&p->yminusx);
  n.t2d = ld_fq(&p->t2d);
  return n;
}
__device__ __forceinline__ void st_niels(pt_niels* p, const pt_niels& n) {
  st_fq(&p->yplusx, n.yplusx);
  st_fq(&p->yminusx, n.yminusx);
  st_fq(&p->t2d, n.t2d);
}

// ---------------------------------------------------------------- generator tables
__global__ void __launch_bounds__(128) table_first_kernel(const fq_t* bases_ark /*n x (x,y)*/, size_t n, pt_niels* T) {
  size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  st_niels(T + j, niels_from_ark_affine(ld_fq(bases_ark + 2 * j), ld_fq(bases_ark + 2 * j + 1)));
}
// T[w][j] = 2^8 * T[w-1][j], renormalised to affine-niels
__global__ void __launch_bounds__(128) table_next_kernel(pt_niels* T, size_t n, size_t stride, int w) {
  size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  pt_ext p = pt_from_niels(ld_niels(T + (size_t)(w - 1) * stride + j));
#pragma unroll 1
  for (int k = 0; k < 8; k++) p = pt_dbl(p);
  fq_t zi = fq_inv(p.Z);
  st_niels(T + (size_t)w * stride + j, niels_from_affine(fq_mul(p.X, zi), fq_mul(p.Y, zi)));
}
void launch_build_table(const fq_t* bases_ark, size_t n, pt_niels* T, size_t stride, int nwindows, cudaStream_t st) {
  unsigned blocks = (unsigned)((n + 127) / 128);
  launch(table_first_kernel, blocks, 128, 0, st, bases_ark, n, T);
  for (int w = 1; w < nwindows; w++) launch(table_next_kernel, blocks, 128, 0, st, T, n, stride, w);
}

// ---------------------------------------------------------------- scalars
// Montgomery Fr -> canonical integer (into_bigint, msm/mod.rs:23-25) + max bit length of the batch
__global__ void __launch_bounds__(256) canonicalize_kernel(const fr_t* in, fr_t* out, size_t n, unsigned* max_bits) {
  unsigned mb = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    fr_t c = fr_to_canonical(ld_fr(in + i));
    st_fr(out + i, c);
    unsigned b = 0;
#pragma unroll
    for (int l = 0; l < 8; l++)
      if (c.v[l]) b = 32 * l + (32 - __clz(c.v[l]));
    mb = b > mb ? b : mb;
  }
  mb = __reduce_max_sync(0xffffffffu, mb);
  if ((threadIdx.x & 31) == 0 && mb) atomicMax(max_bits, mb);
}
void launch_canonicalize(const fr_t* in, fr_t* out, size_t n, unsigned* d_max_bits, cudaStream_t st) {
  size_t b = (n + 255) / 256;
  if (b > (size_t)kNumSMs * 8) b = kNumSMs * 8;
  if (b == 0) return;
  launch(canonicalize_kernel, (unsigned)b, 256, 0, st, in, out, n, d_max_bits);
}

// signed digits (c = 8): byte w of (s + 0x80..80) minus 128.  MsmDigits biases the scalar once; digit(w) with a
// compile-time w (the window loops are fully unrolled) is a shift and a mask.
template <int SL>
struct MsmDigits;
template <>
struct MsmDigits<1> {
  static constexpr int kMaxWindows = 5;
  uint64_t v;
  __device__ __forceinline__ explicit MsmDigits(const uint32_t* s) : v((uint64_t)s[0] + 0x8080808080ull) {}
  __device__ __forceinline__ int digit(int w) const { return (int)((v >> (8 * w)) & 0xff) - 128; }
};
template <>
struct MsmDigits<8> {
  static constexpr int kMaxWindows = 32;
  uint32_t b[8];
  __device__ __forceinline__ explicit MsmDigits(const uint32_t* s) {
    uint32_t carry = 0;
#pragma unroll
    for (int l = 0; l < 8; l++) {
      uint64_t t = (uint64_t)s[l] + 0x80808080u + carry;
      b[l] = (uint32_t)t;
      carry = (uint32_t)(t >> 32);
    }
  }
  __device__ __forceinline__ int digit(int w) const { return (int)((b[w >> 2] >> (8 * (w & 3))) & 0xff) - 128; }
};

// ---------------------------------------------------------------- the bucket kernel
struct MsmSmem {
  int cnt[MSM_NB + 2];
  int off[MSM_NB + 2];
  int cur[MSM_NB + 2];
  int pf_b[MSM_T], pl_b[MSM_T];
  uint16_t list[MSM_CHUNK];
  uint32_t bucket[32 * (MSM_NB + 1)];  // SoA, index 0 unused (digit 0)
  uint32_t pfirst[32 * MSM_T];
  uint32_t plast[32 * MSM_T];
};

template <int SL>
__global__ void __launch_bounds__(MSM_T)
    msm_bucket_kernel(const pt_niels* table, size_t table_stride, int shifted, const uint32_t* scalars,
                      size_t row_stride /*in scalars*/, int ncols, int chunk_cols, int nw, int wpc, int col_mul,
                      int col_add, pt_ext* partials) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MsmSmem& sm = *reinterpret_cast<MsmSmem*>(smem_raw);
  // this CTA: windows [w0, w1) of the columns [c_begin, c_end) of `row`.  With a shifted table every window
  // has the same bucket weights, so all of them share ONE bucket set (wpc = nw): one weighted bucket sum per
  // CTA instead of one per window.  Without it (variable-base) wpc = 1 and the finish kernel does the Horner.
  const int wg = blockIdx.x, row = blockIdx.y, chunk = blockIdx.z, tid = threadIdx.x;
  const int w0 = wg * wpc, w1 = min(nw, w0 + wpc), nwin = w1 - w0;
  const int c_begin = chunk * chunk_cols;
  const int c_end = min(ncols, c_begin + chunk_cols);
  const size_t wstride = shifted ? table_stride : 0;
  const pt_niels* tw = table + (size_t)w0 * wstride;
  const uint32_t* srow = scalars + ((size_t)row * row_stride) * SL;
  constexpr int MAXW = MsmDigits<SL>::kMaxWindows;

  for (int b = tid; b < MSM_NB + 2; b += MSM_T) sm.cnt[b] = 0;
  sm.pf_b[tid] = 0;
  sm.pl_b[tid] = 0;
  __syncthreads();
  // pass 1: histogram of |digit|
  for (int c = c_begin + tid; c < c_end; c += MSM_T) {
    uint32_t s[SL];
#pragma unroll
    for (int l = 0; l < SL; l++) s[l] = srow[(size_t)c * SL + l];
    const MsmDigits<SL> dg(s);
#pragma unroll
    for (int w = 0; w < MAXW; w++) {
      if (w >= w0 && w < w1) {
        int d = dg.digit(w);
        if (d) atomicAdd(&sm.cnt[d < 0 ? -d : d], 1);
      }
    }
  }
  __syncthreads();
  // exclusive scan over buckets 1..128 (one warp, 4 buckets per lane)
  if (tid < 32) {
    int v[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      v[k] = sm.cnt[1 + tid * 4 + k];
      sum += v[k];
    }
    int incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (tid >= d) incl += t;
    }
    int run = incl - sum;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      sm.off[1 + tid * 4 + k] = run;
      sm.cur[1 + tid * 4 + k] = run;
      run += v[k];
    }
    if (tid == 31) sm.off[MSM_NB + 1] = run;
  }
  // every bucket starts as the identity
  sm_store_pt(sm.bucket, MSM_NB + 1, tid + 1, pt_identity());
  __syncthreads();
  const int N = sm.off[MSM_NB + 1];
  if (N == 0) {
    if (tid == 0) partials[((size_t)row * gridDim.x + wg) * gridDim.z + chunk] = pt_identity();
    return;
  }
  // pass 2: scatter ((column-in-chunk * nwin + window-in-group) | sign) into the sorted list
  for (int c = c_begin + tid; c < c_end; c += MSM_T) {
    uint32_t s[SL];
#pragma unroll
    for (int l = 0; l < SL; l++) s[l] = srow[(size_t)c * SL + l];
    const MsmDigits<SL> dg(s);
#pragma unroll
    for (int w = 0; w < MAXW; w++) {
      if (w >= w0 && w < w1) {
        int d = dg.digit(w);
        if (d) {
          int pos = atomicAdd(&sm.cur[d < 0 ? -d : d], 1);
          sm.list[pos] = (uint16_t)(((c - c_begin) * nwin + (w - w0)) | (d < 0 ? 0x8000 : 0));
        }
      }
    }
  }
  __syncthreads();
  // accumulate: thread t owns the contiguous slice [lo, hi) of the sorted list.  ONE flat loop over the
  // slice (every lane of the warp executes the same number of point additions); a change of bucket only
  // triggers a short, predicated flush.  (Looping run by run made the warp pay max-over-lanes per run.)
  // Slices: N >= T -> equal shares; N < T -> the first N threads take one entry each, so that the threads
  // holding entries are always a contiguous range (the stitch below relies on it).
  auto slice_lo = [&](int t) { return N >= MSM_T ? (int)(((long long)t * N) / MSM_T) : min(t, N); };
  {
    const int lo = slice_lo(tid), hi = slice_lo(tid + 1);
    if (lo < hi) {
      int b;  // bucket containing position lo: largest b with off[b] <= lo
      {
        int l = 1, r = MSM_NB;
        while (l < r) {
          int m = (l + r + 1) >> 1;
          if (sm.off[m] <= lo) l = m; else r = m - 1;
        }
        b = l;
      }
      while (sm.off[b + 1] <= lo) b++;  // skip empty buckets that share the offset
      auto flush = [&](int bb, int start, int end, const pt_ext& acc) {
        const bool complete = (start == sm.off[bb]) && (end == sm.off[bb + 1]);
        if (complete) {
          sm_store_pt(sm.bucket, MSM_NB + 1, bb, acc);
        } else if (start == lo) {
          sm_store_pt(sm.pfirst, MSM_T, tid, acc);
          sm.pf_b[tid] = bb;
        } else {
          sm_store_pt(sm.plast, MSM_T, tid, acc);
          sm.pl_b[tid] = bb;
        }
      };
      pt_ext acc = pt_identity();
      int run_start = lo;
      // software pipeline: the next point's 96 B are in flight while the current addition runs.
      // local column c -> generator index c * col_mul + col_add (col_mul = #GPUs when one proof is sharded
      // by the low index bits: this rank owns the columns congruent to its rank)
      auto entry_ptr = [&](uint16_t ee) {
        const int idx = ee & 0x7fff, cl = idx / nwin, wl = idx - cl * nwin;
        return tw + (size_t)wl * wstride + (size_t)(c_begin + cl) * col_mul + col_add;
      };
      uint16_t e = sm.list[lo];
      pt_niels nn = ld_niels(entry_ptr(e));
      for (int p = lo; p < hi; p++) {
        const uint16_t ecur = e;
        const pt_niels ncur = nn;
        if (p + 1 < hi) {
          e = sm.list[p + 1];
          nn = ld_niels(entry_ptr(e));
        }
        if (p >= sm.off[b + 1]) {  // the bucket is exhausted (it received >= 1 point): flush, move on
          flush(b, run_start, p, acc);
          acc = pt_identity();
          run_start = p;
          do { b++; } while (sm.off[b + 1] <= p);
        }
        // P - Q = P + (-Q): negating an affine-niels point is a swap and one negation
        acc = pt_madd(acc, (ecur & 0x8000) ? niels_neg(ncur) : ncur);
      }
      flush(b, run_start, hi, acc);
    }
  }
  // stitch partial runs into their buckets.  A bucket that is not wholly inside one thread's slice was split
  // over a CONTIGUOUS range of threads [t_lo, t_hi]: t_lo holds its tail partial (plast) for the bucket — or a
  // head partial if the bucket starts exactly at its slice — and every later thread of the range a head
  // partial (pfirst).  Step 1: segmented suffix reduction of the head partials keyed by bucket (log steps,
  // stops as soon as no run is longer than the stride: one step for uniform digits, 7 for a window whose
  // digits all fall into one bucket — a serial walk there cost up to 127 additions on one lane while the
  // other warps waited at the barrier).  Step 2: the owner of a bucket adds <= 2 values.
  __syncthreads();
  {
    const int myk = sm.pf_b[tid];  // written by this thread (or 0)
    pt_ext mine;
    if (myk) mine = sm_load_pt(sm.pfirst, MSM_T, tid);
    for (int d = 1; d < MSM_T; d <<= 1) {
      const bool work = myk && (tid + d < MSM_T) && sm.pf_b[tid + d] == myk;
      if (!__syncthreads_or(work)) break;  // barrier: the previous step's stores are visible
      pt_ext other;
      if (work) other = sm_load_pt(sm.pfirst, MSM_T, tid + d);
      __syncthreads();
      if (work) {
        mine = pt_add(mine, other);
        sm_store_pt(sm.pfirst, MSM_T, tid, mine);
      }
    }
    // (loop exit is always through a barrier or after the last step's store: sync before the owners read)
    __syncthreads();
    const int b = tid + 1;
    const int s0 = sm.off[b], s1 = sm.off[b + 1];
    if (s1 > s0) {
      auto thread_of = [&](int pos) {
        if (N < MSM_T) return pos;
        int t = (int)(((long long)pos * MSM_T) / N);
        if (t > MSM_T - 1) t = MSM_T - 1;
        while (t + 1 < MSM_T && slice_lo(t + 1) <= pos) t++;
        while (t > 0 && slice_lo(t) > pos) t--;
        return t;
      };
      const int t_lo = thread_of(s0), t_hi = thread_of(s1 - 1);
      if (t_lo != t_hi) {
        const bool has_l = sm.pl_b[t_lo] == b;
        const int t_f = t_lo + (has_l ? 1 : 0);
        const bool has_f = t_f <= t_hi && sm.pf_b[t_f] == b;
        pt_ext acc = has_l ? sm_load_pt(sm.plast, MSM_T, t_lo) : sm_load_pt(sm.pfirst, MSM_T, t_f);
        if (has_l && has_f) acc = pt_add(acc, sm_load_pt(sm.pfirst, MSM_T, t_f));
        sm_store_pt(sm.bucket, MSM_NB + 1, b, acc);
      }
    }
  }
  __syncthreads();
  // weighted sum  sum_b b * B_b = sum_{k>=1} (sum_{b>=k} B_b): suffix scan, then tree reduction.
  // Reuse pfirst as the ping-pong buffer.
  {
    const int b = tid + 1;
    pt_ext mine = sm_load_pt(sm.bucket, MSM_NB + 1, b);
    uint32_t* bufA = sm.bucket;  // stride MSM_NB+1, index b
    uint32_t* bufB = sm.pfirst;  // stride MSM_T, index tid
    bool inA = true;
    for (int d = 1; d < MSM_NB; d <<= 1) {
      pt_ext other;
      bool has = (tid + d) < MSM_NB;
      if (has) other = inA ? sm_load_pt(bufA, MSM_NB + 1, b + d) : sm_load_pt(bufB, MSM_T, tid + d);
      if (has) mine = pt_add(mine, other);
      if (inA) sm_store_pt(bufB, MSM_T, tid, mine); else sm_store_pt(bufA, MSM_NB + 1, b, mine);
      inA = !inA;
      __syncthreads();
    }
    // `mine` = suffix sum S_b; now sum all S_b
    for (int d = MSM_NB / 2; d >= 1; d >>= 1) {
      pt_ext other;
      bool act = tid < d;
      if (act) other = inA ? sm_load_pt(bufA, MSM_NB + 1, b + d) : sm_load_pt(bufB, MSM_T, tid + d);
      if (act) mine = pt_add(mine, other);
      if (inA) sm_store_pt(bufB, MSM_T, tid, mine); else sm_store_pt(bufA, MSM_NB + 1, b, mine);
      inA = !inA;
      __syncthreads();
    }
    if (tid == 0) partials[((size_t)row * gridDim.x + wg) * gridDim.z + chunk] = mine;
  }
}

// ---------------------------------------------------------------- finish: combine, normalise, emit
__device__ __forceinline__ pt_ext shfl_down_pt(const pt_ext& p, int d) {
  pt_ext r;
#pragma unroll
  for (int l = 0; l < 8; l++) {
    r.X.v[l] = __shfl_down_sync(0xffffffffu, p.X.v[l], d);
    r.Y.v[l] = __shfl_down_sync(0xffffffffu, p.Y.v[l], d);
    r.Z.v[l] = __shfl_down_sync(0xffffffffu, p.Z.v[l], d);
    r.T.v[l] = __shfl_down_sync(0xffffffffu, p.T.v[l], d);
  }
  return r;
}
__device__ __forceinline__ pt_ext ld_pt(const pt_ext* p) {
  pt_ext r;
  r.X = ld_fq(&p->X);
  r.Y = ld_fq(&p->Y);
  r.Z = ld_fq(&p->Z);
  r.T = ld_fq(&p->T);
  return r;
}
// One warp per row.  out_ext: (x,y,t,z=1) arkworks Montgomery limbs; out_comp: 32 B compressed;
// out_raw: un-normalised (X, Y, Z, T) internal limbs, 128 B/row — for host-side normalisation (a couple of
// rows: one inversion is a 265-step serial chain) or for the cross-GPU gather-then-add of partial points.
__global__ void __launch_bounds__(256)
    msm_finish_kernel(const pt_ext* partials, int nrows, int nw, int nchunks, int shifted, fq_t* out_ext,
                      uint32_t* out_comp, uint32_t* out_raw) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row < nrows) {
    const pt_ext* p = partials + (size_t)row * nw * nchunks;
    pt_ext acc = pt_identity();
    if (shifted) {
      const int total = nw * nchunks;
      for (int i = lane; i < total; i += 32) acc = pt_add(acc, ld_pt(p + i));
      if (total > 1) {
#pragma unroll 1
        for (int d = 16; d >= 1; d >>= 1) {
          pt_ext o = shfl_down_pt(acc, d);
          acc = pt_add(acc, o);
        }
      }
    } else if (lane == 0) {
      // msm/mod.rs:150-163: total = sum_w 2^(8w) W_w, high to low with 8 doublings per window
      for (int w = nw - 1; w >= 0; w--) {
        if (w != nw - 1)
          for (int k = 0; k < 8; k++) acc = pt_dbl(acc);
        for (int c = 0; c < nchunks; c++) acc = pt_add(acc, ld_pt(p + (size_t)w * nchunks + c));
      }
    }
    if (lane == 0) {
      if (out_raw) {
#pragma unroll
        for (int l = 0; l < 8; l++) {
          out_raw[(size_t)row * 32 + l] = acc.X.v[l];
          out_raw[(size_t)row * 32 + 8 + l] = acc.Y.v[l];
          out_raw[(size_t)row * 32 + 16 + l] = acc.Z.v[l];
          out_raw[(size_t)row * 32 + 24 + l] = acc.T.v[l];
        }
      }
      if (out_comp || out_ext) {
        fq_t x, y;
        pt_to_affine_canonical(acc, x, y);
        if (out_comp) {
          uint32_t c[8];
          pt_compress_canonical(x, y, c);
#pragma unroll
          for (int l = 0; l < 8; l++) out_comp[(size_t)row * 8 + l] = c[l];
        }
        if (out_ext) {
          fq_t one = fq_one();
          out_ext[(size_t)row * 4 + 0] = fq_to_ark(x);
          out_ext[(size_t)row * 4 + 1] = fq_to_ark(y);
          out_ext[(size_t)row * 4 + 2] = fq_to_ark(fq_mul(x, y));
          out_ext[(size_t)row * 4 + 3] = fq_to_ark(one);
        }
      }
    }
  }
}

// Finish for a handful of rows over a shifted table (the rounds of the opening proofs): ONE CTA, 32 quads
// per row; each quad adds its share of the row's partials, then a 5-level tree through shared memory.
// The result (X, Y, Z canonical) goes to mapped host memory as a tagged message (common.cuh PubDst): no flag,
// no system fence.
__global__ void __launch_bounds__(1024)
    msm_finish_quad_kernel(const pt_ext* partials, int nrows, int P, PubDst pub) {
  __shared__ fq_t sm_pt[8 * 32 * 4];
  const int tid = threadIdx.x, lane = tid & 31, role = tid & 3;
  const int row = tid >> 7, qr = (tid & 127) >> 2;  // blockDim = 128 * nrows
  const fq_t* prow = reinterpret_cast<const fq_t*>(partials + (size_t)row * P);
  fq_t mine = (role == 1 || role == 2) ? fq_one() : fq_zero();  // identity (0, 1, 1, 0)
  for (int i0 = 0; i0 < P; i0 += 32) {  // uniform trip count: the quad shuffles use the full-warp mask
    const int i = i0 + qr;
    if (i0 == 0) {
      if (i < P) mine = ld_fq(prow + 4 * (size_t)i + role);
    } else {
      fq_t r = quad_add(0xffffffffu, lane, mine, prow + 4 * (size_t)(i < P ? i : 0));
      if (i < P) mine = r;
    }
  }
  fq_t* slot = sm_pt + ((size_t)row * 32 + qr) * 4;
  slot[role] = mine;
  __syncthreads();
  for (int d = 16; d >= 1; d >>= 1) {
    fq_t r = mine;
    if (qr < d) r = quad_add(d >= 8 ? 0xffffffffu : (0xfu << (lane & ~3)), lane, mine, slot + 4 * d);
    __syncthreads();
    if (qr < d) {
      mine = r;
      slot[role] = mine;
    }
    __syncthreads();
  }
  if (qr == 0 && role < 3) {  // canonical coordinate < 2^255: element 3*row + {0, 1, 2} of the tagged message
    const fq_t c = fq_canonical(mine);
    pub_store(pub, row * 3 + role, c.v);
  }
}

// ---------------------------------------------------------------- bucket-free MSM over a multiples table
// The MSMs of the opening proofs are short (two rows of ~1-8 K terms) and sit on the critical path ~50 times
// per proof: the bucket method spends most of its time on the fixed 14-step weighted bucket sum.  Memory buys a
// shortcut: for the first `npts` generators (the ones the openings use) keep every digit multiple
//   M[w][j][d-1] = d * 2^(8w) * G_j,  d = 1..128, affine-niels (96 B): 32 * npts * 128 * 96 B (0.8 GB at
//   npts = 2050, the 2^20-lookup configuration),
// so a term is ONE table entry per window and the MSM is a plain sum of (terms x 32) points: quads of lanes
// (quad_add above) add ~4 entries each, a shared-memory tree adds the 128 quads of a CTA, and the quad finish
// kernel adds the CTAs of a row.  No sort, no buckets, no doublings; depth ~ 4 mixed + 7 + 7 full additions
// at quad-lane latency.
// Built once per generator set: thread (w, j) walks d = 1..128 (one mixed addition each) and normalises.
__global__ void __launch_bounds__(128)
    multiples_table_kernel(const pt_niels* T, size_t table_stride, size_t npts, int nwindows, pt_niels* M) {
  const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)nwindows * npts) return;
  const size_t w = id / npts, j = id - w * npts;
  const pt_niels base = ld_niels(T + w * table_stride + j);
  pt_niels* out = M + id * 128;
  st_niels(out, base);
  pt_ext acc = pt_from_niels(base);
  for (int d = 2; d <= 128; d++) {
    acc = pt_madd(acc, base);
    const fq_t zi = fq_inv(acc.Z);
    st_niels(out + (d - 1), niels_from_affine(fq_mul(acc.X, zi), fq_mul(acc.Y, zi)));
  }
}
void launch_build_multiples(const pt_niels* T, size_t table_stride, size_t npts, int nwindows, pt_niels* M, cudaStream_t st) {
  const size_t n = (size_t)nwindows * npts;
  launch(multiples_table_kernel, (unsigned)((n + 127) / 128), 128, 0, st, T, table_stride, npts, nwindows, M);
}

// 16-bit multiples of the COMMITMENT generators (the columns of the Hyrax matrices): M16[j][d-1] = d * G_j,
// d = 1..32768 (3 MB per generator: 12.9 GB for the 4096 columns of the 2^20-lookup configuration).  The
// committed integers (16-bit indices, counters, table values) then cost ONE table entry each instead of one per
// 8-bit digit plus a carry.  Thread (j, b) starts from (256 b) G_j = b * 2^8 G_j (an entry of M) and walks 256
// mixed additions; normalisation is batched 16 at a time (Montgomery's trick: 3 multiplications per point + one
// inversion per batch).
__global__ void __launch_bounds__(128)
    multiples16_table_kernel(const pt_niels* T, const pt_niels* M, size_t npts8, size_t ncols, size_t col_mul, size_t col_add,
                             pt_niels* M16) {
  const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= ncols * 128) return;
  const size_t jl = id >> 7, j = jl * col_mul + col_add;  // local column jl <-> generator j (sharded: this rank's columns)
  const int b = (int)(id & 127);
  const pt_niels base = ld_niels(T + j);  // window 0: G_j
  pt_ext acc = b == 0 ? pt_identity() : pt_from_niels(ld_niels(M + ((size_t)1 * npts8 + j) * 128 + (b - 1)));
  pt_niels* out = M16 + jl * 32768 + (size_t)256 * b;
  for (int g = 0; g < 16; g++) {
    pt_ext pts[16];
    fq_t pref[16];
#pragma unroll 1
    for (int k = 0; k < 16; k++) {
      acc = pt_madd(acc, base);
      pts[k] = acc;
      pref[k] = k == 0 ? acc.Z : fq_mul(pref[k - 1], acc.Z);
    }
    fq_t inv = fq_inv(pref[15]);
#pragma unroll 1
    for (int k = 15; k >= 0; k--) {
      const fq_t zi = k == 0 ? inv : fq_mul(inv, pref[k - 1]);
      inv = fq_mul(inv, pts[k].Z);
      st_niels(out + 16 * g + k, niels_from_affine(fq_mul(pts[k].X, zi), fq_mul(pts[k].Y, zi)));
    }
  }
}
void launch_build_multiples16(const pt_niels* T, const pt_niels* M, size_t npts8, size_t ncols, size_t col_mul, size_t col_add,
                              pt_niels* M16, cudaStream_t st) {
  const size_t n = ncols * 128;
  launch(multiples16_table_kernel, (unsigned)((n + 127) / 128), 128, 0, st, T, M, npts8, ncols, col_mul, col_add, M16);
}

static constexpr int MSMD_T = 512;  // 128 quads
// scalars: nrows x len canonical 256-bit integers; term k uses generator k.
// CTA (chunk, row) takes the terms k = chunk (mod nchunks): an odd nchunks spreads any power-of-two pattern of
// zero scalars evenly.  Quad (w, sub): window w of the terms chunk + nchunks * (sub + 4 i).
__global__ void __launch_bounds__(MSMD_T)
    msm_direct_kernel(const pt_niels* M, size_t npts, const uint32_t* scalars, int len, pt_ext* partials) {
  __shared__ fq_t sm_pt[128 * 4];
  const int tid = threadIdx.x, lane = tid & 31, role = tid & 3, quad = tid >> 2;
  const int w = quad & 31, sub = quad >> 5;
  const int chunk = blockIdx.x, nchunks = gridDim.x, row = blockIdx.y;
  const uint32_t* srow = scalars + (size_t)row * len * 8;
  fq_t mine = (role == 1 || role == 2) ? fq_one() : fq_zero();  // identity (0, 1, 1, 0)
  // operand of an entry for this lane; digit 0 -> the identity entry (1, 1, 0): the control flow stays uniform
  auto fetch = [&](int k, fq_t& op) -> bool {
    uint32_t sw[8];
    uint32_t any = 0;
#pragma unroll
    for (int l = 0; l < 8; l++) {
      sw[l] = srow[(size_t)k * 8 + l];
      any |= sw[l];
    }
    if (any == 0) return false;  // zero scalar: the same for the whole warp (all its quads share k)
    const MsmDigits<8> dg(sw);
    uint32_t limb = 0;
#pragma unroll
    for (int l = 0; l < 8; l++) limb = (l == (w >> 2)) ? dg.b[l] : limb;
    const int d = (int)((limb >> (8 * (w & 3))) & 0xff) - 128;
    const int ad = d < 0 ? -d : d;
    op = role == 3 ? fq_zero() : fq_one();
    if (ad != 0 && role != 2) {
      const pt_niels* e = M + ((size_t)w * npts + k) * 128 + (ad - 1);
      const bool neg = d < 0;
      if (role == 0) op = ld_fq(neg ? &e->yplusx : &e->yminusx);
      else if (role == 1) op = ld_fq(neg ? &e->yminusx : &e->yplusx);
      else {
        op = ld_fq(&e->t2d);
        if (neg) op = fq_neg(op);
      }
    }
    return true;
  };
  const int step = nchunks * 4;
  int k = chunk + nchunks * sub;
  fq_t op, op_next;
  bool have = k < len ? fetch(k, op) : false;
  while (k < len) {  // uniform per warp: its 8 quads share sub, hence k
    const int kn = k + step;
    const bool have_next = kn < len ? fetch(kn, op_next) : false;  // next entry in flight during this addition
    if (have) mine = quad_madd(0xffffffffu, lane, mine, op);
    op = op_next;
    have = have_next;
    k = kn;
  }
  // tree over the 128 quads
  fq_t* slot = sm_pt + quad * 4;
  slot[role] = mine;
  __syncthreads();
  for (int d = 64; d >= 1; d >>= 1) {
    fq_t r = mine;
    if (quad < d) r = quad_add(d >= 8 ? 0xffffffffu : (0xfu << (lane & ~3)), lane, mine, slot + 4 * d);
    __syncthreads();
    if (quad < d) {
      mine = r;
      slot[role] = mine;
    }
    __syncthreads();
  }
  if (quad == 0) {
    fq_t* out = reinterpret_cast<fq_t*>(partials + (size_t)row * nchunks + chunk);
    st_fq(out + role, mine);
  }
}
// ---------------------------------------------------------------- one Bulletproofs round in ONE launch
// bullet.rs:73-134 with unfolded generators (prover.cu file header).  The scalars, the sums of both rows and their
// publication in one launch instead of three dependent ones on the critical path of each of the ~43 rounds of a proof.
//   grid (nchunks, 2): row 0 = L, row 1 = R.  CTA (chunk, row) owns the main terms k = chunk + nchunks * q of its row:
//     k = t * h + p (h = m / 2, t < n / m):   L: generator t*m + h + p, scalar a'[p]     * w'[t]
//                                             R: generator t*m + p,     scalar a'[p + h] * w'[t]
//     a' / b' = the vectors folded with the previous challenge (bullet.rs:127-130), w' = the expanded weights.
//   phase 1: thread q forms the scalar of the CTA's q-th term in shared memory; the threads with t = 0 also own one
//            element of a', b' each (stored for the next round) and one product of c_L = <a'_lo, b'_hi> (row 0) or
//            c_R = <a'_hi, b'_lo> (row 1); the CTA's partial inner product goes to `ip_partial`.
//   phase 2: the quad-lane sum over the multiples table, exactly msm_direct_kernel's, digits read from shared memory.
//   phase 3: the LAST CTA (ticket) finishes both rows: c_L, c_R from the partial inner products, the two tail terms
//            c * Q + blind * h of each row (generators n, n + 1) as 128 more table entries — one per quad —, the
//            per-CTA partial points, a tree over its 64 quads per row, and the tagged publication of X, Y, Z.
static constexpr int kBulletMaxTerms = MSMD_T;  // main terms per CTA (one thread each in phase 1)
__global__ void __launch_bounds__(MSMD_T)
    bullet_fused_kernel(const pt_niels* M, size_t npts, const fr_t* a_in, const fr_t* b_in, const fr_t* w_in, fr_t* a_out,
                        fr_t* b_out, fr_t* w_out, int n, int m, int fold, fr_t u, fr_t uinv, fr_t blind_L, fr_t blind_R,
                        pt_ext* partials, fr_t* ip_partial, unsigned* counter, PubDst pub) {
  __shared__ fq_t sm_pt[128 * 4];
  __shared__ uint32_t s_sc[kBulletMaxTerms * 8];
  __shared__ uint32_t s_col[kBulletMaxTerms];
  __shared__ fr_t s_red[MSMD_T / 32];
  __shared__ fr_t s_tail[4];
  __shared__ int s_last;
  const int tid = threadIdx.x, lane = tid & 31, role = tid & 3, quad = tid >> 2;
  const int w = quad & 31, sub = quad >> 5;
  const int chunk = blockIdx.x, nchunks = gridDim.x, row = blockIdx.y;
  const int h = m >> 1, nmain = n >> 1;
  const int lg_h = 31 - __clz(h);  // h is a power of two (h >= 1)
  // ---- phase 1: scalars of this CTA's terms (+ fold bookkeeping)
  const int nterms = chunk < nmain ? (nmain - chunk + nchunks - 1) / nchunks : 0;
  fr_t ipv[1] = {fr_zero()};
  if (tid < nterms) {
    const int k = chunk + nchunks * tid;
    const int t = k >> lg_h, p = k & (h - 1);
    const int ia = row == 0 ? p : p + h;  // index into a' of this term's factor
    auto folded = [&](const fr_t* v, int i, const fr_t& c0, const fr_t& c1) {
      return fold ? fr_add(fr_mul(ld_fr(v + i), c0), fr_mul(c1, ld_fr(v + m + i))) : ld_fr(v + i);
    };
    const fr_t ai = folded(a_in, ia, u, uinv);
    const fr_t wt = fold ? fr_mul(ld_fr(w_in + (t >> 1)), (t & 1) ? u : uinv) : ld_fr(w_in + t);
    const fr_t sc = fr_to_canonical(fr_mul(ai, wt));
#pragma unroll
    for (int l = 0; l < 8; l++) s_sc[tid * 8 + l] = sc.v[l];
    s_col[tid] = (uint32_t)(t * m + (row == 0 ? h + p : p));
    if (t == 0) {
      // row 0 owns (a'[p], b'[p + h]) and the product of c_L; row 1 owns (a'[p + h], b'[p]) and the product of c_R
      const int ib = row == 0 ? p + h : p;
      const fr_t bi = folded(b_in, ib, uinv, u);
      if (fold) {
        st_fr(a_out + ia, ai);
        st_fr(b_out + ib, bi);
      }
      ipv[0] = fr_mul(ai, bi);
    }
    if (p == 0 && row == 1 && fold) st_fr(w_out + t, wt);
  }
  block_sum_fr<1>(ipv, s_red);
  if (tid == 0) ip_partial[row * nchunks + chunk] = ipv[0];
  __syncthreads();
  // ---- phase 2: quad (w, sub) adds window w of the terms sub, sub + 4, ...
  fq_t mine = (role == 1 || role == 2) ? fq_one() : fq_zero();  // identity (0, 1, 1, 0)
  auto operand = [&](const uint32_t* sw, uint32_t col, fq_t& op) -> bool {
    uint32_t any = 0;
#pragma unroll
    for (int l = 0; l < 8; l++) any |= sw[l];
    if (any == 0) return false;
    const MsmDigits<8> dg(sw);
    uint32_t limb = 0;
#pragma unroll
    for (int l = 0; l < 8; l++) limb = (l == (w >> 2)) ? dg.b[l] : limb;
    const int d = (int)((limb >> (8 * (w & 3))) & 0xff) - 128;
    const int ad = d < 0 ? -d : d;
    op = role == 3 ? fq_zero() : fq_one();
    if (ad != 0 && role != 2) {
      const pt_niels* e = M + ((size_t)w * npts + col) * 128 + (ad - 1);
      const bool neg = d < 0;
      if (role == 0) op = ld_fq(neg ? &e->yplusx : &e->yminusx);
      else if (role == 1) op = ld_fq(neg ? &e->yminusx : &e->yplusx);
      else {
        op = ld_fq(&e->t2d);
        if (neg) op = fq_neg(op);
      }
    }
    return true;
  };
  {
    int q = sub;
    fq_t op, op_next;
    uint32_t sw[8];
    auto fetch = [&](int qq, fq_t& o) -> bool {
#pragma unroll
      for (int l = 0; l < 8; l++) sw[l] = s_sc[qq * 8 + l];
      return operand(sw, s_col[qq], o);
    };
    bool have = q < nterms ? fetch(q, op) : false;
    while (q < nterms) {  // uniform per warp: its 8 quads share sub
      const int qn = q + 4;
      const bool have_next = qn < nterms ? fetch(qn, op_next) : false;
      if (have) mine = quad_madd(0xffffffffu, lane, mine, op);
      op = op_next;
      have = have_next;
      q = qn;
    }
  }
  fq_t* slot = sm_pt + quad * 4;
  slot[role] = mine;
  __syncthreads();
  for (int d = 64; d >= 1; d >>= 1) {
    fq_t r = mine;
    if (quad < d) r = quad_add(d >= 8 ? 0xffffffffu : (0xfu << (lane & ~3)), lane, mine, slot + 4 * d);
    __syncthreads();
    if (quad < d) {
      mine = r;
      slot[role] = mine;
    }
    __syncthreads();
  }
  if (quad == 0) {
    fq_t* out = reinterpret_cast<fq_t*>(partials + (size_t)row * nchunks + chunk);
    st_fq(out + role, mine);
  }
  // ---- ticket
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = (atomicAdd(counter, 1u) == (unsigned)(gridDim.x * gridDim.y) - 1u);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- phase 3 (last CTA): tail scalars, tail entries, row sums, publication
  {
    const int warp = tid >> 5;
    if (warp < 2) {
      fr_t v = fr_zero();
      for (int i = lane; i < nchunks; i += 32) v = fr_add(v, ld_fr_cg(ip_partial + warp * nchunks + i));
      v = warp_sum_fr(v);
      if (lane == 0) {
        s_tail[warp * 2] = fr_to_canonical(v);                                      // c_L / c_R on Q
        s_tail[warp * 2 + 1] = fr_to_canonical(warp == 0 ? blind_L : blind_R);      // blind on h
      }
    }
  }
  __syncthreads();
  const int prow = quad >> 6, pq = quad & 63;  // 64 quads per row
  {
    // quad pq of a row: tail term (pq >> 5) of that row, window pq & 31 — one table entry
    const int term = pq >> 5;
    fq_t op;
    mine = (role == 1 || role == 2) ? fq_one() : fq_zero();
    // (w == pq & 31 == quad & 31 holds: the window used by `operand` is this quad's)
    if (operand(s_tail[prow * 2 + term].v, (uint32_t)(n + term), op)) mine = quad_madd(0xffffffffu, lane, mine, op);
  }
  {
    const fq_t* prow_p = reinterpret_cast<const fq_t*>(partials + (size_t)prow * nchunks);
    for (int i0 = 0; i0 < nchunks; i0 += 64) {  // uniform trip count: full-warp shuffles inside
      const int i = i0 + pq;
      fq_t q4[4];
      const bool ok = i < nchunks;
      if (ok) {
        const fq_t* src = prow_p + 4 * (size_t)i;
#pragma unroll
        for (int k = 0; k < 4; k++) {  // written by other CTAs of this launch: bypass L1
          asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
                       : "=r"(q4[k].v[0]), "=r"(q4[k].v[1]), "=r"(q4[k].v[2]), "=r"(q4[k].v[3]) : "l"(src + k));
          asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
                       : "=r"(q4[k].v[4]), "=r"(q4[k].v[5]), "=r"(q4[k].v[6]), "=r"(q4[k].v[7]) : "l"((const char*)(src + k) + 16));
        }
      } else {  // identity
        q4[0] = fq_zero();
        q4[1] = fq_one();
        q4[2] = fq_one();
        q4[3] = fq_zero();
      }
      const fq_t r = quad_add(0xffffffffu, lane, mine, q4);
      if (ok) mine = r;
    }
  }
  slot[role] = mine;
  __syncthreads();
  for (int d = 32; d >= 1; d >>= 1) {  // tree inside each row: quads prow*64 + [0, 64)
    fq_t r = mine;
    if (pq < d) r = quad_add(d >= 8 ? 0xffffffffu : (0xfu << (lane & ~3)), lane, mine, slot + 4 * d);
    __syncthreads();
    if (pq < d) {
      mine = r;
      slot[role] = mine;
    }
    __syncthreads();
  }
  if (pq == 0 && role < 3) {
    const fq_t c = fq_canonical(mine);
    pub_store(pub, prow * 3 + role, c.v);
  }
  if (tid == 0) *counter = 0;
}
// chunks of the fused round: as msm_direct_chunks for two heavy rows, and few enough that a CTA's main terms fit
// its phase-1 threads
int bullet_fused_chunks(int n) {
  int c = msm_direct_chunks(n / 2 + 2, 2);
  while ((n / 2 + c - 1) / c > kBulletMaxTerms) c += 2;
  return c;
}
void launch_bullet_fused(const pt_niels* M, size_t npts, const fr_t* a_in, const fr_t* b_in, const fr_t* w_in, fr_t* a_out,
                         fr_t* b_out, fr_t* w_out, size_t n, size_t m, int fold, const fr_t& u, const fr_t& uinv,
                         const fr_t& blind_L, const fr_t& blind_R, pt_ext* partials, fr_t* ip_partial, unsigned* counter,
                         const PubDst& pub, cudaStream_t st) {
  if (m < 2 || n < m) throw std::runtime_error("bullet_fused: m >= 2");
  dim3 grid(bullet_fused_chunks((int)n), 2);
  launch(bullet_fused_kernel, grid, MSMD_T, 0, st, M, npts, a_in, b_in, w_in, a_out, b_out, w_out, (int)n, (int)m, fold,
         u, uinv, blind_L, blind_R, partials, ip_partial, counter, pub);
}

// two short MSMs over the multiples table; the points go to mapped host memory (msm_finish_quad_kernel)
int msm_direct_chunks(int len, int heavy_rows) {
  int c = (len * kMsmFullWindows + 128 * 4 - 1) / (128 * 4);  // ~4 entries per quad
  if (heavy_rows < 1) heavy_rows = 1;
  const int cap = (kNumSMs / heavy_rows - 1) | 1;  // about one CTA per SM over the rows that carry the work; odd
  if (c > cap) c = cap;
  if (c < 1) c = 1;
  return c | 1;
}
void launch_msm_direct(const pt_niels* M, size_t npts, const uint32_t* scalars, int len, pt_ext* partials, const PubDst& pub,
                       cudaStream_t st) {
  const int nrows = 2, nchunks = msm_direct_chunks(len, 1);
  dim3 grid(nchunks, nrows);
  launch(msm_direct_kernel, grid, MSMD_T, 0, st, M, npts, scalars, len, partials);
  launch(msm_finish_quad_kernel, 1, 128 * nrows, 0, st, partials, nrows, nchunks, pub);
}

// ---------------------------------------------------------------- Hyrax row commitments over the multiples table
// Integer-valued polynomials (indices, counters, table values: u32 scalars, <= 5 windows): one CTA per row, thread
// t adds the table entries of the columns t, t+128, ... (one mixed addition per non-zero 8-bit digit, no sort, no
// buckets, no 14-step bucket reduction per CTA), then a shared-memory tree over the 128 threads.  Plain
// thread-per-point arithmetic: with thousands of rows this kernel is throughput-bound, not latency-bound.
__global__ void __launch_bounds__(MSM_T)
    msm_rows_direct_u32_kernel(const pt_niels* M, size_t npts, const pt_niels* M16, const pt_ext* K16, const uint32_t* scalars,
                               size_t row_stride, int ncols, int nw, int col_mul, int col_add, pt_ext* partials) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* buf = reinterpret_cast<uint32_t*>(smem_raw);  // SoA point storage, MSM_T points
  const int tid = threadIdx.x, row = blockIdx.x;
  const uint32_t* srow = scalars + (size_t)row * row_stride;
  pt_ext acc = pt_identity();
  uint32_t v = tid < ncols ? srow[tid] : 0u;
  for (int c = tid; c < ncols; c += MSM_T) {
    const uint32_t cur = v;
    if (c + MSM_T < ncols) v = srow[c + MSM_T];
    if (M16) {
      // centred 16-bit digit: v = (v mod 2^16 - 2^15) + 2^15 + 2^16 (v >> 16).  The 2^15 of every column adds up to
      // the constant K16 = 2^15 * sum_j G_j (added once per row below), so EVERY committed integer below 2^16 costs
      // exactly one table entry — no carry term for the upper half of the range, no divergence between lanes;
      // what is left of larger values goes through the 8-bit multiples of the windows 2.. as usual
      const int d16 = (int)(cur & 0xffffu) - 0x8000;
      const uint32_t rest = cur >> 16;
      if (d16 != 0) {
        pt_niels n = ld_niels(M16 + (size_t)c * 32768 + ((d16 < 0 ? -d16 : d16) - 1));
        acc = pt_madd(acc, d16 < 0 ? niels_neg(n) : n);
      }
      if (rest != 0) {
        const uint64_t br = (uint64_t)rest + 0x808080ull;
#pragma unroll
        for (int w = 0; w < 3; w++) {
          const int d = (int)((br >> (8 * w)) & 0xff) - 128;
          if (d != 0) {
            pt_niels n = ld_niels(M + ((size_t)(w + 2) * npts + (size_t)c * col_mul + col_add) * 128 + ((d < 0 ? -d : d) - 1));
            acc = pt_madd(acc, d < 0 ? niels_neg(n) : n);
          }
        }
      }
      continue;
    }
    if (cur == 0) continue;
    const uint64_t b = (uint64_t)cur + 0x8080808080ull;
#pragma unroll
    for (int w = 0; w < 5; w++) {
      if (w < nw) {
        const int d = (int)((b >> (8 * w)) & 0xff) - 128;
        if (d != 0) {
          const pt_niels* e = M + ((size_t)w * npts + (size_t)c * col_mul + col_add) * 128 + ((d < 0 ? -d : d) - 1);
          pt_niels n = ld_niels(e);
          acc = pt_madd(acc, d < 0 ? niels_neg(n) : n);
        }
      }
    }
  }
  sm_store_pt(buf, MSM_T, tid, acc);
  __syncthreads();
  for (int d = MSM_T / 2; d >= 1; d >>= 1) {
    if (tid < d) {
      acc = pt_add(acc, sm_load_pt(buf, MSM_T, tid + d));
      sm_store_pt(buf, MSM_T, tid, acc);
    }
    __syncthreads();
  }
  if (tid == 0) partials[row] = M16 ? pt_add(acc, ld_pt(K16)) : acc;
}
// One THREAD per row: normalise (one Fq inversion = a 265-step dependent chain whatever the row count)
// and emit.  32 rows per CTA so that the chains of a commitment spread over all SMs.
__global__ void __launch_bounds__(32)
    normalize_rows_kernel(const pt_ext* pts, int nrows, fq_t* out_ext, uint32_t* out_comp) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= nrows) return;
  const pt_ext acc = ld_pt(pts + row);
  fq_t x, y;
  pt_to_affine_canonical(acc, x, y);
  if (out_comp) {
    uint32_t c[8];
    pt_compress_canonical(x, y, c);
#pragma unroll
    for (int l = 0; l < 8; l++) out_comp[(size_t)row * 8 + l] = c[l];
  }
  if (out_ext) {
    out_ext[(size_t)row * 4 + 0] = fq_to_ark(x);
    out_ext[(size_t)row * 4 + 1] = fq_to_ark(y);
    out_ext[(size_t)row * 4 + 2] = fq_to_ark(fq_mul(x, y));
    out_ext[(size_t)row * 4 + 3] = fq_to_ark(fq_one());
  }
}
// nrows rows of u32 scalars over the generators 0 .. ncols-1 of the multiples table; outputs as launch_msm_rows
// K16 = 2^15 * sum_{j < ncols} G_j (extended): thread t adds the 2^15-multiples of its columns, tree as above
__global__ void __launch_bounds__(MSM_T) centre_constant_kernel(const pt_niels* M16, int ncols, pt_ext* K16) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* buf = reinterpret_cast<uint32_t*>(smem_raw);
  const int tid = threadIdx.x;
  pt_ext acc = pt_identity();
  for (int c = tid; c < ncols; c += MSM_T) acc = pt_madd(acc, ld_niels(M16 + (size_t)c * 32768 + 32767));
  sm_store_pt(buf, MSM_T, tid, acc);
  __syncthreads();
  for (int d = MSM_T / 2; d >= 1; d >>= 1) {
    if (tid < d) {
      acc = pt_add(acc, sm_load_pt(buf, MSM_T, tid + d));
      sm_store_pt(buf, MSM_T, tid, acc);
    }
    __syncthreads();
  }
  if (tid == 0) *K16 = acc;
}
void launch_centre_constant(const pt_niels* M16, int ncols, pt_ext* K16, cudaStream_t st) {
  launch(centre_constant_kernel, 1, MSM_T, 32 * MSM_T * sizeof(uint32_t), st, M16, ncols, K16);
}
void launch_msm_rows_direct_u32(const pt_niels* M, size_t npts, const pt_niels* M16, const pt_ext* K16, const uint32_t* scalars,
                                size_t row_stride, int nrows, int ncols, int nw, int col_mul, int col_add, pt_ext* partials,
                                fq_t* out_ext, uint32_t* out_comp, uint32_t* out_raw, cudaStream_t st) {
  if (nrows <= 0) return;
  if (nw < 1) nw = 1;
  if (nw > 5) throw std::runtime_error("msm_rows_direct_u32: more than 5 windows");
  launch(msm_rows_direct_u32_kernel, nrows, MSM_T, 32 * MSM_T * sizeof(uint32_t), st, M, npts, M16, K16, scalars,
         row_stride, ncols, nw, col_mul, col_add, partials);
  if (out_raw)
    launch(msm_finish_kernel, nrows, 32, 0, st, partials, nrows, 1, 1, 1, out_ext, out_comp, out_raw);
  else
    launch(normalize_rows_kernel, (nrows + 31) / 32, 32, 0, st, partials, nrows, out_ext, out_comp);
}

// Field-valued polynomials (a caller's table of arbitrary field elements): as msm_rows_direct_u32_kernel, but the
// scalars are Montgomery Fr elements, made canonical in registers, and cut into nw signed 8-bit digits by the offset
// trick over 256 bits: b = v + sum_{w < nw} 128 * 2^(8w), digit w = byte w of b - 128.  Exact when b < 2^(8 nw), so
// for every v below 2^(8 nw - 2) (msm_windows_for_bits); 2^(8 nw - 1) - 1 would carry out of the top window.
// One running 256-bit shift walks the digits, so the loop body (one mixed addition) exists once, whatever nw.
__global__ void __launch_bounds__(MSM_T)
    msm_rows_direct_fr_kernel(const pt_niels* M, size_t npts, const fr_t* scalars, size_t row_stride, int ncols, int nw,
                              int col_mul, int col_add, pt_ext* partials) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* buf = reinterpret_cast<uint32_t*>(smem_raw);  // SoA point storage, MSM_T points
  const int tid = threadIdx.x, row = blockIdx.x;
  const fr_t* srow = scalars + (size_t)row * row_stride;
  uint32_t off[8];  // the offset: 0x80 in each of the nw low bytes
#pragma unroll
  for (int l = 0; l < 8; l++) {
    const int nb = nw - 4 * l;  // bytes of this word below the top window
    off[l] = nb >= 4 ? 0x80808080u : (nb <= 0 ? 0u : 0x80808080u >> (8 * (4 - nb)));
  }
  pt_ext acc = pt_identity();
  for (int c = tid; c < ncols; c += MSM_T) {
    const fr_t x = ld_fr(srow + c);
    if (fr_is_zero(x)) continue;
    const fr_t v = fr_to_canonical(x);
    uint32_t b[8];
    uint64_t carry = 0;
#pragma unroll
    for (int l = 0; l < 8; l++) {
      const uint64_t t = (uint64_t)v.v[l] + off[l] + carry;
      b[l] = (uint32_t)t;
      carry = t >> 32;
    }
    const pt_niels* mc = M + ((size_t)c * col_mul + col_add) * 128;
    for (int w = 0; w < nw; w++) {
      const int d = (int)(b[0] & 0xffu) - 128;
      if (d != 0) {
        pt_niels n = ld_niels(mc + (size_t)w * npts * 128 + ((d < 0 ? -d : d) - 1));
        acc = pt_madd(acc, d < 0 ? niels_neg(n) : n);
      }
#pragma unroll
      for (int l = 0; l < 7; l++) b[l] = __funnelshift_r(b[l], b[l + 1], 8);
      b[7] >>= 8;
    }
  }
  sm_store_pt(buf, MSM_T, tid, acc);
  __syncthreads();
  for (int d = MSM_T / 2; d >= 1; d >>= 1) {
    if (tid < d) {
      acc = pt_add(acc, sm_load_pt(buf, MSM_T, tid + d));
      sm_store_pt(buf, MSM_T, tid, acc);
    }
    __syncthreads();
  }
  if (tid == 0) partials[row] = acc;
}
void launch_msm_rows_direct_fr(const pt_niels* M, size_t npts, const fr_t* scalars, size_t row_stride, int nrows, int ncols,
                               int nw, int col_mul, int col_add, pt_ext* partials, fq_t* out_ext, uint32_t* out_comp,
                               uint32_t* out_raw, cudaStream_t st) {
  if (nrows <= 0) return;
  if (nw < 1 || nw > kMsmFullWindows) throw std::runtime_error("msm_rows_direct_fr: nw must be in 1..32");
  launch(msm_rows_direct_fr_kernel, nrows, MSM_T, 32 * MSM_T * sizeof(uint32_t), st, M, npts, scalars, row_stride, ncols,
         nw, col_mul, col_add, partials);
  if (out_raw)
    launch(msm_finish_kernel, nrows, 32, 0, st, partials, nrows, 1, 1, 1, out_ext, out_comp, out_raw);
  else
    launch(normalize_rows_kernel, (nrows + 31) / 32, 32, 0, st, partials, nrows, out_ext, out_comp);
}

// Launch geometry.  wpc = windows per CTA (all of them over a shifted table), ngroups = window groups,
// chunk_cols = columns per CTA: at most MSM_CHUNK list entries (columns x windows) per CTA; with only a few
// rows (Bulletproofs rounds) the columns are split further so that about one CTA per SM exists.
struct MsmGeom {
  int wpc, ngroups, chunk_cols, nchunks;
};
static MsmGeom msm_geometry(int nrows, int ncols, int nw, int shifted) {
  MsmGeom g;
  g.wpc = shifted ? nw : 1;
  g.ngroups = (nw + g.wpc - 1) / g.wpc;
  int cap = MSM_CHUNK / g.wpc;  // columns whose digits fit the sorted list
  if (cap < 1) cap = 1;
  long long ctas = (long long)nrows * g.ngroups;
  int want = (int)((1LL * kNumSMs + ctas - 1) / ctas);  // chunks needed for ~1 CTA per SM
  int chunk = want > 1 ? (ncols + want - 1) / want : ncols;
  int floor_cols = 1024 / g.wpc;  // keep >= ~1k entries per CTA: the bucket reduction is a fixed 14 steps
  if (floor_cols < 8) floor_cols = 8;
  if (chunk < floor_cols) chunk = floor_cols;
  if (chunk > cap) chunk = cap;
  if (chunk > ncols) chunk = ncols;
  if (chunk < 1) chunk = 1;
  g.chunk_cols = chunk;
  g.nchunks = (ncols + chunk - 1) / chunk;
  if (g.nchunks < 1) g.nchunks = 1;
  return g;
}
size_t msm_partials_count(int nrows, int ncols, int nw) {  // upper bound over both table kinds
  if (nw < 1) nw = 1;
  MsmGeom a = msm_geometry(nrows, ncols, nw, 0), b = msm_geometry(nrows, ncols, nw, 1);
  size_t ca = (size_t)a.ngroups * a.nchunks, cb = (size_t)b.ngroups * b.nchunks;
  return (size_t)nrows * (ca > cb ? ca : cb);
}

// function attributes are per device: called from ctx_create for the context's device
void msm_init_device() {
  LB_CUDA_CHECK(cudaFuncSetAttribute(msm_bucket_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MsmSmem)));
  LB_CUDA_CHECK(cudaFuncSetAttribute(msm_bucket_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MsmSmem)));
}
void launch_msm_rows(const pt_niels* table, size_t table_stride, int shifted, const void* scalars, int scalar_limbs,
                     size_t row_stride, int nrows, int ncols, int nw, int col_mul, int col_add, pt_ext* partials,
                     fq_t* out_ext, uint32_t* out_comp, uint32_t* out_raw, cudaStream_t st) {
  if (nrows <= 0) return;
  if (nw < 1) nw = 1;
  const MsmGeom g = msm_geometry(nrows, ncols, nw, shifted);
  const int nchunks = g.nchunks, chunk_cols = g.chunk_cols;
  if (nchunks > 65535) throw std::runtime_error("msm_rows: too many column chunks for one launch");
  // gridDim.y is limited to 65535 rows per launch
  for (int r0 = 0; r0 < nrows; r0 += 65535) {
    int nr = nrows - r0 < 65535 ? nrows - r0 : 65535;
    dim3 grid(g.ngroups, nr, nchunks);
    pt_ext* part = partials + (size_t)r0 * g.ngroups * nchunks;
    if (scalar_limbs == 1)
      launch(msm_bucket_kernel<1>, grid, MSM_T, sizeof(MsmSmem), st,
             table, table_stride, shifted, (const uint32_t*)scalars + (size_t)r0 * row_stride, row_stride, ncols,
             chunk_cols, nw, g.wpc, col_mul, col_add, part);
    else
      launch(msm_bucket_kernel<8>, grid, MSM_T, sizeof(MsmSmem), st,
             table, table_stride, shifted, (const uint32_t*)scalars + (size_t)r0 * row_stride * 8, row_stride, ncols,
             chunk_cols, nw, g.wpc, col_mul, col_add, part);
  }
  launch(msm_finish_kernel, nrows, 32, 0, st, partials, nrows, g.ngroups, nchunks, shifted, out_ext, out_comp, out_raw);
}

// Cross-GPU "bucket-sum reduce": raw[(k * nrows + row) * 32 ..] = partial (X,Y,Z,T) of source k for `row`
// (k < nsrc: the all-gathered per-rank partials, plus optionally a replicated tail term).  One warp-lane
// per row adds the nsrc points; output raw again (few rows -> host normalisation) and/or compressed.
__global__ void __launch_bounds__(64)
    sum_raw_points_kernel(const uint32_t* raw, int nsrc, int nrows, uint32_t* out_raw, uint32_t* out_comp,
                          fq_t* out_ext) {
  int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= nrows) return;
  pt_ext acc = pt_identity();
  for (int k = 0; k < nsrc; k++) {
    const uint32_t* p = raw + ((size_t)k * nrows + row) * 32;
    pt_ext q;
#pragma unroll
    for (int l = 0; l < 8; l++) {
      q.X.v[l] = p[l];
      q.Y.v[l] = p[8 + l];
      q.Z.v[l] = p[16 + l];
      q.T.v[l] = p[24 + l];
    }
    acc = pt_add(acc, q);
  }
  if (out_raw) {
#pragma unroll
    for (int l = 0; l < 8; l++) {
      out_raw[(size_t)row * 32 + l] = acc.X.v[l];
      out_raw[(size_t)row * 32 + 8 + l] = acc.Y.v[l];
      out_raw[(size_t)row * 32 + 16 + l] = acc.Z.v[l];
      out_raw[(size_t)row * 32 + 24 + l] = acc.T.v[l];
    }
  }
  if (out_comp || out_ext) {
    fq_t x, y;
    pt_to_affine_canonical(acc, x, y);
    if (out_comp) {
      uint32_t c[8];
      pt_compress_canonical(x, y, c);
#pragma unroll
      for (int l = 0; l < 8; l++) out_comp[(size_t)row * 8 + l] = c[l];
    }
    if (out_ext) {
      out_ext[(size_t)row * 4 + 0] = fq_to_ark(x);
      out_ext[(size_t)row * 4 + 1] = fq_to_ark(y);
      out_ext[(size_t)row * 4 + 2] = fq_to_ark(fq_mul(x, y));
      out_ext[(size_t)row * 4 + 3] = fq_to_ark(fq_one());
    }
  }
}
void launch_sum_raw_points(const uint32_t* raw, int nsrc, int nrows, uint32_t* out_raw, uint32_t* out_comp, fq_t* out_ext,
                           cudaStream_t st) {
  launch(sum_raw_points_kernel, (nrows + 63) / 64, 64, 0, st, raw, nsrc, nrows, out_raw, out_comp, out_ext);
}

}  // namespace lb
