// lasso_b200 — CUDA kernels (sm_90a) for the multilinear-polynomial side of the Lasso prover
// hot path: bind (K1), sumcheck round evaluation (K2, K3), eq evals (K4), subtable
// materialisation + gather (K5), and the supporting reductions (K7).  SURVEY.md §2.2.
//
// All of these are streaming integer kernels over 32-byte field elements: one element per
// thread per pair of 128-bit loads (a warp covers 1 KiB contiguous), grid sized as a multiple of the
// 132 SMs, grid-stride loops, warp-shuffle + shared-memory reductions for partial sums.
// No tensor cores: this is 256-bit modular integer arithmetic, not a dense contraction.
#include "kernels.cuh"

namespace lb {

static constexpr int kThreads = 256;
static constexpr int kBlocksPerSM = 4;
static constexpr int kMaxBlocks = kNumSMs * kBlocksPerSM;  // 528
// bind_top launch shape, measured with tools/bind_sweep.py on 5 x 2^22 elements (GB/s of the 96 B per output), one
// H100 80GB HBM3 SXM at a 400 W power limit, CTAs per SM: 4: 2681, 5: 2617, 6: 2415.  A variant with two outputs
// per thread measured 2599 / 2302 / 2419 at the same CTA counts and was dropped.
static constexpr int kBindBlocksPerSM = 4;

static inline int grid_for(size_t n, int threads = kThreads, int max_blocks = kMaxBlocks) {
  size_t b = (n + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > (size_t)max_blocks) b = max_blocks;
  return (int)b;
}
int sumcheck_max_blocks() { return kMaxBlocks; }

// ------------------------------------------------------------------------------------ K1
// dense_mlpoly.rs:209-216 — algorithmic traffic 96 B per output element, 1 modmul.
__global__ void __launch_bounds__(kThreads) bind_top_kernel(fr_t* base, size_t stride, size_t half, fr_t r) {
  fr_t* Z = base + (size_t)blockIdx.y * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fr_t lo = ld_fr_stream(Z + i), hi = ld_fr_stream(Z + half + i);
    st_fr(Z + i, fr_add(lo, fr_mul(r, fr_sub(hi, lo))));
  }
}
__global__ void __launch_bounds__(kThreads) bind_top_ptrs_kernel(fr_t* const* ptrs, size_t half, fr_t r) {
  fr_t* Z = ptrs[blockIdx.y];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fr_t lo = ld_fr_stream(Z + i), hi = ld_fr_stream(Z + half + i);
    st_fr(Z + i, fr_add(lo, fr_mul(r, fr_sub(hi, lo))));
  }
}
// out of place: dst[y][i] <- bind of src[y] (grand products over a caller's polynomials, whose buffers stay untouched)
__global__ void __launch_bounds__(kThreads) bind_ptrs_kernel(fr_t* const* src, fr_t* const* dst, size_t half, fr_t r) {
  const fr_t* Z = src[blockIdx.y];
  fr_t* out = dst[blockIdx.y];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fr_t lo = ld_fr_stream(Z + i), hi = ld_fr_stream(Z + half + i);
    st_fr(out + i, fr_add(lo, fr_mul(r, fr_sub(hi, lo))));
  }
}
// dense_mlpoly.rs:218-225
__global__ void __launch_bounds__(kThreads) bind_bot_kernel(const fr_t* Z, fr_t* out, size_t half, fr_t r) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fr_t lo = ld_fr(Z + 2 * i), hi = ld_fr(Z + 2 * i + 1);
    st_fr(out + i, fr_add(lo, fr_mul(r, fr_sub(hi, lo))));
  }
}
// experiment knob (tools/bind_sweep.py): resident CTAs per SM the grid is sized for
static int bind_env(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}
void launch_bind_top(fr_t* base, size_t stride, int npolys, size_t half, const fr_t& r, cudaStream_t st) {
  if (half == 0 || npolys == 0) return;
  static const int bps = bind_env("LASSO_B200_BIND_BLOCKS", kBindBlocksPerSM);
  int per = kNumSMs * bps / npolys;
  if (per < kNumSMs / 4) per = kNumSMs / 4;
  dim3 grid(grid_for(half, kThreads, per), npolys);
  launch(bind_top_kernel, grid, kThreads, 0, st, base, stride, half, r);
}
void launch_bind_top_ptrs(fr_t* const* d_ptrs, int npolys, size_t half, const fr_t& r, cudaStream_t st) {
  if (half == 0 || npolys == 0) return;
  int per = kMaxBlocks / npolys;
  if (per < kNumSMs / 4) per = kNumSMs / 4;
  dim3 grid(grid_for(half, kThreads, per), npolys);
  launch(bind_top_ptrs_kernel, grid, kThreads, 0, st, d_ptrs, half, r);
}
void launch_bind_ptrs(fr_t* const* d_src, fr_t* const* d_dst, int npolys, size_t half, const fr_t& r, cudaStream_t st) {
  if (half == 0 || npolys == 0) return;
  int per = kMaxBlocks / npolys;
  if (per < kNumSMs / 4) per = kNumSMs / 4;
  dim3 grid(grid_for(half, kThreads, per), npolys);
  launch(bind_ptrs_kernel, grid, kThreads, 0, st, d_src, d_dst, half, r);
}
void launch_bind_bot(const fr_t* Z, fr_t* out, size_t half, const fr_t& r, cudaStream_t st) {
  if (half == 0) return;
  launch(bind_bot_kernel, grid_for(half), kThreads, 0, st, Z, out, half, r);
}

// ------------------------------------------------------------------------------------ K4
// eq_poly.rs:21-38.  evals[i] = prod_j (bit_{l-1-j}(i) ? r_j : 1 - r_j), r[0] <-> MSB.
// Small tables by the reference's doubling recurrence inside one CTA; big tables as the outer
// product T_hi (x) T_lo: one modmul and one 32-byte write per output.
__global__ void __launch_bounds__(1024) eq_small_kernel(FrVec r, int r_off, int ell, fr_t* out) {
  // out has 2^ell entries, ell <= 12
  if (threadIdx.x == 0) out[0] = fr_one();
  __syncthreads();
  int size = 1;
  for (int j = 0; j < ell; j++) {
    fr_t rj = r.v[r_off + j];
    fr_t old[2];
    int cnt = 0;
    for (int i = threadIdx.x; i < size; i += blockDim.x) old[cnt++] = out[i];
    __syncthreads();
    cnt = 0;
    for (int i = threadIdx.x; i < size; i += blockDim.x) {
      fr_t s = old[cnt++];
      fr_t hi = fr_mul(s, rj);
      out[2 * i + 1] = hi;
      out[2 * i] = fr_sub(s, hi);
    }
    __syncthreads();
    size *= 2;
  }
}
__global__ void __launch_bounds__(kThreads) eq_outer_kernel(const fr_t* t_hi, const fr_t* t_lo, int ell_lo,
                                                            size_t n, fr_t* out) {
  size_t mask = ((size_t)1 << ell_lo) - 1;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    fr_t a = t_hi[i >> ell_lo], b = t_lo[i & mask];
    st_fr(out + i, fr_mul(a, b));
  }
}
void launch_eq_evals(const FrVec& r, int ell, fr_t* out, fr_t* scratch, cudaStream_t st) {
  if (ell <= 11) {
    launch(eq_small_kernel, 1, 1024, 0, st, r, 0, ell, out);
    return;
  }
  int ell_lo = ell / 2 > 11 ? 11 : ell / 2;
  int ell_hi = ell - ell_lo;
  if (ell_hi > 11) {
    // > 2^22 entries: the high table (2^ell_hi <= 2^17 entries) is itself an outer product.  Build it in the
    // tail of `out`, stage it in scratch (+4096) because the final pass overwrites that tail, then expand.
    fr_t* hi_tab = out + (((size_t)1 << ell) - ((size_t)1 << ell_hi));
    launch_eq_evals(r, ell_hi, hi_tab, scratch, st);
    launch(eq_small_kernel, 1, 1024, 0, st, r, ell_hi, ell_lo, scratch);
    cudaMemcpyAsync(scratch + 4096, hi_tab, sizeof(fr_t) << ell_hi, cudaMemcpyDeviceToDevice, st);
    size_t n = (size_t)1 << ell;
    launch(eq_outer_kernel, grid_for(n), kThreads, 0, st, scratch + 4096, scratch, ell_lo, n, out);
    return;
  }
  launch(eq_small_kernel, 1, 1024, 0, st, r, 0, ell_hi, scratch);
  launch(eq_small_kernel, 1, 1024, 0, st, r, ell_hi, ell_lo, scratch + 4096);
  size_t n = (size_t)1 << ell;
  launch(eq_outer_kernel, grid_for(n), kThreads, 0, st, scratch, scratch + 4096, ell_lo, n, out);
}

// ------------------------------------------------------------------------------------ partial-sum reduce
// partial: [nv][nblocks]; out[v] = sum_b partial[v][b].  One CTA per value.
__global__ void __launch_bounds__(kThreads) reduce_partials_kernel(const fr_t* partial, int nblocks, fr_t* out) {
  __shared__ fr_t scratch[kThreads / 32];
  const fr_t* p = partial + (size_t)blockIdx.x * nblocks;
  fr_t acc[1] = {fr_zero()};
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) acc[0] = fr_add(acc[0], p[i]);
  block_sum_fr<1>(acc, scratch);
  if (threadIdx.x == 0) out[blockIdx.x] = acc[0];
}

// ------------------------------------------------------------------------------------ K2
// sumcheck.rs:179-237 for the strategies whose g is linear in the E_k:
//   g(E, eq) = (sum_k 2^(k*inc) E_k) * eq      (and.rs:45-53, or.rs, xor.rs, range_check.rs:78-86)
// degree 2 -> evaluation points t = 0, 1, 2 with P(t) = lo + t (hi - lo) built incrementally.
// The weighted sum is a Horner chain of shifts (fr_mul_pow2: ~35 instructions against ~250 for a Montgomery
// multiplication), which leaves 3 multiplications per index pair and makes the big rounds HBM-bound.
// Reads 2 * 32 B per polynomial per index pair (64 B/pair/poly algorithmic).
__global__ void __launch_bounds__(kThreads)
    sc_eval_linear_kernel(const fr_t* base, size_t stride, int alpha, size_t half, int inc, Finalize fin) {
  __shared__ fr_t scratch[3 * kThreads / 32];
  fr_t acc[3] = {fr_zero(), fr_zero(), fr_zero()};
  const fr_t* eq = base + (size_t)alpha * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t* P = base + (size_t)(alpha - 1) * stride;
    fr_t c0 = ld_fr_stream(P + i), c1 = ld_fr_stream(P + half + i);
    for (int k = alpha - 2; k >= 0; k--) {
      P = base + (size_t)k * stride;
      c0 = fr_add(fr_mul_pow2(c0, inc), ld_fr_stream(P + i));
      c1 = fr_add(fr_mul_pow2(c1, inc), ld_fr_stream(P + half + i));
    }
    fr_t q0 = ld_fr_stream(eq + i), q1 = ld_fr_stream(eq + half + i);
    acc[0] = fr_add(acc[0], fr_mul(c0, q0));
    acc[1] = fr_add(acc[1], fr_mul(c1, q1));
    fr_t c2 = fr_sub(fr_dbl(c1), c0), q2 = fr_sub(fr_dbl(q1), q0);
    acc[2] = fr_add(acc[2], fr_mul(c2, q2));
  }
  block_sum_fr<3>(acc, scratch);
  finalize_block<3>(fin, acc, 0, blockIdx.x, gridDim.x, 3, gridDim.x);
}

// The bind of round j-1 (sumcheck.rs:247-253, dense_mlpoly.rs:209-216) and the evaluation of round j in ONE pass
// over the polynomials: thread i owns the four elements i, i+q, i+2q, i+3q of every polynomial (q = a quarter of
// the length before the bind), folds them to the two elements i, i+q of the bound polynomial, stores those in place
// and feeds them to round j's sums.  192 B per poly per i instead of 96 + 96 (bind) + 64 + 64 (evaluation).
// Compiled for 2 resident CTAs per SM (128 registers); the grid is one wave of those.
__global__ void __launch_bounds__(kThreads, 2)
    sc_bind_eval_linear_kernel(fr_t* base, size_t stride, int alpha, size_t q, fr_t r, int inc, Finalize fin) {
  __shared__ fr_t scratch[3 * kThreads / 32];
  fr_t acc[3] = {fr_zero(), fr_zero(), fr_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < q; i += (size_t)gridDim.x * blockDim.x) {
    fr_t c0 = fr_zero(), c1 = fr_zero();
    for (int k = alpha - 1; k >= 0; k--) {
      fr_t* P = base + (size_t)k * stride;
      const fr_t a0 = ld_fr_stream(P + i), a1 = ld_fr_stream(P + q + i);
      const fr_t a2 = ld_fr_stream(P + 2 * q + i), a3 = ld_fr_stream(P + 3 * q + i);
      const fr_t n0 = fr_add(a0, fr_mul(r, fr_sub(a2, a0))), n1 = fr_add(a1, fr_mul(r, fr_sub(a3, a1)));
      st_fr(P + i, n0);
      st_fr(P + q + i, n1);
      c0 = fr_add(fr_mul_pow2(c0, inc), n0);
      c1 = fr_add(fr_mul_pow2(c1, inc), n1);
    }
    fr_t* E = base + (size_t)alpha * stride;
    const fr_t e0 = ld_fr_stream(E + i), e1 = ld_fr_stream(E + q + i);
    const fr_t e2 = ld_fr_stream(E + 2 * q + i), e3 = ld_fr_stream(E + 3 * q + i);
    const fr_t q0 = fr_add(e0, fr_mul(r, fr_sub(e2, e0))), q1 = fr_add(e1, fr_mul(r, fr_sub(e3, e1)));
    st_fr(E + i, q0);
    st_fr(E + q + i, q1);
    acc[0] = fr_add(acc[0], fr_mul(c0, q0));
    acc[1] = fr_add(acc[1], fr_mul(c1, q1));
    const fr_t c2 = fr_sub(fr_dbl(c1), c0), q2 = fr_sub(fr_dbl(q1), q0);
    acc[2] = fr_add(acc[2], fr_mul(c2, q2));
  }
  block_sum_fr<3>(acc, scratch);
  finalize_block<3>(fin, acc, 0, blockIdx.x, gridDim.x, 3, gridDim.x);
}

// LT strategy (lt.rs:60-69): g = sum_i LT_i prod_{j<i} EQ_j, memories ordered LT_0, EQ_0, LT_1, ...
// Evaluated by Horner from the last pair, h_t <- LT_k(t) + EQ_k(t) * h_t, for all C+2 points t at once
// so only two polynomials' values are live at a time.
template <int C>
__global__ void __launch_bounds__(128)
    sc_eval_lt_kernel(const fr_t* base, size_t stride, size_t half, Finalize fin) {
  constexpr int NP = C + 2;  // degree C+1
  __shared__ fr_t scratch[NP * 128 / 32];
  fr_t acc[NP];
#pragma unroll
  for (int t = 0; t < NP; t++) acc[t] = fr_zero();
  const fr_t* eq = base + (size_t)(2 * C) * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fr_t h[NP];
#pragma unroll
    for (int t = 0; t < NP; t++) h[t] = fr_zero();
#pragma unroll 1
    for (int k = C - 1; k >= 0; k--) {
      const fr_t* PL = base + (size_t)(2 * k) * stride;
      const fr_t* PE = base + (size_t)(2 * k + 1) * stride;
      fr_t l0 = ld_fr(PL + i), l1 = ld_fr(PL + half + i);
      fr_t e0 = ld_fr(PE + i), e1 = ld_fr(PE + half + i);
      fr_t dl = fr_sub(l1, l0), de = fr_sub(e1, e0);
      fr_t cl = l0, ce = e0;
#pragma unroll
      for (int t = 0; t < NP; t++) {
        h[t] = fr_add(cl, fr_mul(ce, h[t]));
        cl = fr_add(cl, dl);
        ce = fr_add(ce, de);
      }
    }
    fr_t q0 = ld_fr(eq + i), q1 = ld_fr(eq + half + i);
    fr_t dq = fr_sub(q1, q0), cq = q0;
#pragma unroll
    for (int t = 0; t < NP; t++) {
      acc[t] = fr_add(acc[t], fr_mul(h[t], cq));
      cq = fr_add(cq, dq);
    }
  }
  block_sum_fr<NP>(acc, scratch);
  finalize_block<NP>(fin, acc, 0, blockIdx.x, gridDim.x, NP, gridDim.x);
}

// The same evaluation with TWO lanes per index pair, each forming half of the C+2 evaluation points: the live state per
// thread halves (5 running products + 5 sums instead of 10 + 10 for C = 8: 255 registers and 8 warps per SM in the
// kernel above), the two lanes of a pair load the same addresses (a warp still reads 512 contiguous bytes per array).
// Sums over the lanes of equal parity by xor-shuffles, then as block_sum_fr.
template <int C>
__global__ void __launch_bounds__(128, 3)
    sc_eval_lt2_kernel(const fr_t* base, size_t stride, size_t half, Finalize fin) {
  constexpr int NP = C + 2, HP = (NP + 1) / 2;
  __shared__ fr_t scratch[NP * 128 / 32];
  const int part = threadIdx.x & 1, t0 = part * HP, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  fr_t acc[HP];
#pragma unroll
  for (int t = 0; t < HP; t++) acc[t] = fr_zero();
  const fr_t* eq = base + (size_t)(2 * C) * stride;
  const size_t pairs_per_step = ((size_t)gridDim.x * blockDim.x) >> 1;
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 1; i < half; i += pairs_per_step) {
    fr_t h[HP];
#pragma unroll
    for (int t = 0; t < HP; t++) h[t] = fr_zero();
#pragma unroll 1
    for (int k = C - 1; k >= 0; k--) {
      const fr_t* PL = base + (size_t)(2 * k) * stride;
      const fr_t* PE = base + (size_t)(2 * k + 1) * stride;
      const fr_t l0 = ld_fr(PL + i), l1 = ld_fr(PL + half + i), e0 = ld_fr(PE + i), e1 = ld_fr(PE + half + i);
      const fr_t dl = fr_sub(l1, l0), de = fr_sub(e1, e0);
      fr_t cl = l0, ce = e0;
      if (part) {  // start at t = HP: HP additions (cheaper than a multiplication by the constant)
#pragma unroll
        for (int j = 0; j < HP; j++) {
          cl = fr_add(cl, dl);
          ce = fr_add(ce, de);
        }
      }
#pragma unroll
      for (int t = 0; t < HP; t++) {
        h[t] = fr_add(cl, fr_mul(ce, h[t]));
        cl = fr_add(cl, dl);
        ce = fr_add(ce, de);
      }
    }
    const fr_t q0 = ld_fr(eq + i), q1 = ld_fr(eq + half + i), dq = fr_sub(q1, q0);
    fr_t cq = q0;
    if (part) {
#pragma unroll
      for (int j = 0; j < HP; j++) cq = fr_add(cq, dq);
    }
#pragma unroll
    for (int t = 0; t < HP; t++) {
      acc[t] = fr_add(acc[t], fr_mul(h[t], cq));
      cq = fr_add(cq, dq);
    }
  }
  // lanes of equal parity: xor-shuffles with strides 16 .. 2; lane 0 / 1 then hold the warp's sums of the two halves
#pragma unroll
  for (int t = 0; t < HP; t++) {
    fr_t a = acc[t];
#pragma unroll
    for (int d = 16; d >= 2; d >>= 1) {
      fr_t o;
#pragma unroll
      for (int l = 0; l < 8; l++) o.v[l] = __shfl_xor_sync(0xffffffffu, a.v[l], d);
      a = fr_add(a, o);
    }
    if (lane < 2 && t0 + t < NP) scratch[(t0 + t) * nwarps + warp] = a;
  }
  __syncthreads();
  fr_t vals[NP];
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NP; k++) {
      const fr_t x = lane < nwarps ? scratch[k * nwarps + lane] : fr_zero();
      vals[k] = warp_sum_fr(x);
    }
  }
  __syncthreads();
  finalize_block<NP>(fin, vals, 0, blockIdx.x, gridDim.x, NP, gridDim.x);
}

// Any other C (the reference is generic in C, lt.rs:13-14): the C+2 evaluation points are processed TB at a time so
// the live state stays in registers whatever C is; every pass re-reads the polynomials (a fallback, not a hot path).
// tv.v[t] = F::from(t).
template <int TB>
__global__ void __launch_bounds__(128)
    sc_eval_lt_generic_kernel(const fr_t* base, size_t stride, size_t half, int C, FrVec tv, Finalize fin) {
  __shared__ fr_t scratch[TB * 128 / 32];
  __shared__ fr_t res[32];
  __shared__ int s_last;
  const int NP = C + 2;
  const fr_t* eq = base + (size_t)(2 * C) * stride;
  for (int t0 = 0; t0 < NP; t0 += TB) {
    fr_t acc[TB];
#pragma unroll
    for (int t = 0; t < TB; t++) acc[t] = fr_zero();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
      fr_t h[TB];
#pragma unroll
      for (int t = 0; t < TB; t++) h[t] = fr_zero();
#pragma unroll 1
      for (int k = C - 1; k >= 0; k--) {
        const fr_t* PL = base + (size_t)(2 * k) * stride;
        const fr_t* PE = base + (size_t)(2 * k + 1) * stride;
        const fr_t l0 = ld_fr(PL + i), l1 = ld_fr(PL + half + i), e0 = ld_fr(PE + i), e1 = ld_fr(PE + half + i);
        const fr_t dl = fr_sub(l1, l0), de = fr_sub(e1, e0);
        fr_t cl = fr_add(l0, fr_mul(tv.v[t0], dl)), ce = fr_add(e0, fr_mul(tv.v[t0], de));
#pragma unroll
        for (int t = 0; t < TB; t++) {
          h[t] = fr_add(cl, fr_mul(ce, h[t]));
          cl = fr_add(cl, dl);
          ce = fr_add(ce, de);
        }
      }
      const fr_t q0 = ld_fr(eq + i), q1 = ld_fr(eq + half + i), dq = fr_sub(q1, q0);
      fr_t cq = fr_add(q0, fr_mul(tv.v[t0], dq));
#pragma unroll
      for (int t = 0; t < TB; t++) {
        acc[t] = fr_add(acc[t], fr_mul(h[t], cq));
        cq = fr_add(cq, dq);
      }
    }
    block_sum_fr<TB>(acc, scratch);
    if (threadIdx.x == 0) {
#pragma unroll
      for (int t = 0; t < TB; t++)
        if (t0 + t < NP) res[t0 + t] = acc[t];
    }
    __syncthreads();
  }
  if (gridDim.x == 1) {
    if ((int)threadIdx.x < NP) finalize_publish(fin, threadIdx.x, res[threadIdx.x]);
    return;
  }
  if ((int)threadIdx.x < NP) fin.partial[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = res[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(fin.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  finalize_last_stage(fin, gridDim.x, NP);
}

// ------------------------------------------------------------------------------------ K2/K7 for custom strategies
// combine_lookups is a straight-line program (CustomIns, kernels.cuh) run by one interpreter per thread.  The program
// and its constants are staged into shared memory once per CTA; the intermediate values of a thread live in
// shared memory too, in n_slots physical slots (the host allocates them by liveness).  A memory value operand is
// formed on the fly from the polynomial (after the first evaluation point the loads hit L1).  The instruction stream is
// the same for every thread, so the dispatch on the opcode never diverges.
static constexpr int kCustomThreads = 128;

// d * t for a small integer t (t <= kCustomMaxDegree + 1): double-and-add, cheaper than a Montgomery product
__device__ __forceinline__ fr_t fr_mul_small(const fr_t& d, int t) {
  fr_t r = fr_zero();
#pragma unroll 1
  for (int b = 4; b >= 0; b--) {
    r = fr_dbl(r);
    if ((t >> b) & 1) r = fr_add(r, d);
  }
  return r;
}
// slot s of this thread: 8 words, word-major across the CTA so that a warp's accesses are conflict-free
__device__ __forceinline__ fr_t custom_ld(const uint32_t* sm, int s) {
  fr_t r;
#pragma unroll
  for (int l = 0; l < 8; l++) r.v[l] = sm[(s * 8 + l) * kCustomThreads + threadIdx.x];
  return r;
}
__device__ __forceinline__ void custom_st(uint32_t* sm, int s, const fr_t& x) {
#pragma unroll
  for (int l = 0; l < 8; l++) sm[(s * 8 + l) * kCustomThreads + threadIdx.x] = x.v[l];
}
// g(x_0, .., x_{alpha-1}); input(k) yields x_k
template <class Input>
__device__ __forceinline__ fr_t custom_run(const CustomIns* ops, int n_ops, const fr_t* consts, uint32_t* slots,
                                           Input input) {
  fr_t r = fr_zero();
#pragma unroll 1
  for (int j = 0; j < n_ops; j++) {
    const CustomIns in = ops[j];
    const fr_t a = in.a >= 0 ? custom_ld(slots, in.a) : input(-1 - in.a);
    if (in.op == CUSTOM_MULK) {
      r = fr_mul(a, consts[in.b]);
    } else if (in.op == CUSTOM_ADDK) {
      r = fr_add(a, consts[in.b]);
    } else {
      const fr_t b = in.b >= 0 ? custom_ld(slots, in.b) : input(-1 - in.b);
      r = in.op == CUSTOM_ADD ? fr_add(a, b) : (in.op == CUSTOM_SUB ? fr_sub(a, b) : fr_mul(a, b));
    }
    if (j + 1 < n_ops) custom_st(slots, in.dst, r);
  }
  return r;
}
// shared memory: instructions | constants | slots of every thread | (round kernel) accumulators of every thread
// (Prog: a CustomStrategy or a CombProgram)
template <class Prog>
static size_t custom_smem_bytes(const Prog& cs, int npoints) {
  return (size_t)cs.n_ops * sizeof(CustomIns) + (size_t)cs.n_consts * sizeof(fr_t) +
         (size_t)(cs.n_slots + npoints) * sizeof(fr_t) * kCustomThreads;
}
template <class Prog>
__device__ __forceinline__ void custom_stage(const Prog& cs, CustomIns*& ops, fr_t*& consts, uint32_t*& slots) {
  extern __shared__ __align__(32) unsigned char custom_sm[];
  consts = (fr_t*)custom_sm;  // first: 32-byte alignment
  ops = (CustomIns*)(consts + cs.n_consts);
  slots = (uint32_t*)(ops + cs.n_ops);
  for (int j = threadIdx.x; j < cs.n_ops; j += blockDim.x) ops[j] = cs.d_ops[j];
  for (int j = threadIdx.x; j < cs.n_consts; j += blockDim.x) consts[j] = cs.d_consts[j];
  __syncthreads();
}

// One round of prove_arbitrary (sumcheck.rs:179-237) for any program: per index pair i and point t = 0..npts-1,
// eq(t) * g(x(t)) with x_k(t) = lo_k + t (hi_k - lo_k).  The npts accumulators sit after the slots.
__global__ void __launch_bounds__(kCustomThreads)
    sc_eval_custom_kernel(CustomStrategy cs, const fr_t* base, size_t stride, size_t half, int npts, Finalize fin) {
  __shared__ fr_t scratch[kCustomThreads / 32];
  __shared__ fr_t res[kCustomMaxDegree + 2];
  __shared__ int s_last;
  CustomIns* ops;
  fr_t* consts;
  uint32_t* slots;
  custom_stage(cs, ops, consts, slots);
  uint32_t* acc = slots + cs.n_slots * 8 * kCustomThreads;
  for (int t = 0; t < npts; t++) custom_st(acc, t, fr_zero());
  const fr_t* eq = base + (size_t)cs.alpha * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t q0 = ld_fr(eq + i), dq = fr_sub(ld_fr(eq + half + i), q0);
    fr_t cq = q0;
#pragma unroll 1
    for (int t = 0; t < npts; t++) {
      const fr_t g = custom_run(ops, cs.n_ops, consts, slots, [&](int k) {
        const fr_t* P = base + (size_t)k * stride;
        const fr_t lo = ld_fr(P + i);
        if (t == 0) return lo;
        const fr_t hi = ld_fr(P + half + i);
        return t == 1 ? hi : fr_add(lo, fr_mul_small(fr_sub(hi, lo), t));
      });
      custom_st(acc, t, fr_add(custom_ld(acc, t), fr_mul(g, cq)));
      cq = fr_add(cq, dq);
    }
  }
  for (int t = 0; t < npts; t++) {
    fr_t v[1] = {custom_ld(acc, t)};
    block_sum_fr<1>(v, scratch);
    if (threadIdx.x == 0) res[t] = v[0];
  }
  __syncthreads();
  if (gridDim.x == 1) {
    if ((int)threadIdx.x < npts) finalize_publish(fin, threadIdx.x, res[threadIdx.x]);
    return;
  }
  if ((int)threadIdx.x < npts) fin.partial[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = res[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(fin.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  finalize_last_stage(fin, gridDim.x, npts);
}

// subtables/mod.rs:186-216 for any program: sum_k eq[k] * g(E_1[k], ..., E_alpha[k])
__global__ void __launch_bounds__(kCustomThreads)
    claim_custom_kernel(CustomStrategy cs, const fr_t* base, size_t stride, size_t n, fr_t* partial) {
  __shared__ fr_t scratch[kCustomThreads / 32];
  CustomIns* ops;
  fr_t* consts;
  uint32_t* slots;
  custom_stage(cs, ops, consts, slots);
  fr_t acc[1] = {fr_zero()};
  const fr_t* eq = base + (size_t)cs.alpha * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t g = custom_run(ops, cs.n_ops, consts, slots, [&](int k) { return ld_fr(base + (size_t)k * stride + i); });
    acc[0] = fr_add(acc[0], fr_mul(g, ld_fr(eq + i)));
  }
  block_sum_fr<1>(acc, scratch);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc[0];
}

// ------------------------------------------------------------------------------------ K2 over a caller's polynomials
// prove_arbitrary (sumcheck.rs:149-260) for a combining function g of k independent polynomials, no eq factor (a caller
// that wants one passes eq as an input).  The same interpreter as the custom strategies; the inputs are k pointers.
// acc[t] += g(x(t)) for the pair i, x_k(t) = lo_k + t (hi_k - lo_k), lo_k = in.p[k][i], hi_k = in.p[k][half + i]
__device__ __forceinline__ void comb_accumulate(const CombProgram& pg, const CustomIns* ops, const fr_t* consts,
                                                uint32_t* slots, uint32_t* acc, const CombPtrs& in, size_t half, size_t i,
                                                int npts) {
#pragma unroll 1
  for (int t = 0; t < npts; t++) {
    const fr_t g = custom_run(ops, pg.n_ops, consts, slots, [&](int k) {
      const fr_t* P = in.p[k];
      const fr_t lo = ld_fr(P + i);
      if (t == 0) return lo;
      const fr_t hi = ld_fr(P + half + i);
      return t == 1 ? hi : fr_add(lo, fr_mul_small(fr_sub(hi, lo), t));
    });
    custom_st(acc, t, fr_add(custom_ld(acc, t), g));
  }
}
// the npts sums of the CTA -> block partials -> the last CTA adds them and publishes (as sc_eval_custom_kernel)
__device__ __forceinline__ void comb_finish(uint32_t* acc, int npts, const Finalize& fin) {
  __shared__ fr_t scratch[kCustomThreads / 32];
  __shared__ fr_t res[kCustomMaxDegree + 1];
  __shared__ int s_last;
  for (int t = 0; t < npts; t++) {
    fr_t v[1] = {custom_ld(acc, t)};
    block_sum_fr<1>(v, scratch);
    if (threadIdx.x == 0) res[t] = v[0];
  }
  __syncthreads();
  if (gridDim.x == 1) {
    if ((int)threadIdx.x < npts) finalize_publish(fin, threadIdx.x, res[threadIdx.x]);
    return;
  }
  if ((int)threadIdx.x < npts) fin.partial[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = res[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(fin.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  finalize_last_stage(fin, gridDim.x, npts);
}
// One round: degree + 1 evaluation points, the accumulators after the slots in shared memory
__global__ void __launch_bounds__(kCustomThreads)
    sc_eval_comb_kernel(CombProgram pg, const __grid_constant__ CombPtrs in, size_t half, Finalize fin) {
  CustomIns* ops;
  fr_t* consts;
  uint32_t* slots;
  custom_stage(pg, ops, consts, slots);
  const int npts = pg.degree + 1;
  uint32_t* acc = slots + pg.n_slots * 8 * kCustomThreads;
  for (int t = 0; t < npts; t++) custom_st(acc, t, fr_zero());
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x)
    comb_accumulate(pg, ops, consts, slots, acc, in, half, i, npts);
  comb_finish(acc, npts, fin);
}
// The bind of round j-1 and the evaluation of round j in one pass: thread i folds src elements i, i+q, i+2q, i+3q of
// every input to dst elements i, i+q, then evaluates the pair i of the bound inputs.  The bound values are read back
// from dst after the stores (this thread's own stores: L1 or L2 hits) rather than kept in shared memory, which at
// 64 B per input per thread would not fit next to the slots and accumulators for k = 16.  Every element of src is read
// once, so the round costs 4 reads + 2 writes of 32 B per input and pair instead of 4 + 2 (bind) + 2 (evaluation).
// In place (src == dst) is safe: elements i and i+q are read and written by thread i only.
__global__ void __launch_bounds__(kCustomThreads)
    sc_bind_eval_comb_kernel(CombProgram pg, const __grid_constant__ CombPtrs src, const __grid_constant__ CombPtrs dst, size_t q,
                             fr_t r, Finalize fin) {
  CustomIns* ops;
  fr_t* consts;
  uint32_t* slots;
  custom_stage(pg, ops, consts, slots);
  const int npts = pg.degree + 1;
  uint32_t* acc = slots + pg.n_slots * 8 * kCustomThreads;
  for (int t = 0; t < npts; t++) custom_st(acc, t, fr_zero());
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < q; i += (size_t)gridDim.x * blockDim.x) {
#pragma unroll 1
    for (int k = 0; k < pg.n_inputs; k++) {
      const fr_t* S = src.p[k];
      fr_t* D = dst.p[k];
      const fr_t a0 = ld_fr_stream(S + i), a1 = ld_fr_stream(S + q + i);
      const fr_t a2 = ld_fr_stream(S + 2 * q + i), a3 = ld_fr_stream(S + 3 * q + i);
      st_fr(D + i, fr_add(a0, fr_mul(r, fr_sub(a2, a0))));
      st_fr(D + q + i, fr_add(a1, fr_mul(r, fr_sub(a3, a1))));
    }
    comb_accumulate(pg, ops, consts, slots, acc, dst, q, i, npts);
  }
  comb_finish(acc, npts, fin);
}
// dense_mlpoly.rs:209-216 over the pointer descriptor, one input per blockIdx.y
__global__ void __launch_bounds__(kThreads) bind_comb_kernel(const __grid_constant__ CombPtrs src, const __grid_constant__ CombPtrs dst,
                                                             size_t half, fr_t r) {
  const fr_t* Z = src.p[blockIdx.y];
  fr_t* out = dst.p[blockIdx.y];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t lo = ld_fr_stream(Z + i), hi = ld_fr_stream(Z + half + i);
    st_fr(out + i, fr_add(lo, fr_mul(r, fr_sub(hi, lo))));
  }
}
// the final evaluations: only element 0 of the last bind is read (sumcheck.rs:258), so only it is computed
__global__ void final_comb_kernel(const __grid_constant__ CombPtrs src, int n, size_t half, fr_t r, Finalize fin) {
  const int k = threadIdx.x;
  if (k >= n) return;
  const fr_t lo = ld_fr(src.p[k]), hi = ld_fr(src.p[k] + half);
  finalize_publish(fin, k, fr_add(lo, fr_mul(r, fr_sub(hi, lo))));
}
// out[i] = g(in.p[0][i], .., in.p[k-1][i]): a polynomial formed pointwise from others, one element per thread
__global__ void __launch_bounds__(kCustomThreads)
    comb_map_kernel(CombProgram pg, const __grid_constant__ CombPtrs in, size_t n, fr_t* out) {
  CustomIns* ops;
  fr_t* consts;
  uint32_t* slots;
  custom_stage(pg, ops, consts, slots);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    st_fr(out + i, custom_run(ops, pg.n_ops, consts, slots, [&](int k) { return ld_fr(in.p[k] + i); }));
}

// dynamic shared memory above the default 48 KiB needs an opt-in per kernel and device (at context creation): the
// largest program's
void poly_init_device() {
  CustomStrategy cs{};
  cs.n_ops = kCustomMaxOps;
  cs.n_consts = kCustomMaxConsts;
  cs.n_slots = kCustomMaxSlots;
  const int bytes = (int)custom_smem_bytes(cs, kCustomMaxDegree + 2);
  LB_CUDA_CHECK(cudaFuncSetAttribute(sc_eval_custom_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  LB_CUDA_CHECK(cudaFuncSetAttribute(claim_custom_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  const int comb_bytes = (int)custom_smem_bytes(cs, kCustomMaxDegree + 1);
  LB_CUDA_CHECK(cudaFuncSetAttribute(sc_eval_comb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, comb_bytes));
  LB_CUDA_CHECK(cudaFuncSetAttribute(sc_bind_eval_comb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, comb_bytes));
  LB_CUDA_CHECK(cudaFuncSetAttribute(comb_map_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)custom_smem_bytes(cs, 0)));
}
// grid: one wave of as many CTAs as fit an SM at this shared-memory size
static int custom_grid(size_t n, size_t smem) {
  int per_sm = (int)((200u << 10) / (smem + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > kBlocksPerSM * 2) per_sm = kBlocksPerSM * 2;
  return grid_for(n, kCustomThreads, kNumSMs * per_sm);
}
static void launch_eval_custom(const CustomStrategy& cs, const fr_t* base, size_t stride, size_t half, int npts,
                               const Finalize& fin, cudaStream_t st) {
  const size_t smem = custom_smem_bytes(cs, npts);
  launch(sc_eval_custom_kernel, custom_grid(half, smem), kCustomThreads, smem, st, cs, base, stride, half, npts, fin);
}

// combine_lookups weights are F::from(1u64 << (i * inc)): inc = log2 of the chunk size (and.rs:45-53, range_check.rs:78-86)
static int linear_inc(const Strategy& S) { return S.kind == STRAT_RANGE ? S.log_m : S.log_m / 2; }

template <int C>
static void launch_lt(const fr_t* base, size_t stride, size_t half, const Finalize& fin, int blocks, cudaStream_t st) {
  launch(sc_eval_lt_kernel<C>, blocks, 128, 0, st, base, stride, half, fin);
}

void launch_sumcheck_eval_arbitrary(const Strategy& S, const fr_t* base, size_t stride, size_t half, const Finalize& fin,
                                    cudaStream_t st) {
  int blocks;
  if (S.kind == STRAT_CUSTOM) {
    launch_eval_custom(*S.custom, base, stride, half, S.sumcheck_poly_degree() + 1, fin, st);
  } else if (S.kind == STRAT_LT) {
    blocks = grid_for(half, 128, kMaxBlocks);
    switch (S.C) {
      case 1: launch_lt<1>(base, stride, half, fin, blocks, st); break;
      case 2: launch_lt<2>(base, stride, half, fin, blocks, st); break;
      case 3: launch_lt<3>(base, stride, half, fin, blocks, st); break;
      case 4: launch_lt<4>(base, stride, half, fin, blocks, st); break;
      case 8:
        if (half >= 4096) {  // throughput-bound rounds: two lanes per pair (3 CTAs per SM instead of 2, no spills)
          launch(sc_eval_lt2_kernel<8>, grid_for(2 * half, 128, kNumSMs * 6), 128, 0, st, base, stride, half, fin);
        } else {
          launch_lt<8>(base, stride, half, fin, blocks, st);
        }
        break;
      default: {
        FrVec tv;
        for (int t = 0; t < 32; t++) tv.v[t] = fr_from_u64((uint64_t)t);
        launch(sc_eval_lt_generic_kernel<6>, blocks, 128, 0, st, base, stride, half, S.C, tv, fin);
      }
    }
  } else {
    blocks = grid_for(half);
    launch(sc_eval_linear_kernel, blocks, kThreads, 0, st, base, stride, S.num_memories(), half, linear_inc(S), fin);
  }
}
// bind with r (length 4q -> 2q) then evaluate the round over the bound polynomials, one launch; only the strategies
// with a linear g have a fused kernel (false: the caller binds and evaluates separately)
// Fusing pays on the large rounds; below q = 2^15 a round is a latency chain and the longer per-thread chain of the
// fused kernel can cost more than the two short launches it replaces — those rounds stay unfused (min_q = 0: that
// default; 1: always fuse).  tools/ab_primary.py compares the two in one process.
bool launch_sumcheck_bind_eval_arbitrary(const Strategy& S, fr_t* base, size_t stride, size_t q, const fr_t& r,
                                         const Finalize& fin, size_t min_q, cudaStream_t st) {
  static const size_t dflt_min_q = (size_t)bind_env("LASSO_B200_FUSED_MIN_Q", 1 << 15);
  if (S.kind == STRAT_LT || S.kind == STRAT_CUSTOM || q == 0 || q < (min_q ? min_q : dflt_min_q)) return false;
  launch(sc_bind_eval_linear_kernel, grid_for(q, kThreads, kNumSMs * 2), kThreads, 0, st, base, stride, S.num_memories(),
         q, r, linear_inc(S), fin);
  return true;
}

// ---- sumcheck over a caller's polynomials
void launch_sumcheck_eval_comb(const CombProgram& g, const CombPtrs& in, size_t half, const Finalize& fin, cudaStream_t st) {
  const size_t smem = custom_smem_bytes(g, g.degree + 1);
  launch(sc_eval_comb_kernel, custom_grid(half, smem), kCustomThreads, smem, st, g, in, half, fin);
}
void launch_bind_comb(const CombPtrs& src, const CombPtrs& dst, int n, size_t half, const fr_t& r, cudaStream_t st) {
  if (half == 0 || n == 0) return;
  int per = kNumSMs * kBindBlocksPerSM / n;
  if (per < kNumSMs / 4) per = kNumSMs / 4;
  launch(bind_comb_kernel, dim3(grid_for(half, kThreads, per), n), kThreads, 0, st, src, dst, half, r);
}
// The same threshold as the primary sumcheck's fused rounds: below q = 2^15 a round is a latency chain
bool launch_sumcheck_bind_eval_comb(const CombProgram& g, const CombPtrs& src, const CombPtrs& dst, size_t q, const fr_t& r,
                                    const Finalize& fin, size_t min_q, cudaStream_t st) {
  static const size_t dflt_min_q = (size_t)bind_env("LASSO_B200_FUSED_MIN_Q", 1 << 15);
  if (q == 0 || q < (min_q ? min_q : dflt_min_q)) return false;
  const size_t smem = custom_smem_bytes(g, g.degree + 1);
  launch(sc_bind_eval_comb_kernel, custom_grid(q, smem), kCustomThreads, smem, st, g, src, dst, q, r, fin);
  return true;
}
void launch_final_comb(const CombPtrs& src, int n, size_t half, const fr_t& r, const Finalize& fin, cudaStream_t st) {
  launch(final_comb_kernel, 1, 32, 0, st, src, n, half, r, fin);
}
void launch_comb_map(const CombProgram& g, const CombPtrs& in, size_t n, fr_t* out, cudaStream_t st) {
  const size_t smem = custom_smem_bytes(g, 0);
  launch(comb_map_kernel, custom_grid(n, smem), kCustomThreads, smem, st, g, in, n, out);
}

// subtables/mod.rs:186-216: sum_k eq[k] * g(E_1[k], ..., E_alpha[k]) over the whole hypercube
__global__ void __launch_bounds__(kThreads)
    claim_linear_kernel(const fr_t* base, size_t stride, int alpha, size_t n, int inc, fr_t* partial) {
  __shared__ fr_t scratch[kThreads / 32];
  fr_t acc[1] = {fr_zero()};
  const fr_t* eq = base + (size_t)alpha * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    fr_t c = ld_fr_stream(base + (size_t)(alpha - 1) * stride + i);
    for (int k = alpha - 2; k >= 0; k--) c = fr_add(fr_mul_pow2(c, inc), ld_fr_stream(base + (size_t)k * stride + i));
    acc[0] = fr_add(acc[0], fr_mul(c, ld_fr_stream(eq + i)));
  }
  block_sum_fr<1>(acc, scratch);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc[0];
}
__global__ void __launch_bounds__(kThreads)
    claim_lt_kernel(const fr_t* base, size_t stride, int C, size_t n, fr_t* partial) {
  __shared__ fr_t scratch[kThreads / 32];
  fr_t acc[1] = {fr_zero()};
  const fr_t* eq = base + (size_t)(2 * C) * stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    fr_t h = fr_zero();
    for (int k = C - 1; k >= 0; k--) {
      fr_t l = ld_fr(base + (size_t)(2 * k) * stride + i), e = ld_fr(base + (size_t)(2 * k + 1) * stride + i);
      h = fr_add(l, fr_mul(e, h));
    }
    acc[0] = fr_add(acc[0], fr_mul(h, ld_fr(eq + i)));
  }
  block_sum_fr<1>(acc, scratch);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc[0];
}
void launch_sumcheck_claim(const Strategy& S, const fr_t* base, size_t stride, size_t n, fr_t* partial, fr_t* out,
                           cudaStream_t st) {
  int blocks = grid_for(n);
  if (S.kind == STRAT_CUSTOM) {
    const size_t smem = custom_smem_bytes(*S.custom, 0);
    blocks = custom_grid(n, smem);
    launch(claim_custom_kernel, blocks, kCustomThreads, smem, st, *S.custom, base, stride, n, partial);
  } else if (S.kind == STRAT_LT)
    launch(claim_lt_kernel, blocks, kThreads, 0, st, base, stride, S.C, n, partial);
  else
    launch(claim_linear_kernel, blocks, kThreads, 0, st, base, stride, S.num_memories(), n, linear_inc(S), partial);
  launch(reduce_partials_kernel, 1, kThreads, 0, st, partial, blocks, out);
}

// ------------------------------------------------------------------------------------ K3
// sumcheck.rs:49-93: per circuit (e0, e2, e3) = sum_i A B C at t = 0, 2, 3, with the batching coefficients folded in.
// prove_cubic_batched only ever uses  sum_k coeff_k * (e0, e2, e3)_k  (sumcheck.rs:95-104), and everything in a
// round is linear in A_k.  So the FIRST bind of a layer stores coeff_k * A_k, every later round works on the
// scaled arrays, and a round evaluates  sum_i C_i(t) * sum_k A'_k,i(t) B_k,i(t):  per element pair 7
// multiplications per circuit (4 binds + 3 products) + 5 shared (2 eq binds + 3 times C(t)) instead of 12 per
// circuit; the round message is 3 elements instead of 3 per circuit.  The layer's claims A_k(r) are recovered on the
// host with the inverse coefficients (one batch inversion per layer, off the critical path).
//   scale != 0: the arrays A_k in memory are still unscaled; multiply by coeff_k on the fly (and store the scaled
//   value when binding).  Circuits are strided over blockIdx.y so that small rounds still fill the machine.
__global__ void __launch_bounds__(kThreads)
    sc_eval_cubic_comb_kernel(fr_t* const* A, fr_t* const* B, const fr_t* Ceq, size_t half, int ncirc, CubicCoeffs cf,
                              int scale, Finalize fin) {
  __shared__ fr_t scratch[3 * kThreads / 32];
  fr_t acc[3] = {fr_zero(), fr_zero(), fr_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x) {
    fr_t s0 = fr_zero(), s2 = fr_zero(), s3 = fr_zero();
    for (int k = blockIdx.y; k < ncirc; k += gridDim.y) {
      const fr_t* a = A[k];
      const fr_t* b = B[k];
      fr_t a0 = ld_fr_stream(a + i), a1 = ld_fr_stream(a + half + i);
      if (scale) {
        a0 = fr_mul(cf.v[k], a0);
        a1 = fr_mul(cf.v[k], a1);
      }
      const fr_t b0 = ld_fr_stream(b + i), b1 = ld_fr_stream(b + half + i);
      const fr_t da = fr_sub(a1, a0), db = fr_sub(b1, b0);
      const fr_t a2 = fr_add(a1, da), b2 = fr_add(b1, db);
      s0 = fr_add(s0, fr_mul(a0, b0));
      s2 = fr_add(s2, fr_mul(a2, b2));
      s3 = fr_add(s3, fr_mul(fr_add(a2, da), fr_add(b2, db)));
    }
    const fr_t c0 = ld_fr(Ceq + i), c1 = ld_fr(Ceq + half + i), dc = fr_sub(c1, c0), c2 = fr_add(c1, dc);
    acc[0] = fr_add(acc[0], fr_mul(s0, c0));
    acc[1] = fr_add(acc[1], fr_mul(s2, c2));
    acc[2] = fr_add(acc[2], fr_mul(s3, fr_add(c2, dc)));
  }
  block_sum_fr<3>(acc, scratch);
  const int total = gridDim.x * gridDim.y;
  finalize_block<3>(fin, acc, 0, blockIdx.y * gridDim.x + blockIdx.x, total, 3, total);
}
// h = number of bound outputs per polynomial (current length / 2), must be >= 2.
__global__ void __launch_bounds__(kThreads)
    sc_bind_eval_cubic_comb_kernel(fr_t* const* A, fr_t* const* B, const fr_t* Cin, fr_t* Cout, size_t h, fr_t r, int ncirc,
                                   CubicCoeffs cf, int scale, Finalize fin) {
  __shared__ fr_t scratch[3 * kThreads / 32];
  const size_t q = h / 2;
  fr_t acc[3] = {fr_zero(), fr_zero(), fr_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < q; i += (size_t)gridDim.x * blockDim.x) {
    fr_t s0 = fr_zero(), s2 = fr_zero(), s3 = fr_zero();
    fr_t lo, hi;
    for (int k = blockIdx.y; k < ncirc; k += gridDim.y) {
      fr_t* a = A[k];
      fr_t* b = B[k];
      lo = ld_fr_stream(a + i); hi = ld_fr_stream(a + i + h);
      fr_t a0 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
      lo = ld_fr_stream(a + i + q); hi = ld_fr_stream(a + i + q + h);
      fr_t a1 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
      if (scale) {
        a0 = fr_mul(cf.v[k], a0);
        a1 = fr_mul(cf.v[k], a1);
      }
      st_fr(a + i, a0);
      st_fr(a + i + q, a1);
      lo = ld_fr_stream(b + i); hi = ld_fr_stream(b + i + h);
      const fr_t b0 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
      lo = ld_fr_stream(b + i + q); hi = ld_fr_stream(b + i + q + h);
      const fr_t b1 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
      st_fr(b + i, b0);
      st_fr(b + i + q, b1);
      const fr_t da = fr_sub(a1, a0), db = fr_sub(b1, b0);
      const fr_t a2 = fr_add(a1, da), b2 = fr_add(b1, db);
      s0 = fr_add(s0, fr_mul(a0, b0));
      s2 = fr_add(s2, fr_mul(a2, b2));
      s3 = fr_add(s3, fr_mul(fr_add(a2, da), fr_add(b2, db)));
    }
    lo = ld_fr(Cin + i); hi = ld_fr(Cin + i + h);
    const fr_t c0 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
    lo = ld_fr(Cin + i + q); hi = ld_fr(Cin + i + q + h);
    const fr_t c1 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
    if (blockIdx.y == 0) {
      st_fr(Cout + i, c0);
      st_fr(Cout + i + q, c1);
    }
    const fr_t dc = fr_sub(c1, c0), c2 = fr_add(c1, dc);
    acc[0] = fr_add(acc[0], fr_mul(s0, c0));
    acc[1] = fr_add(acc[1], fr_mul(s2, c2));
    acc[2] = fr_add(acc[2], fr_mul(s3, fr_add(c2, dc)));
  }
  block_sum_fr<3>(acc, scratch);
  const int total = gridDim.x * gridDim.y;
  finalize_block<3>(fin, acc, 0, blockIdx.y * gridDim.x + blockIdx.x, total, 3, total);
}
// Latency-oriented variant of the two kernels above for the small and medium rounds (most of the ~300 rounds of
// a grand-product argument move a few KB: what the host waits for is the dependent chain inside one thread,
// 12 field multiplications).  FOUR lanes per (circuit k, pair index i):
//   lane 0 / 1 / 2 binds its side (A_k / B_k / eq) at i and i+q (2 multiplications, do_bind != 0) and forms
//   the side's values at t = 0, 2, 3; three quad shuffles hand lane t the three factors of its evaluation
//   point, which it multiplies (2 multiplications): 4 dependent multiplications instead of 12.
// Sums over i: xor-shuffles inside the warp, shared memory across warps, then either a direct tagged
// publication (single CTA: no ticket, no fence) or the usual Finalize last-CTA stage.
//   do_bind = 1: arrays hold 4q elements, pairs (i, i+2q) are bound with r into (i), then evaluated as (i, i+q)
//   do_bind = 0: arrays hold 2q elements, evaluated as (i, i+q)               (q a power of two)
__global__ void __launch_bounds__(1024)
    sc_cubic_quad_kernel(fr_t* const* A, fr_t* const* B, const fr_t* Cin, fr_t* Cout, size_t q, int lg_q, int do_bind,
                         fr_t r, int ncirc, CubicCoeffs cf, int scale, Finalize fin) {
  // cf / scale: see the kernels above — scale: lane 0 multiplies its side by coeff_k (stored when binding); the CTA
  // yields 3 values, summed over all its circuits
  __shared__ fr_t s_part[32 * 3];  // per warp
  __shared__ int s_last;
  const int tid = threadIdx.x, role = tid & 3, lane = tid & 31;
  const int upb = blockDim.x >> 2;  // (circuit, pair) units per CTA
  const size_t U = (size_t)blockIdx.x * upb + (tid >> 2), total = (size_t)ncirc << lg_q;
  const bool valid = U < total;
  const int k = valid ? (int)(U >> lg_q) : 0;
  const size_t i = U & (q - 1), h = 2 * q;
  fr_t x0 = fr_zero(), x1 = fr_zero();
  if (valid && role < 3) {
    fr_t* src = role == 0 ? A[k] : role == 1 ? B[k] : const_cast<fr_t*>(Cin);
    if (do_bind) {
      fr_t lo = ld_fr(src + i), hi = ld_fr(src + i + h);
      x0 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
      lo = ld_fr(src + i + q);
      hi = ld_fr(src + i + q + h);
      x1 = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
    } else {
      x0 = ld_fr(src + i);
      x1 = ld_fr(src + i + q);
    }
    if (scale && role == 0) {
      x0 = fr_mul(cf.v[k], x0);
      x1 = fr_mul(cf.v[k], x1);
    }
    if (do_bind) {
      fr_t* dst = role == 2 ? (k == 0 ? Cout : nullptr) : src;
      if (dst) {
        st_fr(dst + i, x0);
        st_fr(dst + i + q, x1);
      }
    }
  }
  // this side at t = 0, 2, 3
  fr_t e0 = x0, d = fr_sub(x1, x0), e2 = fr_add(x1, d), e3 = fr_add(e2, d);
  // round j: side s offers its value at t = (s + j) % 3; lane t reads side (t - j) mod 3 -> that side at t
  fr_t P;
  const int qbase = lane & ~3;
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const int sel = (role + j) % 3;
    const fr_t offer = sel == 0 ? e0 : (sel == 1 ? e2 : e3);
    const int src_lane = qbase + (role + 3 - j) % 3;
    fr_t got;
#pragma unroll
    for (int l = 0; l < 8; l++) got.v[l] = __shfl_sync(0xffffffffu, offer.v[l], src_lane);
    P = j == 0 ? got : fr_mul(P, got);
  }
  if (!valid || role == 3) P = fr_zero();
  // sum over the 8 units of the warp, whatever their circuit
  for (int off = 1; off < 8; off <<= 1) {
    fr_t o;
#pragma unroll
    for (int l = 0; l < 8; l++) o.v[l] = __shfl_xor_sync(0xffffffffu, P.v[l], off * 4);
    P = fr_add(P, o);
  }
  const int unit = tid >> 2;
  if ((unit & 7) == 0 && role < 3) s_part[(unit / 8) * 3 + role] = P;
  __syncthreads();
  // block outputs: 3 values, each the sum over all warps
  fr_t val = fr_zero();
  if (tid < 3) {
    const int nw = blockDim.x >> 5;
    for (int w = 0; w < nw; w++) val = fr_add(val, s_part[w * 3 + tid]);
  }
  if (gridDim.x == 1) {
    if (tid < 3) finalize_publish(fin, tid, val);
    return;
  }
  if (tid < 3) {
    fin.partial[(size_t)tid * gridDim.x + blockIdx.x] = val;
    __threadfence();
  }
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(fin.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  finalize_last_stage(fin, gridDim.x, 3);
}
static constexpr size_t kQuadMaxQ = 2048;  // beyond this the rounds are throughput-bound: thread-per-pair kernels
static void launch_cubic_quad(fr_t* const* d_A, fr_t* const* d_B, const fr_t* Cin, fr_t* Cout, int ncirc, size_t q,
                              int do_bind, const fr_t& r, const CubicCoeffs& cf, int scale, const Finalize& fin,
                              cudaStream_t st) {
  int lg_q = 0;
  while (((size_t)1 << lg_q) < q) lg_q++;
  const size_t threads = 4 * (size_t)ncirc * q;
  if (threads <= 1024) {
    unsigned t = (unsigned)((threads + 31) / 32 * 32);
    launch(sc_cubic_quad_kernel, 1, t, 0, st, d_A, d_B, Cin, Cout, q, lg_q, do_bind, r, ncirc, cf, scale, fin);
  } else {
    unsigned blocks = (unsigned)(((size_t)ncirc * q + 63) / 64);
    launch(sc_cubic_quad_kernel, blocks, 256, 0, st, d_A, d_B, Cin, Cout, q, lg_q, do_bind, r, ncirc, cf, scale, fin);
  }
}
// circuits are strided over blockIdx.y: enough CTAs for ~2 per SM even when a round has few pairs
static dim3 comb_grid(size_t pairs, int ncirc) {
  int bx = grid_for(pairs, kThreads, kMaxBlocks);
  int gy = (2 * kNumSMs + bx - 1) / bx;
  if (gy > ncirc) gy = ncirc;
  if (gy < 1) gy = 1;
  return dim3(bx, gy);
}
void launch_sumcheck_bind_eval_cubic_comb(fr_t* const* d_A, fr_t* const* d_B, const fr_t* Cin, fr_t* Cout, int ncirc, size_t h,
                                          const fr_t& r, const CubicCoeffs& cf, int scale, const Finalize& fin, cudaStream_t st) {
  size_t q = h / 2;
  if (q <= kQuadMaxQ && (q & (q - 1)) == 0) return launch_cubic_quad(d_A, d_B, Cin, Cout, ncirc, q, 1, r, cf, scale, fin, st);
  launch(sc_bind_eval_cubic_comb_kernel, comb_grid(q, ncirc), kThreads, 0, st, d_A, d_B, Cin, Cout, h, r, ncirc, cf,
         scale, fin);
}
void launch_sumcheck_eval_cubic_comb(fr_t* const* d_A, fr_t* const* d_B, const fr_t* Ceq, int ncirc, size_t half,
                                     const CubicCoeffs& cf, int scale, const Finalize& fin, cudaStream_t st) {
  if (half <= kQuadMaxQ && (half & (half - 1)) == 0)
    return launch_cubic_quad(d_A, d_B, Ceq, nullptr, ncirc, half, 0, fr_zero(), cf, scale, fin, st);
  launch(sc_eval_cubic_comb_kernel, comb_grid(half, ncirc), kThreads, 0, st, d_A, d_B, Ceq, half, ncirc, cf, scale, fin);
}

// ------------------------------------------------------------------------------------ K5
__device__ __forceinline__ uint32_t subtable_value(int kind, int sub, uint32_t idx, int log_m, int log_r) {
  if (kind == STRAT_RANGE) {  // range_check.rs:15-34
    if (sub == 0) return idx;
    if (sub == 1) return idx < (1u << (log_r % log_m)) ? idx : 0u;
    return 0u;
  }
  int bits = log_m / 2;  // utils/mod.rs:82-89 split_bits: (high, low)
  uint32_t lhs = (idx >> bits) & ((1u << bits) - 1), rhs = idx & ((1u << bits) - 1);
  switch (kind) {
    case STRAT_AND: return lhs & rhs;
    case STRAT_OR: return lhs | rhs;
    case STRAT_XOR: return lhs ^ rhs;
    default: return sub == 0 ? (lhs < rhs) : (lhs == rhs);  // lt.rs:16-30
  }
}
__global__ void __launch_bounds__(kThreads)
    materialize_kernel(int kind, int nsub, int log_m, int log_r, fr_t* tables_fr, uint32_t* tables_u32) {
  size_t M = (size_t)1 << log_m, n = M * nsub;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t v = subtable_value(kind, (int)(i >> log_m), (uint32_t)(i & (M - 1)), log_m, log_r);
    if (tables_u32) tables_u32[i] = v;
    if (tables_fr) st_fr(tables_fr + i, fr_from_u64(v));
  }
}
void launch_materialize_subtables(const Strategy& S, fr_t* tables_fr, uint32_t* tables_u32, cudaStream_t st) {
  if (S.kind == STRAT_CUSTOM) throw std::runtime_error("a custom strategy's tables are uploaded, not materialised");
  size_t n = (size_t)S.M() * S.num_subtables();
  launch(materialize_kernel, grid_for(n), kThreads, 0, st, S.kind, S.num_subtables(), S.log_m, S.log_r, tables_fr,
         tables_u32);
}
struct GatherMap {
  int sub[32], dim[32];
};
// subtables/mod.rs:78-92: E_k[j] = T_sub(k)[nz_dim(k)[j]]; 32 B written per (memory, lookup)
__global__ void __launch_bounds__(kThreads)
    gather_kernel(GatherMap map, int log_m, const fr_t* tables_fr, const uint32_t* tables_u32, const uint32_t* nz,
                  size_t s, fr_t* E_fr, size_t E_stride, uint32_t* E_u32) {
  int k = blockIdx.y;
  const uint32_t* idx = nz + (size_t)map.dim[k] * s;
  size_t toff = (size_t)map.sub[k] << log_m;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < s; j += (size_t)gridDim.x * blockDim.x) {
    uint32_t a = idx[j];
    if (E_fr) st_fr(E_fr + (size_t)k * E_stride + j, ld_fr(tables_fr + toff + a));
    if (E_u32) E_u32[(size_t)k * s + j] = tables_u32[toff + a];
  }
}
void launch_gather_lookup_polys(const Strategy& S, const fr_t* tables_fr, const uint32_t* tables_u32,
                                const uint32_t* nz, size_t s, fr_t* E_fr, size_t E_stride, uint32_t* E_u32,
                                cudaStream_t st) {
  GatherMap map;
  for (int k = 0; k < S.num_memories(); k++) {
    map.sub[k] = S.memory_to_subtable_index(k);
    map.dim[k] = S.memory_to_dimension_index(k);
  }
  dim3 grid(grid_for(s, kThreads, kMaxBlocks / S.num_memories() + 1), S.num_memories());
  launch(gather_kernel, grid, kThreads, 0, st, map, S.log_m, tables_fr, tables_u32, nz, s, E_fr, E_stride, E_u32);
}
__global__ void __launch_bounds__(kThreads) from_u32_kernel(const uint32_t* in, fr_t* out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    st_fr(out + i, fr_from_u64(in[i]));
}
void launch_from_u32(const uint32_t* in, fr_t* out, size_t n, cudaStream_t st) {
  if (n) launch(from_u32_kernel, grid_for(n), kThreads, 0, st, in, out, n);
}
void launch_fill_zero(fr_t* out, size_t n, cudaStream_t st) {
  if (n) cudaMemsetAsync(out, 0, n * sizeof(fr_t), st);
}

// ------------------------------------------------------------------------------------ K7
// dense_mlpoly.rs:183-207 (bound) and dense_mlpoly.rs:228-235 + utils/mod.rs:63-73 (dot products with one eq table)
// for INTEGER-valued polynomials (dim, read, final, E: everything the prover commits to and
// opens is an index, a counter or a table value < 2^32, kept as a u32 mirror next to the field form).  A field element
// times a 32-bit integer is 8 IMAD.WIDE instead of a ~235-instruction Montgomery product, and the sum can be carried
// as a plain 320-bit integer (X = sum_j L_j * z_j < 2^288 * #terms) and reduced ONCE: L_j is stored as L_j*R mod l, so
// X mod l is already the Montgomery form of the result.  Reads 4 B per element instead of 32 B.
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
// LZ[i] = sum_j L[j] z[j*R + i]: thread = column (coalesced across the warp), rows split into chunks over blockIdx.y
// (<= 2^20 rows per chunk), a second pass sums the chunk partials
static constexpr int kBoundChunks = 64;
int bound_max_chunks() { return kBoundChunks; }
__global__ void __launch_bounds__(kThreads)
    bound_u32_kernel(const uint32_t* Z, const fr_t* L, size_t L_size, size_t R_size, size_t rows_per_chunk, fr_t* partial) {
  __shared__ fr_t sL[64];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t j0 = (size_t)blockIdx.y * rows_per_chunk;
  size_t j1 = j0 + rows_per_chunk;
  if (j1 > L_size) j1 = L_size;
  wide_t acc;
  wide_zero(acc);
  for (size_t jb = j0; jb < j1; jb += 64) {  // the row weights of 64 rows at a time through shared memory
    __syncthreads();
    if (threadIdx.x < 64 && jb + threadIdx.x < j1) sL[threadIdx.x] = ld_fr(L + jb + threadIdx.x);
    __syncthreads();
    const size_t je = jb + 64 < j1 ? jb + 64 : j1;
    if (i < R_size)
      for (size_t j = jb; j < je; j++) wide_mad(acc, sL[j - jb], Z[j * R_size + i]);
  }
  if (i < R_size) st_fr(partial + (size_t)blockIdx.y * R_size + i, wide_reduce(acc));
}
__global__ void __launch_bounds__(kThreads) bound_reduce_kernel(const fr_t* partial, int chunks, size_t R_size, fr_t* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R_size) return;
  fr_t acc = fr_zero();
  for (int c = 0; c < chunks; c++) acc = fr_add(acc, ld_fr(partial + (size_t)c * R_size + i));
  st_fr(out + i, acc);
}
void launch_bound_u32(const uint32_t* Z, const fr_t* L, size_t L_size, size_t R_size, fr_t* partial, fr_t* out, cudaStream_t st) {
  int chunks = (int)(L_size < (size_t)kBoundChunks ? L_size : (size_t)kBoundChunks);
  size_t rows_per_chunk = (L_size + chunks - 1) / chunks;
  if (rows_per_chunk > ((size_t)1 << 20)) throw std::runtime_error("bound_u32: too many rows per chunk");
  dim3 grid((unsigned)((R_size + kThreads - 1) / kThreads), chunks);
  launch(bound_u32_kernel, grid, kThreads, 0, st, Z, L, L_size, R_size, rows_per_chunk, partial);
  launch(bound_reduce_kernel, (unsigned)((R_size + kThreads - 1) / kThreads), kThreads, 0, st, partial, chunks, R_size,
         out);
}
// out[k] = <z_k, eq>, z_k = base + k*stride (u32), k < npolys
__global__ void __launch_bounds__(kThreads)
    multi_dot_u32_kernel(const uint32_t* base, size_t stride, const fr_t* eq, size_t n, fr_t* partial) {
  __shared__ fr_t scratch[kThreads / 32];
  const uint32_t* P = base + (size_t)blockIdx.y * stride;
  wide_t w;
  wide_zero(w);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    wide_mad(w, ld_fr(eq + i), P[i]);  // a thread adds at most n / (gridDim.x * 256) < 2^32 terms
  fr_t acc[1] = {wide_reduce(w)};
  block_sum_fr<1>(acc, scratch);
  if (threadIdx.x == 0) partial[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = acc[0];
}
void launch_multi_dot_u32(const uint32_t* base, size_t stride, int npolys, const fr_t* eq, size_t n, fr_t* partial, fr_t* out,
                          cudaStream_t st) {
  int per = kMaxBlocks / npolys;
  if (per < 1) per = 1;
  int bx = grid_for(n, kThreads, per);
  dim3 grid(bx, npolys);
  launch(multi_dot_u32_kernel, grid, kThreads, 0, st, base, stride, eq, n, partial);
  launch(reduce_partials_kernel, npolys, kThreads, 0, st, partial, bx, out);
}
// The Fr twins, for the lookup values of a caller's table of arbitrary field elements (no u32 mirror): a Montgomery
// product per term.  Same chunks x R_size partials and the same second passes as the u32 forms.
__global__ void __launch_bounds__(kThreads)
    bound_fr_kernel(const fr_t* Z, const fr_t* L, size_t L_size, size_t R_size, size_t rows_per_chunk, fr_t* partial) {
  __shared__ fr_t sL[64];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t j0 = (size_t)blockIdx.y * rows_per_chunk;
  size_t j1 = j0 + rows_per_chunk;
  if (j1 > L_size) j1 = L_size;
  fr_t acc = fr_zero();
  for (size_t jb = j0; jb < j1; jb += 64) {
    __syncthreads();
    if (threadIdx.x < 64 && jb + threadIdx.x < j1) sL[threadIdx.x] = ld_fr(L + jb + threadIdx.x);
    __syncthreads();
    const size_t je = jb + 64 < j1 ? jb + 64 : j1;
    if (i < R_size)
      for (size_t j = jb; j < je; j++) acc = fr_add(acc, fr_mul(sL[j - jb], ld_fr(Z + j * R_size + i)));
  }
  if (i < R_size) st_fr(partial + (size_t)blockIdx.y * R_size + i, acc);
}
void launch_bound_fr(const fr_t* Z, const fr_t* L, size_t L_size, size_t R_size, fr_t* partial, fr_t* out, cudaStream_t st) {
  int chunks = (int)(L_size < (size_t)kBoundChunks ? L_size : (size_t)kBoundChunks);
  size_t rows_per_chunk = (L_size + chunks - 1) / chunks;
  dim3 grid((unsigned)((R_size + kThreads - 1) / kThreads), chunks);
  launch(bound_fr_kernel, grid, kThreads, 0, st, Z, L, L_size, R_size, rows_per_chunk, partial);
  launch(bound_reduce_kernel, (unsigned)((R_size + kThreads - 1) / kThreads), kThreads, 0, st, partial, chunks, R_size,
         out);
}
__global__ void __launch_bounds__(kThreads)
    multi_dot_fr_kernel(const fr_t* base, size_t stride, const fr_t* eq, size_t n, fr_t* partial) {
  __shared__ fr_t scratch[kThreads / 32];
  const fr_t* P = base + (size_t)blockIdx.y * stride;
  fr_t acc[1] = {fr_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    acc[0] = fr_add(acc[0], fr_mul(ld_fr(eq + i), ld_fr(P + i)));
  block_sum_fr<1>(acc, scratch);
  if (threadIdx.x == 0) partial[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = acc[0];
}
void launch_multi_dot_fr(const fr_t* base, size_t stride, int npolys, const fr_t* eq, size_t n, fr_t* partial, fr_t* out,
                         cudaStream_t st) {
  int per = kMaxBlocks / npolys;
  if (per < 1) per = 1;
  int bx = grid_for(n, kThreads, per);
  dim3 grid(bx, npolys);
  launch(multi_dot_fr_kernel, grid, kThreads, 0, st, base, stride, eq, n, partial);
  launch(reduce_partials_kernel, npolys, kThreads, 0, st, partial, bx, out);
}
// The pointer-table forms, for k independent polynomials of one length (lasso_poly_evaluate_batch): CTA row blockIdx.y
// takes the group of kDotGroup inputs from kDotGroup * blockIdx.y, and a thread reads each eq element once for all the
// inputs of its group, which keeps them in kDotGroup accumulators.  Block partials of input j go to
// partial[j * gridDim.x + blockIdx.x], the layout reduce_partials_kernel sums.
__global__ void __launch_bounds__(kThreads)
    multi_dot_ptrs_u32_kernel(const __grid_constant__ DotPtrs in, int k, const fr_t* eq, size_t n, fr_t* partial) {
  __shared__ fr_t scratch[kDotGroup * kThreads / 32];
  const int j0 = kDotGroup * blockIdx.y, m = k - j0 < kDotGroup ? k - j0 : kDotGroup;
  wide_t w[kDotGroup];
#pragma unroll
  for (int j = 0; j < kDotGroup; j++) wide_zero(w[j]);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t e = ld_fr(eq + i);
#pragma unroll
    for (int j = 0; j < kDotGroup; j++)
      if (j < m) wide_mad(w[j], e, static_cast<const uint32_t*>(in.p[j0 + j])[i]);
  }
  fr_t acc[kDotGroup];
#pragma unroll
  for (int j = 0; j < kDotGroup; j++) acc[j] = wide_reduce(w[j]);
  block_sum_fr<kDotGroup>(acc, scratch);
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < kDotGroup; j++)
      if (j < m) partial[(size_t)(j0 + j) * gridDim.x + blockIdx.x] = acc[j];
}
__global__ void __launch_bounds__(kThreads)
    multi_dot_ptrs_fr_kernel(const __grid_constant__ DotPtrs in, int k, const fr_t* eq, size_t n, fr_t* partial) {
  __shared__ fr_t scratch[kDotGroup * kThreads / 32];
  const int j0 = kDotGroup * blockIdx.y, m = k - j0 < kDotGroup ? k - j0 : kDotGroup;
  fr_t acc[kDotGroup];
#pragma unroll
  for (int j = 0; j < kDotGroup; j++) acc[j] = fr_zero();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const fr_t e = ld_fr(eq + i);
#pragma unroll
    for (int j = 0; j < kDotGroup; j++)
      if (j < m) acc[j] = fr_add(acc[j], fr_mul(e, ld_fr(static_cast<const fr_t*>(in.p[j0 + j]) + i)));
  }
  block_sum_fr<kDotGroup>(acc, scratch);
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < kDotGroup; j++)
      if (j < m) partial[(size_t)(j0 + j) * gridDim.x + blockIdx.x] = acc[j];
}
void launch_multi_dot_ptrs(const DotPtrs& in, int k, bool u32, const fr_t* eq, size_t n, fr_t* partial, fr_t* out,
                           cudaStream_t st) {
  const int groups = (k + kDotGroup - 1) / kDotGroup;
  int per = kMaxBlocks / groups;
  if (per < 1) per = 1;
  const int bx = grid_for(n, kThreads, per);
  const dim3 grid(bx, groups);
  if (u32)
    launch(multi_dot_ptrs_u32_kernel, grid, kThreads, 0, st, in, k, eq, n, partial);
  else
    launch(multi_dot_ptrs_fr_kernel, grid, kThreads, 0, st, in, k, eq, n, partial);
  launch(reduce_partials_kernel, k, kThreads, 0, st, partial, bx, out);
}

// memory_checking.rs:249-252: hash(a, v, t) = t*gamma^2 + v*gamma + a - tau
__global__ void __launch_bounds__(kThreads)
    fp_mem_kernel(const fr_t* table, const fr_t* final_fr, size_t M, int G, int g, fr_t gamma, fr_t gamma2, fr_t tau,
                  fr_t* out_init, fr_t* out_final) {
  // M = local cells; local cell i is global address i*G + g (low-bit partition); `table` is the full table
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (size_t)gridDim.x * blockDim.x) {
    size_t gi = i * G + g;
    fr_t h0 = fr_sub(fr_add(fr_mul(ld_fr(table + gi), gamma), fr_from_u64(gi)), tau);  // ts = 0
    st_fr(out_init + i, h0);
    st_fr(out_final + i, fr_add(h0, fr_mul(ld_fr(final_fr + i), gamma2)));
  }
}
__global__ void __launch_bounds__(kThreads)
    fp_ops_kernel(const fr_t* dim_fr, const fr_t* E_fr, const fr_t* read_fr, size_t s, fr_t gamma, fr_t gamma2,
                  fr_t tau, fr_t* out_read, fr_t* out_write) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < s; i += (size_t)gridDim.x * blockDim.x) {
    fr_t av = fr_sub(fr_add(fr_mul(ld_fr_stream(E_fr + i), gamma), ld_fr_stream(dim_fr + i)), tau);
    fr_t hr = fr_add(av, fr_mul(ld_fr_stream(read_fr + i), gamma2));
    st_fr(out_read + i, hr);
    st_fr(out_write + i, fr_add(hr, gamma2));  // write ts = read ts + 1
  }
}
void launch_gp_fingerprints_mem(const fr_t* table, const fr_t* final_fr, size_t M_local, int G, int g,
                                const fr_t& gamma, const fr_t& tau, fr_t* out_init, fr_t* out_final, cudaStream_t st) {
  launch(fp_mem_kernel, grid_for(M_local), kThreads, 0, st, table, final_fr, M_local, G, g, gamma, fr_sqr(gamma), tau,
         out_init, out_final);
}
void launch_gp_fingerprints_ops(const fr_t* dim_fr, const fr_t* E_fr, const fr_t* read_fr, size_t s,
                                const fr_t& gamma, const fr_t& tau, fr_t* out_read, fr_t* out_write,
                                cudaStream_t st) {
  launch(fp_ops_kernel, grid_for(s), kThreads, 0, st, dim_fr, E_fr, read_fr, s, gamma, fr_sqr(gamma), tau, out_read,
         out_write);
}

// grand_product.rs:20-58, all product trees of one size at once (single GPU).  A tree is one contiguous array: layer 0 (N elements),
// then layer 1 (N/2), ...; layer k+1[i] = layer k[i] * layer k[i + len/2].  One launch per layer for every
// tree (blockIdx.y) while the layers are large, then ONE CTA per tree walks the remaining small layers with
// a barrier in between and publishes the two elements of the top layer (grand_product.rs:60-65 `evaluate`)
// as tagged values 2*slot0 + 2*tree + {0, 1}: ~16 launches per proof instead of ~270 + 16 small copies.
// stop_len = 2: a whole tree (single GPU).  stop_len = 1: the tree of a low-bit SHARD (N = local length) — the walk ends
// with the rank's single element of the layer of global length G, published as value slot0 + tree.
__global__ void __launch_bounds__(kThreads) product_layers_kernel(TreePtrs trees, size_t in_off, size_t n_out) {
  const fr_t* in = trees.p[blockIdx.y] + in_off;
  fr_t* out = trees.p[blockIdx.y] + in_off + 2 * n_out;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += (size_t)gridDim.x * blockDim.x)
    st_fr(out + i, fr_mul(ld_fr(in + i), ld_fr(in + n_out + i)));
}
__global__ void __launch_bounds__(1024)
    product_tail_kernel(TreePtrs trees, size_t off, size_t len, int slot0, int stop_len, Finalize fin) {
  fr_t* base = trees.p[blockIdx.x];
  while (len > (size_t)stop_len) {
    const size_t n_out = len / 2;
    for (size_t i = threadIdx.x; i < n_out; i += blockDim.x)
      st_fr(base + off + len + i, fr_mul(ld_fr(base + off + i), ld_fr(base + off + n_out + i)));
    __syncthreads();
    off += len;
    len = n_out;
  }
  if ((int)threadIdx.x < stop_len)
    finalize_publish(fin, stop_len * (slot0 + (int)blockIdx.x) + (int)threadIdx.x, ld_fr(base + off + threadIdx.x));
}
void launch_product_trees(const TreePtrs& trees, int ntrees, size_t N, int slot0, int stop_len, const Finalize& fin,
                          cudaStream_t st) {
  size_t off = 0, len = N;
  while (len > 4096) {
    const size_t n_out = len / 2;
    dim3 grid(grid_for(n_out, kThreads, kMaxBlocks / ntrees + 1), ntrees);
    launch(product_layers_kernel, grid, kThreads, 0, st, trees, off, n_out);
    off += len;
    len = n_out;
  }
  launch(product_tail_kernel, ntrees, 1024, 0, st, trees, off, len, slot0, stop_len, fin);
}
// layer 1 of a caller's circuit from its polynomial P (layer 0, only read): out[i] = P[i] * P[i + half]
__global__ void __launch_bounds__(kThreads) product_layer1_kernel(const fr_t* P, fr_t* out, size_t half) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (size_t)gridDim.x * blockDim.x)
    st_fr(out + i, fr_mul(ld_fr(P + i), ld_fr(P + half + i)));
}
void launch_product_layer1(const fr_t* P, fr_t* out, size_t half, cudaStream_t st) {
  launch(product_layer1_kernel, grid_for(half), kThreads, 0, st, P, out, half);
}
// last round of a batched cubic sumcheck (one element pair left per array): bind the 2*ncirc heads with r in
// place and publish them — they are the layer's claims (grand_product.rs:139-150)
__global__ void bind_heads_kernel(fr_t* const* AB, int n, fr_t r, Finalize fin) {
  const int k = threadIdx.x;
  if (k >= n) return;
  fr_t* x = AB[k];
  const fr_t lo = ld_fr(x), hi = ld_fr(x + 1);
  const fr_t v = fr_add(lo, fr_mul(r, fr_sub(hi, lo)));
  st_fr(x, v);
  finalize_publish(fin, k, v);
}
void launch_bind_heads(fr_t* const* d_AB, int n, const fr_t& r, const Finalize& fin, cudaStream_t st) {
  launch(bind_heads_kernel, 1, (n + 31) / 32 * 32, 0, st, d_AB, n, r, fin);
}

// ---- Bulletproofs scalar-side helpers (bullet.rs:73-134) ----
__global__ void __launch_bounds__(kThreads) fold_ab_kernel(fr_t* a, fr_t* b, size_t h, fr_t u, fr_t uinv) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < h; i += (size_t)gridDim.x * blockDim.x) {
    fr_t aL = ld_fr(a + i), aR = ld_fr(a + h + i), bL = ld_fr(b + i), bR = ld_fr(b + h + i);
    st_fr(a + i, fr_add(fr_mul(aL, u), fr_mul(uinv, aR)));
    st_fr(b + i, fr_add(fr_mul(bL, uinv), fr_mul(u, bR)));
  }
}
void launch_fold_ab(fr_t* a, fr_t* b, size_t h, const fr_t& u, const fr_t& uinv, cudaStream_t st) {
  launch(fold_ab_kernel, grid_for(h), kThreads, 0, st, a, b, h, u, uinv);
}
__global__ void __launch_bounds__(kThreads) cross_ip_kernel(const fr_t* a, const fr_t* b, size_t h, fr_t* partial) {
  __shared__ fr_t scratch[2 * kThreads / 32];
  fr_t acc[2] = {fr_zero(), fr_zero()};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < h; i += (size_t)gridDim.x * blockDim.x) {
    acc[0] = fr_add(acc[0], fr_mul(ld_fr(a + i), ld_fr(b + h + i)));
    acc[1] = fr_add(acc[1], fr_mul(ld_fr(a + h + i), ld_fr(b + i)));
  }
  block_sum_fr<2>(acc, scratch);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = acc[0];
    partial[gridDim.x + blockIdx.x] = acc[1];
  }
}
void launch_cross_inner_products(const fr_t* a, const fr_t* b, size_t h, fr_t* partial, fr_t* out, cudaStream_t st) {
  int bx = grid_for(h, kThreads, 64);
  launch(cross_ip_kernel, bx, kThreads, 0, st, a, b, h, partial);
  launch(reduce_partials_kernel, 2, kThreads, 0, st, partial, bx, out);
}
__global__ void __launch_bounds__(kThreads)
    expand_weights_kernel(const fr_t* w, fr_t* w_out, size_t n_in, fr_t u, fr_t uinv) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_in; t += (size_t)gridDim.x * blockDim.x) {
    fr_t x = ld_fr(w + t);
    st_fr(w_out + 2 * t, fr_mul(x, uinv));
    st_fr(w_out + 2 * t + 1, fr_mul(x, u));
  }
}
void launch_expand_weights(const fr_t* w, fr_t* w_out, size_t n_in, const fr_t& u, const fr_t& uinv, cudaStream_t st) {
  launch(expand_weights_kernel, grid_for(n_in), kThreads, 0, st, w, w_out, n_in, u, uinv);
}
// Round with current vector length m (half h = m/2) over n original generators, weights w[t], t < n/m.
// Global column j = t*m + pos:   sL[j] = a[pos-h] * w[t] for pos >= h (else 0),
//                                sR[j] = a[h+pos] * w[t] for pos <  h (else 0).
// Sharded over G GPUs this rank owns the columns j = j'*G + g (n_loc of them).  `a` is either this rank's
// low-bit shard of the folded vector (a_rep = 0, valid while m >= 2G: element p lives at p / G) or the
// replicated full vector of the tail rounds (a_rep = 1).
__global__ void __launch_bounds__(kThreads)
    bullet_scalars_kernel(const fr_t* a, const fr_t* w, size_t n_loc, size_t m, int G, int g, int a_rep, fr_t* sL,
                          fr_t* sR) {
  size_t h = m / 2;
  for (size_t jl = (size_t)blockIdx.x * blockDim.x + threadIdx.x; jl < n_loc; jl += (size_t)gridDim.x * blockDim.x) {
    size_t j = jl * G + g;
    size_t t = j / m, pos = j % m;
    fr_t wt = ld_fr(w + t);
    if (pos >= h) {
      size_t idx = pos - h;
      st_fr(sL + jl, fr_mul(ld_fr(a + (a_rep ? idx : idx / G)), wt));
      st_fr(sR + jl, fr_zero());
    } else {
      size_t idx = h + pos;
      st_fr(sL + jl, fr_zero());
      st_fr(sR + jl, fr_mul(ld_fr(a + (a_rep ? idx : idx / G)), wt));
    }
  }
}
void launch_bullet_scalars(const fr_t* a, const fr_t* w, size_t n_loc, size_t m, int G, int g, int a_rep, fr_t* sL,
                           fr_t* sR, cudaStream_t st) {
  launch(bullet_scalars_kernel, grid_for(n_loc), kThreads, 0, st, a, w, n_loc, m, G, g, a_rep, sL, sR);
}
// Two MSM rows over the n + 2 generators (G_0..G_{n-1}, Q, h) in canonical form:
//   row 0 = (k * v[0..n), t00, t01)    row 1 = (0 .. 0, t10, t11)
// i.e. (Cx, Cy) of dot_product.rs:192-197 and (delta, beta) of dot_product.rs:219-230 as ONE two-row MSM.
__global__ void __launch_bounds__(kThreads)
    two_row_scalars_kernel(const fr_t* v, int scale, fr_t k, fr_t t00, fr_t t01, fr_t t10, fr_t t11, size_t n, fr_t* out) {
  const size_t stride = n + 2;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < stride; j += (size_t)gridDim.x * blockDim.x) {
    fr_t r0, r1 = fr_zero();
    if (j < n) {
      fr_t x = ld_fr(v + j);
      r0 = fr_to_canonical(scale ? fr_mul(x, k) : x);
    } else {
      r0 = fr_to_canonical(j == n ? t00 : t01);
      r1 = fr_to_canonical(j == n ? t10 : t11);
    }
    st_fr(out + j, r0);
    st_fr(out + stride + j, r1);
  }
}
void launch_two_row_scalars(const fr_t* v, int scale, const fr_t& k, const fr_t& t00, const fr_t& t01, const fr_t& t10,
                            const fr_t& t11, size_t n, fr_t* out, cudaStream_t st) {
  launch(two_row_scalars_kernel, grid_for(n + 2), kThreads, 0, st, v, scale, k, t00, t01, t10, t11, n, out);
}
__global__ void __launch_bounds__(kThreads) scale_kernel(const fr_t* in, fr_t* out, size_t n, fr_t k) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    st_fr(out + i, fr_mul(ld_fr(in + i), k));
}
void launch_scale(const fr_t* in, fr_t* out, size_t n, const fr_t& k, cudaStream_t st) {
  launch(scale_kernel, grid_for(n), kThreads, 0, st, in, out, n, k);
}

}  // namespace lb
