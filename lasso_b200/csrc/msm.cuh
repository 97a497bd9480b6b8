// lasso_b200 — launcher interface of the MSM kernels (msm_kernels.cu).
#pragma once
#include "common.cuh"

namespace lb {

static constexpr int kMsmWindowBits = 8;
static constexpr int kMsmFullWindows = 32;  // 253-bit scalars + signed-digit headroom

// T[w][j] = 2^(8w) * G_j in affine-niels form, w < nwindows, rows `stride` points apart
void launch_build_table(const fq_t* bases_ark, size_t n, pt_niels* T, size_t stride, int nwindows, cudaStream_t st);
// Montgomery -> canonical integers, atomicMax of the bit length into *d_max_bits
void launch_canonicalize(const fr_t* in, fr_t* out, size_t n, unsigned* d_max_bits, cudaStream_t st);
size_t msm_partials_count(int nrows, int ncols, int nw);
// nrows independent MSMs over the same ncols bases.
//   scalars: scalar_limbs == 1 -> u32 integers; == 8 -> canonical 256-bit integers (8 x u32)
//   row r uses scalars[r*row_stride .. +ncols); nw = number of 8-bit windows to process
//   (must cover max_bits + 2; <= 5 for u32, <= 32 for 256-bit)
//   shifted != 0: `table` holds nw window tables (fixed-base); else only window 0 (variable-base)
// Outputs (any may be null): out_ext = nrows x (x,y,t,z) arkworks Montgomery limbs with z = 1;
// out_comp = nrows x 32 bytes ark-serialize compressed; out_raw = nrows x 128 B un-normalised (X,Y,Z,T)
// internal limbs for host-side normalisation (host_fq64.hpp) or the cross-GPU gather-then-add.
// Local column c uses generator index c*col_mul + col_add.
void launch_msm_rows(const pt_niels* table, size_t table_stride, int shifted, const void* scalars, int scalar_limbs,
                     size_t row_stride, int nrows, int ncols, int nw, int col_mul, int col_add, pt_ext* partials,
                     fq_t* out_ext, uint32_t* out_comp, uint32_t* out_raw, cudaStream_t st);
// raw[(k*nrows + row)*32 ..): (X,Y,Z,T) of source k; adds the nsrc sources per row (cross-GPU gather-then-add)
void launch_sum_raw_points(const uint32_t* raw, int nsrc, int nrows, uint32_t* out_raw, uint32_t* out_comp, fq_t* out_ext,
                           cudaStream_t st);
// multiples table M[w][j][d-1] = d * 2^(8w) * G_j (d = 1..128) of the first npts generators, from the window table T
void launch_build_multiples(const pt_niels* T, size_t table_stride, size_t npts, int nwindows, pt_niels* M, cudaStream_t st);
// CTAs per row of a bucket-free MSM over M with len terms per row when heavy_rows of the rows carry non-zero scalars
int msm_direct_chunks(int len, int heavy_rows);
// bucket-free MSM of two short rows over M (msm_kernels.cu): scalars = 2 x len canonical integers, term k of a row
// uses generator k; the CTAs per row are sized for one row carrying the terms; partials: 2 x msm_direct_chunks(len, 1);
// pub: tagged publication to mapped pinned host memory (common.cuh PubDst) — element 3*row + {0,1,2} = canonical
// X, Y, Z; the host waits for the message and clears it (Ctx::wait_points)
void launch_msm_direct(const pt_niels* M, size_t npts, const uint32_t* scalars, int len, pt_ext* partials, const PubDst& pub,
                       cudaStream_t st);
// One Bulletproofs round (bullet.rs:73-134, unfolded generators) in ONE launch over the multiples table: scalars from
// the (folded) a, b, w vectors, both rows L / R summed, tail terms c * Q + blind * h, publication of the two points.
// a_in / b_in: 2m elements when fold != 0 (folded with u / uinv into a_out / b_out, m elements), else m;
// w_in: n / (2m) weights when fold (expanded into w_out, n / m), else n / m.
// partials: 2 * bullet_fused_chunks(n) points; ip_partial: 2 * bullet_fused_chunks(n) elements; counter: zeroed u32.
int bullet_fused_chunks(int n);
void launch_bullet_fused(const pt_niels* M, size_t npts, const fr_t* a_in, const fr_t* b_in, const fr_t* w_in, fr_t* a_out,
                         fr_t* b_out, fr_t* w_out, size_t n, size_t m, int fold, const fr_t& u, const fr_t& uinv,
                         const fr_t& blind_L, const fr_t& blind_R, pt_ext* partials, fr_t* ip_partial, unsigned* counter,
                         const PubDst& pub, cudaStream_t st);
// Hyrax row commitments of integer-valued polynomials as direct sums over the multiples table (no buckets)
// M16 (may be null): 16-bit multiples M16[j][d-1] = d * G_j, d = 1..32768, of the generators 0 .. ncols-1
// local column jl <-> generator jl * col_mul + col_add (one proof sharded over col_mul GPUs: this rank's columns)
void launch_build_multiples16(const pt_niels* T, const pt_niels* M, size_t npts8, size_t ncols, size_t col_mul, size_t col_add,
                              pt_niels* M16, cudaStream_t st);
// K16 (with M16): the centring constant 2^15 * sum_{j < ncols} G_j for exactly this ncols (launch_centre_constant)
void launch_centre_constant(const pt_niels* M16, int ncols, pt_ext* K16, cudaStream_t st);
// M is indexed by generator (local column c -> c * col_mul + col_add), M16 / K16 by LOCAL column
void launch_msm_rows_direct_u32(const pt_niels* M, size_t npts, const pt_niels* M16, const pt_ext* K16, const uint32_t* scalars,
                                size_t row_stride, int nrows, int ncols, int nw, int col_mul, int col_add, pt_ext* partials,
                                fq_t* out_ext, uint32_t* out_comp, uint32_t* out_raw, cudaStream_t st);
// the same rows over Montgomery Fr scalars (made canonical in the kernel), nw signed 8-bit windows over M only: every
// scalar v needs v + sum_{w < nw} 128 * 2^(8w) < 2^(8 nw), which msm_windows_for_bits(bits of v) guarantees; column map
// and outputs as launch_msm_rows_direct_u32
void launch_msm_rows_direct_fr(const pt_niels* M, size_t npts, const fr_t* scalars, size_t row_stride, int nrows, int ncols,
                               int nw, int col_mul, int col_add, pt_ext* partials, fq_t* out_ext, uint32_t* out_comp,
                               uint32_t* out_raw, cudaStream_t st);
void msm_init_device();

// ---- one large variable-base MSM (msm_large.cu): the reference's Pippenger with a large window, buckets in HBM
struct MsmLargePlan {
  size_t n = 0;
  int nbits = 0, c = 0, nw = 0;  // widest scalar, window bits, windows
  uint32_t NB = 0, NB1 = 0;      // buckets per window (|digit| = 1..NB), NB + 1
  int nlev = 0;                  // bucket reduction: levels of running sums over groups of lev_L items
  uint32_t lev_L[8] = {}, lev_n[8] = {};  // group size and number of groups (outputs) per level
  size_t level_pts = 0;          // sum of lev_n
  uint32_t S = 0;                // entries per accumulation unit (a larger bucket is split)
  uint32_t total = 0;            // nw * NB1 counters
  size_t max_entries = 0, max_units = 0;
};
int msm_large_window_bits(size_t n);
// c_force != 0 replaces msm_large_window_bits(n) (tests of the widths the size rule never picks); the small-scalar
// clamp and the limits below still apply
MsmLargePlan msm_large_plan(size_t n, unsigned max_bits, int c_force = 0);
size_t msm_large_scratch_bytes(const MsmLargePlan& p);
void msm_large_init_device();
// bases: arkworks affine (x, y) Montgomery limbs; term i uses base i % n_pool when n_pool != 0 (bench inputs), else base i
void launch_msm_large_prep(const fq_t* bases_ark, const fr_t* scalars_mont, size_t n, size_t n_pool, pt_niels* niels,
                           fr_t* canon, unsigned* d_max_bits, cudaStream_t st);
void launch_msm_large(const MsmLargePlan& p, const pt_niels* niels, const fr_t* canon, void* scratch, fq_t* out_ext,
                      uint32_t* out_raw, cudaStream_t st);
// msm_final.cu: A = nw x nlev level sums; lgL[k] = log2 of level k's group size
void launch_msm_final(const pt_ext* A, int nlev, const int* lgL, int nw, int c, fq_t* out_ext, uint32_t* out_raw, cudaStream_t st);
// independent evaluation for the parity tests: per-term double-and-add + tree sum (partial: kNumSMs * 8 points of scratch)
void launch_msm_naive(const fq_t* bases_ark, const fr_t* scalars_mont, size_t n, size_t n_pool, pt_ext* partial, fq_t* out_ext,
                      cudaStream_t st);

inline int msm_windows_for_bits(unsigned max_bits) {
  int nw = (int)((max_bits + 2 + kMsmWindowBits - 1) / kMsmWindowBits);
  return nw < 1 ? 1 : nw;
}

}  // namespace lb
