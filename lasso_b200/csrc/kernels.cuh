// lasso_b200 — launcher interface between the host prover / C-ABI and the CUDA kernels.
// All pointers are device pointers unless named h_*.  Every launcher is asynchronous on
// the given stream.
#pragma once
#include "common.cuh"

namespace lb {

// STRAT_CUSTOM is internal: a caller-defined strategy (lasso_strategy_create), described by a CustomStrategy
enum StrategyKind { STRAT_AND = 0, STRAT_OR = 1, STRAT_XOR = 2, STRAT_LT = 3, STRAT_RANGE = 4, STRAT_CUSTOM = 5 };

// ---- caller-defined strategies: tables as data, combine_lookups as a straight-line program over Fr
// Limits: 2 * alpha circuits must fit one batched grand product (32), the round message (degree + 2 elements) one
// publication region, the program and its constants the shared memory of a CTA.
static constexpr int kCustomMaxMemories = 16, kCustomMaxOps = 128, kCustomMaxConsts = 64, kCustomMaxDegree = 16;
static constexpr int kCustomMaxSlots = 16;  // live intermediate values of a program (after slot allocation)
enum CustomOp { CUSTOM_ADD = 0, CUSTOM_SUB = 1, CUSTOM_MUL = 2, CUSTOM_MULK = 3, CUSTOM_ADDK = 4 };
// One instruction after slot allocation: dst is a physical slot; an operand a (and b for ADD, SUB, MUL) is a physical
// slot when >= 0 and memory value k when it is -1 - k; for MULK and ADDK b indexes the constants.
struct CustomIns {
  int op, dst, a, b;
};
struct CustomStrategy {
  int C, log_m, nsub, alpha, degree;       // degree: the declared g_poly_degree
  int n_ops, n_consts, n_slots;
  int sub[kCustomMaxMemories], dim[kCustomMaxMemories];
  unsigned tbits;                          // bit width of the largest table entry (>= 1, <= 253)
  const CustomIns* d_ops = nullptr;        // device: n_ops instructions
  const fr_t* d_consts = nullptr;          // device: n_consts Montgomery constants
  const fr_t* d_tables_fr = nullptr;       // device: nsub x M Montgomery elements
  const uint32_t* d_tables_u32 = nullptr;  // device: nsub x M values; null when full_width()
  // an entry at or above 2^32: the lookup values are committed and opened from their Montgomery form only
  bool full_width() const { return tbits > 32; }
};

// Runtime stand-in for the reference's `impl SubtableStrategy<F, C, M>` const generics
// (src/subtables/mod.rs:31-93).
struct Strategy {
  int kind, C, log_m, log_r;
  const CustomStrategy* custom = nullptr;  // kind == STRAT_CUSTOM
  int M() const { return 1 << log_m; }
  int num_subtables() const {
    if (kind == STRAT_CUSTOM) return custom->nsub;
    return kind == STRAT_LT ? 2 : (kind == STRAT_RANGE ? 3 : 1);
  }
  int num_memories() const {
    if (kind == STRAT_CUSTOM) return custom->alpha;
    return kind == STRAT_LT ? 2 * C : C;
  }
  int g_poly_degree() const {
    if (kind == STRAT_CUSTOM) return custom->degree;
    return kind == STRAT_LT ? C : 1;
  }
  int sumcheck_poly_degree() const { return g_poly_degree() + 1; }
  // src/subtables/mod.rs:64-74, range_check.rs:62-73
  int memory_to_subtable_index(int i) const {
    if (kind == STRAT_CUSTOM) return custom->sub[i];
    if (kind == STRAT_RANGE) {
      if (i * log_m > log_r) return 2;
      return ((i + 1) * log_m > log_r) ? 1 : 0;
    }
    return i % num_subtables();
  }
  int memory_to_dimension_index(int i) const {
    if (kind == STRAT_CUSTOM) return custom->dim[i];
    return kind == STRAT_RANGE ? i : i / num_subtables();
  }
  // built-in strategies only: a custom one is validated when it is created (capi.cu)
  bool valid() const {
    if (!(kind >= 0 && kind <= 4 && C >= 1 && C <= 16 && log_m >= 2 && log_m <= 24 && (log_m % 2 == 0 || kind == STRAT_RANGE)))
      return false;
    // combine_lookups weights are F::from(1u64 << (i * inc)) (and.rs:45-53, range_check.rs:78-86): the shift must
    // stay below 64 (the debug-build reference panics on overflow); RangeCheck<LOG_R> needs LOG_R >= 0
    if (kind != STRAT_LT && (num_memories() - 1) * (kind == STRAT_RANGE ? log_m : log_m / 2) >= 64) return false;
    if (kind == STRAT_RANGE && log_r < 0) return false;
    return true;
  }
  // valid() and a proof the prover can run: every memory makes two grand-product circuits and one batched grand
  // product holds 32 (CubicCoeffs, TreePtrs), so LT needs C <= 8; the round entry points take C up to 16
  bool provable() const { return valid() && 2 * num_memories() <= 32; }
};

struct FrVec {  // small vector passed by value as a kernel parameter (challenge points, weights)
  fr_t v[32];
};

// ---- K1: bind (dense_mlpoly.rs:209-225) ----
// Z_k[i] <- Z_k[i] + r (Z_k[i+half] - Z_k[i]) for k < npolys, Z_k = base + k*stride, i < half
void launch_bind_top(fr_t* base, size_t stride, int npolys, size_t half, const fr_t& r, cudaStream_t st);
// same over an array of independent device pointers (grand-product circuits)
void launch_bind_top_ptrs(fr_t* const* d_ptrs, int npolys, size_t half, const fr_t& r, cudaStream_t st);
// out of place: d_dst[k][i] <- Z[i] + r (Z[half + i] - Z[i]), Z = d_src[k], k < npolys (device pointer tables)
void launch_bind_ptrs(fr_t* const* d_src, fr_t* const* d_dst, int npolys, size_t half, const fr_t& r, cudaStream_t st);
// out[i] <- Z[2i] + r (Z[2i+1] - Z[2i]), out-of-place
void launch_bind_bot(const fr_t* Z, fr_t* out, size_t half, const fr_t& r, cudaStream_t st);

// ---- K4: eq evals (eq_poly.rs:21-38) ----
// ell <= 11: no scratch.  12..22: the two factor tables, 2 * 4096 elements.  23..28: the low table (4096 elements) and
// the staged high table (2^(ell - 11) elements) after it, 4096 + 2^17 at ell = 28; kEqScratchElems covers every ell <= 28
// with 4096 elements to spare.
static constexpr size_t kEqScratchElems = 4096 + ((size_t)1 << 17) + 4096;
void launch_eq_evals(const FrVec& r, int ell, fr_t* out, fr_t* scratch, cudaStream_t st);

// ---- K2: primary sumcheck round evaluation (sumcheck.rs:179-237) ----
// polys = (alpha+1) arrays of length 2*half at base + k*stride (the last one is eq).
// One launch: the last CTA reduces the block partials and publishes the deg+1 results (see Finalize).
void launch_sumcheck_eval_arbitrary(const Strategy& S, const fr_t* base, size_t stride, size_t half, const Finalize& fin,
                                    cudaStream_t st);
// The previous round's bind (with r) fused with this round's evaluation: base holds polynomials of length 4q, bound
// in place to 2q.  Returns false (nothing launched) when the strategy has no fused kernel or q < min_q (0: the
// default threshold below which a round is latency-bound and two short launches are quicker).
bool launch_sumcheck_bind_eval_arbitrary(const Strategy& S, fr_t* base, size_t stride, size_t q, const fr_t& r,
                                         const Finalize& fin, size_t min_q, cudaStream_t st);
int sumcheck_max_blocks();
// per-device function attributes (dynamic shared memory opt-in of the custom-strategy and combining-function kernels)
void poly_init_device();

// ---- K2 over a caller's polynomials (lasso_sumcheck_prove): g(P_0, .., P_{k-1}) with no eq factor ----
// A combining function g of n_inputs values in the program format of the custom strategies (CustomIns after slot
// allocation); d_ops and d_consts are device copies.
static constexpr int kCombMaxInputs = 16;
struct CombProgram {
  int n_inputs, degree, n_ops, n_consts, n_slots;
  const CustomIns* d_ops;
  const fr_t* d_consts;
};
// the k input polynomials as independent device pointers, passed by value
struct CombPtrs {
  fr_t* p[kCombMaxInputs];
};
// One round (sumcheck.rs:179-237): the degree + 1 sums over i < half of g(x(t)), x_k(t) = lo_k + t (hi_k - lo_k),
// lo_k = in.p[k][i], hi_k = in.p[k][half + i]; one launch, published through fin.
void launch_sumcheck_eval_comb(const CombProgram& g, const CombPtrs& in, size_t half, const Finalize& fin, cudaStream_t st);
// dst.p[k][i] <- src.p[k][i] + r (src.p[k][half + i] - src.p[k][i]) for k < n, i < half; dst == src binds in place
void launch_bind_comb(const CombPtrs& src, const CombPtrs& dst, int n, size_t half, const fr_t& r, cudaStream_t st);
// The bind above from length 4q to 2q fused with the evaluation of the next round over the bound values, one launch.
// Returns false (nothing launched) when q < min_q (0: the default threshold below which two launches are quicker).
bool launch_sumcheck_bind_eval_comb(const CombProgram& g, const CombPtrs& src, const CombPtrs& dst, size_t q, const fr_t& r,
                                    const Finalize& fin, size_t min_q, cudaStream_t st);
// value k < n: src.p[k][0] + r (src.p[k][half] - src.p[k][0]), element 0 of the last bind, published through fin
void launch_final_comb(const CombPtrs& src, int n, size_t half, const fr_t& r, const Finalize& fin, cudaStream_t st);
// out[i] <- g(in.p[0][i], .., in.p[n_inputs-1][i]) for i < n (g.degree is not used)
void launch_comb_map(const CombProgram& g, const CombPtrs& in, size_t n, fr_t* out, cudaStream_t st);

// ---- K3: batched cubic round evaluation (sumcheck.rs:49-93) ----
// A, B: ncirc device pointers each to 2*half elements; Ceq: 2*half elements.  The batching coefficients of
// sumcheck.rs:95-97 are folded in (poly_kernels.cu): out = 3 elements  sum_k coeff_k (e0, e2, e3)_k.  scale != 0: the
// arrays A_k are still unscaled in memory (the first evaluation and the first bind of a layer); the first bind stores
// coeff_k * A_k and later rounds use scale = 0.
struct CubicCoeffs {
  fr_t v[32];
};
void launch_sumcheck_eval_cubic_comb(fr_t* const* d_A, fr_t* const* d_B, const fr_t* Ceq, int ncirc, size_t half,
                                     const CubicCoeffs& cf, int scale, const Finalize& fin, cudaStream_t st);
// fused: bind A_k, B_k (in place) and eq (Cin -> Cout) with r, then evaluate the next round on the bound values;
// h = bound length (>= 2)
void launch_sumcheck_bind_eval_cubic_comb(fr_t* const* d_A, fr_t* const* d_B, const fr_t* Cin, fr_t* Cout, int ncirc, size_t h,
                                          const fr_t& r, const CubicCoeffs& cf, int scale, const Finalize& fin, cudaStream_t st);

// ---- K5: subtables (subtables/*.rs) ----
// tables_fr: nsub x M Montgomery elements; tables_u32: nsub x M raw values.  Built-in strategies only: a custom
// strategy's tables are uploaded once when it is created and used in place.
void launch_materialize_subtables(const Strategy& S, fr_t* tables_fr, uint32_t* tables_u32, cudaStream_t st);
// E_k[j] = T_sub(k)[nz_dim(k)[j]] for k < alpha (subtables/mod.rs:78-92). nz: C x s (u32).
void launch_gather_lookup_polys(const Strategy& S, const fr_t* tables_fr, const uint32_t* tables_u32,
                                const uint32_t* nz, size_t s, fr_t* E_fr, size_t E_stride, uint32_t* E_u32,
                                cudaStream_t st);
// out[i] = F::from(in[i])  (dense_mlpoly.rs:263-269)
void launch_from_u32(const uint32_t* in, fr_t* out, size_t n, cudaStream_t st);
void launch_fill_zero(fr_t* out, size_t n, cudaStream_t st);

// ---- K7: supporting reductions ----
// sum_k eq[k] * g(E_1[k..]) (subtables/mod.rs:186-216)
void launch_sumcheck_claim(const Strategy& S, const fr_t* base, size_t stride, size_t n, fr_t* partial, fr_t* out,
                           cudaStream_t st);
// Over the u32 mirror of an INTEGER-valued polynomial (dim, read, final, E): 8 IMAD per term instead of a Montgomery
// product, 4 B read per element instead of 32 B, one reduction at the end.
// LZ[i] = sum_j L[j] Z[j*R_size + i] (dense_mlpoly.rs:183-207); partial: chunks x R_size scratch
void launch_bound_u32(const uint32_t* Z, const fr_t* L, size_t L_size, size_t R_size, fr_t* partial, fr_t* out, cudaStream_t st);
int bound_max_chunks();
// out[k] = <z_k, eq>, z_k = base + k*stride, k < npolys, n elements each
void launch_multi_dot_u32(const uint32_t* base, size_t stride, int npolys, const fr_t* eq, size_t n, fr_t* partial, fr_t* out,
                          cudaStream_t st);
// the same two over Montgomery Fr polynomials (lookup values of a table of arbitrary field elements)
void launch_bound_fr(const fr_t* Z, const fr_t* L, size_t L_size, size_t R_size, fr_t* partial, fr_t* out, cudaStream_t st);
void launch_multi_dot_fr(const fr_t* base, size_t stride, int npolys, const fr_t* eq, size_t n, fr_t* partial, fr_t* out,
                         cudaStream_t st);
// out[j] = <P_j, eq> for k independent polynomials of n elements each, P_j = in.p[j] (uint32_t* when u32, the integer
// mirrors, else fr_t*), 1 <= k <= kDotMaxPolys.  A thread reads each eq element once per group of kDotGroup inputs.
// Two launches: the dot kernel (ceil(k / kDotGroup) CTA rows, at most kMaxBlocks CTAs) and reduce_partials over k values;
// partial needs k x kMaxBlocks elements.
static constexpr int kDotGroup = 8, kDotMaxPolys = 64;
struct DotPtrs {
  const void* p[kDotMaxPolys];
};
void launch_multi_dot_ptrs(const DotPtrs& in, int k, bool u32, const fr_t* eq, size_t n, fr_t* partial, fr_t* out,
                           cudaStream_t st);
// Reed-Solomon fingerprints (memory_checking.rs:236-310).  init/final over M cells, read/write over s ops.
// M_local cells of this rank; local cell i = global address i*G + g; `table` is the full M-entry table
void launch_gp_fingerprints_mem(const fr_t* table, const fr_t* final_fr, size_t M_local, int G, int g,
                                const fr_t& gamma, const fr_t& tau, fr_t* out_init, fr_t* out_final, cudaStream_t st);
void launch_gp_fingerprints_ops(const fr_t* dim_fr, const fr_t* E_fr, const fr_t* read_fr, size_t s,
                                const fr_t& gamma, const fr_t& tau, fr_t* out_read, fr_t* out_write,
                                cudaStream_t st);
// every product tree of one size N (grand_product.rs:20-58; contiguous layers, see poly_kernels.cu) + tagged publication of the two
// top-layer elements of tree t as values 2*(slot0 + t) + {0, 1}
struct TreePtrs {
  fr_t* p[32];
};
void launch_product_trees(const TreePtrs& trees, int ntrees, size_t N, int slot0, int stop_len, const Finalize& fin,
                          cudaStream_t st);
// layer 1 of a grand-product circuit over a caller's polynomial P of 2*half elements: out[i] = P[i] * P[i + half]
void launch_product_layer1(const fr_t* P, fr_t* out, size_t half, cudaStream_t st);
// x_k[0] <- x_k[0] + r (x_k[1] - x_k[0]) for the n arrays x_k = d_AB[k]; results also published (Finalize)
void launch_bind_heads(fr_t* const* d_AB, int n, const fr_t& r, const Finalize& fin, cudaStream_t st);
// elementwise helpers for the Bulletproofs scalar folds (bullet.rs:125-130)
// a[i] <- a[i]*u + uinv*a[i+h];  b[i] <- b[i]*uinv + u*b[i+h]
void launch_fold_ab(fr_t* a, fr_t* b, size_t h, const fr_t& u, const fr_t& uinv, cudaStream_t st);
// out[0] = <a[0..h), b[h..2h)>, out[1] = <a[h..2h), b[0..h)>  (bullet.rs:78-79)
void launch_cross_inner_products(const fr_t* a, const fr_t* b, size_t h, fr_t* partial, fr_t* out, cudaStream_t st);
// w'[2t] = w[t]*uinv, w'[2t+1] = w[t]*u  (weights of the unfolded generators, see msm_kernels.cu)
void launch_expand_weights(const fr_t* w, fr_t* w_out, size_t n_in, const fr_t& u, const fr_t& uinv, cudaStream_t st);
void launch_two_row_scalars(const fr_t* v, int scale, const fr_t& k, const fr_t& t00, const fr_t& t01, const fr_t& t10,
                            const fr_t& t11, size_t n, fr_t* out, cudaStream_t st);
void launch_bullet_scalars(const fr_t* a, const fr_t* w, size_t n_loc, size_t m, int G, int g, int a_rep, fr_t* sL,
                           fr_t* sR, cudaStream_t st);
void launch_scale(const fr_t* in, fr_t* out, size_t n, const fr_t& k, cudaStream_t st);

// ---- ingest of a caller's dense polynomial (dense_poly_kernels.cu) ----
// dst[i] <- row i of src (4 u64 Montgomery limbs, rows row_stride u64 apart; src == dst with row_stride 4 is allowed);
// flags[0] |= 1 when a row is not a canonical residue (< l), flags[1] = max bit width of the canonical values
void launch_poly_ingest(const uint64_t* src, size_t row_stride, size_t n, fr_t* dst, unsigned* flags, cudaStream_t st);
// out[i] <- the integer value of in[i] (every value below 2^32)
void launch_poly_mirror_u32(const fr_t* in, size_t n, uint32_t* out, cudaStream_t st);

// ---- densify on the GPU (densify_kernels.cu; densified.rs:33-56): stable LSD radix sort by address ----
void densify_init_device();
bool densify_gpu_supported(size_t s, size_t log_m);
size_t densify_scratch_words(size_t s, int C, size_t log_m);
// The index matrix as the extract kernel reads it, on the device: entry (k, i) is p[k * row_stride + i * col_stride]
// (strides in elements), an unsigned integer of elem_bytes = 4 or 8.
struct DzIndices {
  const void* p;
  int elem_bytes;
  size_t row_stride, col_stride;
};
// For entries nobody has range-checked: the extract kernel raises a flag when an entry is >= m (and uses address 0
// instead); launch_densify copies the flag to h_bad (pinned) and records ev right after the extract, before it enqueues
// the rest of the sort.  ev also marks the last read of the index matrix.
struct DzRangeCheck {
  unsigned* h_bad;
  cudaEvent_t ev;
};
// All C dimensions at once; outputs are this rank's shards (rank g of G: accesses k = i*G + g, addresses a = i*G + g):
// dim_i at dim_loc + i*dim_stride, read_i at read_loc + i*read_stride, final_i likewise.  check may be null.
void launch_densify(const DzIndices& idx, const DzRangeCheck* check, size_t n, size_t s, int C, size_t log_m, int G, int g,
                    uint32_t* scratch, uint32_t* dim_loc, size_t dim_stride, uint32_t* read_loc, size_t read_stride,
                    uint32_t* final_loc, size_t final_stride, cudaStream_t st);

}  // namespace lb
