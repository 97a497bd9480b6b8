// lasso_b200 — extern "C" boundary (include/lasso_b200.h).  Plain pointers and sizes only; every entry
// point states the reference item it replaces in the header.
#include "../../include/lasso_b200.h"

#include "host_fq64.hpp"
#include "program_check.hpp"
#include "prover.cuh"

using namespace lb;

struct lasso_ctx {
  Ctx* c;
};
struct lasso_gens {
  Gens* g;
};
struct lasso_dense {
  Dense* d;
};
// a caller-defined SubtableStrategy, resident on the context's device
struct lasso_strategy {
  Ctx* c = nullptr;
  CustomStrategy cs;
  DBuf<CustomIns> ops;
  DBuf<fr_t> consts, tables_fr;
  DBuf<uint32_t> tables_u32;
  Strategy S() const {
    Strategy s{STRAT_CUSTOM, cs.C, cs.log_m, 0};
    s.custom = &cs;
    return s;
  }
};

// host objects: a caller's Fiat-Shamir transcript and random tape, continued across calls
struct lasso_transcript {
  Transcript t;
};
struct lasso_random_tape {
  RandomTape t;
};
// PolyCommitmentGens: a generator set of one R = 2^(num_vars - num_vars/2)
struct lasso_poly_gens {
  Gens* g;
  size_t num_vars;
};
struct lasso_poly {
  Poly* p;
};
// a combining function of lasso_sumcheck_prove: a host object
struct lasso_comb {
  Comb g;
};
// MultiCommitGens of the zero-knowledge sumcheck and dot-product proof
struct lasso_mc_gens {
  McGens* g;
};
// GrandProductCircuit over a caller's polynomial (layer 0, not owned); proving binds its layers, so it is proven once
struct lasso_gp_circuit {
  Ctx* c;
  std::unique_ptr<Circuit> ci;
  fr_t product;
  mutable bool proven;
};

struct lasso_msm_job {
  Ctx* c = nullptr;
  size_t n = 0, n_pool = 0;
  DBuf<fq_t> bases;     // n_pool x (x, y) arkworks limbs
  DBuf<fr_t> scalars;   // n Montgomery scalars
  DBuf<pt_niels> niels; // n
  DBuf<fr_t> canon;     // n
  DBuf<uint8_t> scratch;
  DBuf<fq_t> out_ext;
  DBuf<uint32_t> raw;   // (G + 1) x 32 words: partial points of the ranks
  DBuf<pt_ext> naive_part;
  MsmLargePlan plan;    // of the last run
};

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define LB_TRY try {
// every entry point that takes a context makes the context's device current first: a process may hold contexts on
// several GPUs, and kernel launches / allocations go to the CURRENT device
#define LB_TRY_CTX(h) \
  try {               \
    if (!(h) || !(h)->c) return fail(-1, "null context"); \
    LB_CUDA_CHECK(cudaSetDevice((h)->c->device));
#define LB_CATCH                                  \
  }                                               \
  catch (const LbError& e) {                      \
    return fail(e.code, e.what());                \
  }                                               \
  catch (const std::exception& e) {               \
    return fail(-1, e.what());                    \
  }

static bool is_pow2(size_t x) { return x && !(x & (x - 1)); }
static constexpr size_t kMsmLargeMin = 1 << 14;  // below this the row kernels (c = 8, buckets in shared memory) win
static Strategy mkS(int kind, int C, int log_M, int log_R) { return Strategy{kind, C, log_M, log_R}; }

// The output tail of every proof and commitment.  out_room publishes the size the caller must provide and refuses a
// null or short buffer; it runs before anything moves, so a refused call leaves transcripts and tapes as they were.
// timed runs the producing call into one of the context's timers; out_copy checks the produced size and copies it out.
static int out_room(const char* what, size_t need, const uint8_t* out, size_t cap, size_t* out_len) {
  if (out_len) *out_len = need;
  if (!out || cap < need) return fail(LASSO_ERR_LENGTH, std::string(what) + ": output buffer too small");
  return 0;
}
template <class F>
static auto timed(double& ms, F&& produce) {
  const auto t0 = std::chrono::steady_clock::now();
  auto out = produce();
  ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return out;
}
static int out_copy(const char* what, const std::vector<uint8_t>& b, size_t need, uint8_t* out) {
  if (b.size() != need) return fail(-1, std::string(what) + ": unexpected proof size");
  memcpy(out, b.data(), need);
  return 0;
}

// Checks a custom strategy's descriptor and that its tables (of either kind) are there, but not their contents, and
// fills cs with its shape, the degree of g and the instructions with SSA slots mapped to physical slots.  Nulls *out
// first; every failure is LASSO_ERR_STRATEGY.
template <class T>
static int custom_check(int C, int log_m, int nsub, int alpha, const int* sub, const int* dim, const int32_t* prog,
                        int n_ops, const uint64_t* consts, int n_consts, int degree, const T* const* tables,
                        lasso_strategy** out, CustomStrategy& cs, std::vector<CustomIns>& ins) {
  if (out) *out = nullptr;
  auto bad = [](const std::string& why) { return fail(LASSO_ERR_STRATEGY, "strategy: " + why); };
  if (C < 1 || C > 16) return bad("C must be in 1..16");
  if (log_m < 2 || log_m > 24) return bad("log_m must be in 2..24");
  if (alpha < 1 || alpha > kCustomMaxMemories) return bad("num_memories must be in 1..16");
  if (nsub < 1 || nsub > alpha) return bad("num_subtables must be in 1..num_memories");
  if (!sub || !dim || !prog) return bad("null map or program");
  for (int i = 0; i < alpha; i++) {
    if (sub[i] < 0 || sub[i] >= nsub) return bad("memory_to_subtable_index out of range");
    if (dim[i] < 0 || dim[i] >= C) return bad("memory_to_dimension_index out of range");
  }
  int n_slots = 0;
  const std::string why = program_check(alpha, prog, n_ops, consts, n_consts, degree, "g_poly_degree", ins, &n_slots);
  if (!why.empty()) return bad(why);
  if (!out || !tables) return bad("null tables or output");
  for (int k = 0; k < nsub; k++)
    if (!tables[k]) return bad("null table");
  cs = CustomStrategy{};
  cs.C = C;
  cs.log_m = log_m;
  cs.nsub = nsub;
  cs.alpha = alpha;
  cs.degree = degree;
  cs.n_ops = n_ops;
  cs.n_consts = n_consts;
  cs.n_slots = n_slots;
  for (int i = 0; i < alpha; i++) {
    cs.sub[i] = sub[i];
    cs.dim[i] = dim[i];
  }
  return 0;
}

extern "C" {

const char* lasso_last_error(void) { return g_err.c_str(); }

int lasso_ctx_create(lasso_ctx** out, int device_id) {
  LB_TRY
  *out = nullptr;
  Ctx* c = ctx_create(device_id);
  *out = new lasso_ctx{c};
  return 0;
  LB_CATCH
}
void lasso_ctx_destroy(lasso_ctx* ctx) {
  if (!ctx) return;
  try {
    comm_destroy(ctx->c);
  } catch (...) {
  }
  ctx_destroy(ctx->c);
  delete ctx;
}
int lasso_comm_unique_id(uint8_t out[128]) {
  LB_TRY
  comm_unique_id(out);
  return 0;
  LB_CATCH
}
int lasso_ctx_init_comm(lasso_ctx* h, const uint8_t id[128], int rank, int world) {
  LB_TRY_CTX(h)
  comm_init(h->c, id, rank, world);
  return 0;
  LB_CATCH
}

int lasso_ctx_bind_host_threads(lasso_ctx* h) {
  if (!h || !h->c) return -1;
  return bind_host_threads(h->c->device, &h->c->helper_mask, &h->c->have_helper_mask);
}

// one bound_poly_var_top / _bot of a host array: Z[0 .. len/2) receives the bound values
static int bind_host(Ctx* c, uint64_t* Z, size_t len, const uint64_t r[4], bool top) {
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "bind: len must be a power of two >= 2");
  DBuf<fr_t> d(c, len), o(c, top ? 0 : len / 2);  // a top bind is in place
  LB_CUDA_CHECK(cudaMemcpyAsync(d.p, Z, len * 32, cudaMemcpyHostToDevice, c->st));
  fr_t rr;
  memcpy(rr.v, r, 32);
  if (top)
    launch_bind_top(d.p, 0, 1, len / 2, rr, c->st);
  else
    launch_bind_bot(d.p, o.p, len / 2, rr, c->st);
  LB_CUDA_CHECK(cudaMemcpyAsync(Z, top ? d.p : o.p, (len / 2) * 32, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
}
int lasso_bind_top(lasso_ctx* h, uint64_t* Z, size_t len, const uint64_t r[4]) {
  LB_TRY_CTX(h)
  return bind_host(h->c, Z, len, r, true);
  LB_CATCH
}
int lasso_bind_bot(lasso_ctx* h, uint64_t* Z, size_t len, const uint64_t r[4]) {
  LB_TRY_CTX(h)
  return bind_host(h->c, Z, len, r, false);
  LB_CATCH
}
int lasso_eq_evals(lasso_ctx* h, const uint64_t* r, int ell, uint64_t* out) {
  LB_TRY_CTX(h)
  if (ell < 0 || ell > 28) return fail(LASSO_ERR_LENGTH, "eq_evals: 0 <= ell <= 28");
  Ctx* c = h->c;
  FrVec rv;
  for (int i = 0; i < ell; i++) memcpy(rv.v[i].v, r + 4 * i, 32);
  size_t n = (size_t)1 << ell;
  DBuf<fr_t> d(c, n);
  launch_eq_evals(rv, ell, d.p, c->d_eq_scratch, c->st);
  LB_CUDA_CHECK(cudaMemcpyAsync(out, d.p, n * 32, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
  LB_CATCH
}
// one round of the primary sumcheck of a checked strategy: num_memories + 1 host arrays of len elements
static int sumcheck_round(Ctx* c, const Strategy& S, const uint64_t* const* polys, size_t len, uint64_t* evals_out) {
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "len must be a power of two >= 2");
  const int np = S.num_memories() + 1, npts = S.sumcheck_poly_degree() + 1;
  DBuf<fr_t> d(c, (size_t)np * len);
  for (int k = 0; k < np; k++)
    LB_CUDA_CHECK(cudaMemcpyAsync(d.p + (size_t)k * len, polys[k], len * 32, cudaMemcpyHostToDevice, c->st));
  const Finalize f = c->fin_begin();
  launch_sumcheck_eval_arbitrary(S, d.p, len, len / 2, f, c->st);
  c->fin_wait(f, (fr_t*)evals_out, npts);
  return 0;
}
int lasso_sumcheck_round_arbitrary(lasso_ctx* h, int strategy, int C, int log_M, int log_R,
                                   const uint64_t* const* polys, size_t len, uint64_t* evals_out) {
  LB_TRY_CTX(h)
  Strategy S = mkS(strategy, C, log_M, log_R);
  if (!S.valid()) return fail(LASSO_ERR_STRATEGY, "unsupported strategy parameters");
  return sumcheck_round(h->c, S, polys, len, evals_out);
  LB_CATCH
}
int lasso_sumcheck_bind_round_arbitrary(lasso_ctx* h, int strategy, int C, int log_M, int log_R, uint64_t* const* polys,
                                        size_t len, const uint64_t r[4], uint64_t* evals_out) {
  LB_TRY_CTX(h)
  Strategy S = mkS(strategy, C, log_M, log_R);
  if (!S.valid()) return fail(LASSO_ERR_STRATEGY, "unsupported strategy parameters");
  if (!is_pow2(len) || len < 4) return fail(LASSO_ERR_NOT_POW2, "len must be a power of two >= 4");
  Ctx* c = h->c;
  const int np = S.num_memories() + 1, npts = S.sumcheck_poly_degree() + 1;
  DBuf<fr_t> d(c, (size_t)np * len);
  for (int k = 0; k < np; k++)
    LB_CUDA_CHECK(cudaMemcpyAsync(d.p + (size_t)k * len, polys[k], len * 32, cudaMemcpyHostToDevice, c->st));
  fr_t rr;
  memcpy(&rr, r, 32);
  const Finalize f = c->fin_begin();
  if (!launch_sumcheck_bind_eval_arbitrary(S, d.p, len, len / 4, rr, f, 1, c->st)) {
    launch_bind_top(d.p, len, np, len / 2, rr, c->st);
    launch_sumcheck_eval_arbitrary(S, d.p, len, len / 4, f, c->st);
  }
  c->fin_wait(f, (fr_t*)evals_out, npts);
  for (int k = 0; k < np; k++) c->d2h(polys[k], d.p + (size_t)k * len, (len / 2) * 32);
  return 0;
  LB_CATCH
}
int lasso_sumcheck_round_cubic(lasso_ctx* h, int n_circuits, const uint64_t* const* A, const uint64_t* const* B,
                               const uint64_t* Ceq, size_t len, uint64_t* out) {
  LB_TRY_CTX(h)
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "len must be a power of two >= 2");
  if (n_circuits < 1 || n_circuits > 512) return fail(LASSO_ERR_LENGTH, "1 <= n_circuits <= 512");
  Ctx* c = h->c;
  DBuf<fr_t> dA(c, (size_t)n_circuits * len), dB(c, (size_t)n_circuits * len), dC(c, len);
  DBuf<fr_t*> pA(c, n_circuits), pB(c, n_circuits);
  std::vector<fr_t*> hA(n_circuits), hB(n_circuits);
  for (int k = 0; k < n_circuits; k++) {
    hA[k] = dA.p + (size_t)k * len;
    hB[k] = dB.p + (size_t)k * len;
    LB_CUDA_CHECK(cudaMemcpyAsync(hA[k], A[k], len * 32, cudaMemcpyHostToDevice, c->st));
    LB_CUDA_CHECK(cudaMemcpyAsync(hB[k], B[k], len * 32, cudaMemcpyHostToDevice, c->st));
  }
  LB_CUDA_CHECK(cudaMemcpyAsync(dC.p, Ceq, len * 32, cudaMemcpyHostToDevice, c->st));
  LB_CUDA_CHECK(cudaMemcpyAsync(pA.p, hA.data(), n_circuits * sizeof(fr_t*), cudaMemcpyHostToDevice, c->st));
  LB_CUDA_CHECK(cudaMemcpyAsync(pB.p, hB.data(), n_circuits * sizeof(fr_t*), cudaMemcpyHostToDevice, c->st));
  // one circuit at a time through the prover's batched kernels: with scale = 0 no coefficient is applied, so the 3
  // values of a batch of one are that circuit's (e0, e2, e3).  Each message is read before the next launch, so the
  // ring of publication regions never wraps.
  const CubicCoeffs cf = {};
  for (int k = 0; k < n_circuits; k++) {
    const Finalize f = c->fin_begin();
    launch_sumcheck_eval_cubic_comb(pA.p + k, pB.p + k, dC.p, 1, len / 2, cf, 0, f, c->st);
    c->fin_wait(f, (fr_t*)out + 3 * (size_t)k, 3);
  }
  return 0;
  LB_CATCH
}
int lasso_materialize_subtables(lasso_ctx* h, int strategy, int C, int log_M, int log_R, uint64_t* const* tables_out) {
  LB_TRY_CTX(h)
  Strategy S = mkS(strategy, C, log_M, log_R);
  if (!S.valid()) return fail(LASSO_ERR_STRATEGY, "unsupported strategy parameters");
  Ctx* c = h->c;
  size_t M = (size_t)S.M();
  DBuf<fr_t> t(c, M * S.num_subtables());
  launch_materialize_subtables(S, t.p, nullptr, c->st);
  for (int k = 0; k < S.num_subtables(); k++)
    LB_CUDA_CHECK(cudaMemcpyAsync(tables_out[k], t.p + (size_t)k * M, M * 32, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
  LB_CATCH
}
int lasso_gather_lookup_polys(lasso_ctx* h, int strategy, int C, int log_M, int log_R, const uint64_t* const* nz,
                              size_t s, uint64_t* const* E_out) {
  LB_TRY_CTX(h)
  Strategy S = mkS(strategy, C, log_M, log_R);
  if (!S.valid()) return fail(LASSO_ERR_STRATEGY, "unsupported strategy parameters");
  Ctx* c = h->c;
  size_t M = (size_t)S.M();
  std::vector<uint32_t> idx((size_t)C * s);
  for (int d = 0; d < C; d++)
    for (size_t j = 0; j < s; j++) {
      if (nz[d][j] >= M) return fail(LASSO_ERR_INDEX_RANGE, "lookup index out of range");
      idx[(size_t)d * s + j] = (uint32_t)nz[d][j];
    }
  DBuf<fr_t> t(c, M * S.num_subtables()), E(c, (size_t)S.num_memories() * s);
  DBuf<uint32_t> dn(c, (size_t)C * s);
  LB_CUDA_CHECK(cudaMemcpyAsync(dn.p, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, c->st));
  launch_materialize_subtables(S, t.p, nullptr, c->st);
  launch_gather_lookup_polys(S, t.p, nullptr, dn.p, s, E.p, s, nullptr, c->st);
  for (int k = 0; k < S.num_memories(); k++)
    LB_CUDA_CHECK(cudaMemcpyAsync(E_out[k], E.p + (size_t)k * s, s * 32, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
  LB_CATCH
}

// shared by lasso_msm / lasso_commit_rows: variable bases (window-0 table only), Montgomery scalars
static void msm_variable_base(Ctx* c, const uint64_t* bases_affine, size_t nbases, const uint64_t* scalars, size_t nrows,
                              size_t ncols, uint64_t* out_ext) {
  DBuf<fq_t> db(c, nbases * 2);
  DBuf<pt_niels> tab(c, nbases);
  DBuf<fr_t> sc(c, nrows * ncols), canon(c, nrows * ncols);
  LB_CUDA_CHECK(cudaMemcpyAsync(db.p, bases_affine, nbases * 64, cudaMemcpyHostToDevice, c->st));
  LB_CUDA_CHECK(cudaMemcpyAsync(sc.p, scalars, nrows * ncols * 32, cudaMemcpyHostToDevice, c->st));
  launch_build_table(db.p, nbases, tab.p, nbases, 1, c->st);
  LB_CUDA_CHECK(cudaMemsetAsync(c->d_flag, 0, 4, c->st));
  launch_canonicalize(sc.p, canon.p, nrows * ncols, c->d_flag, c->st);
  unsigned max_bits = 0;
  c->d2h(&max_bits, c->d_flag, 4);
  // the reference's small-scalar shortcut (msm/mod.rs:95-106) only changes the schedule, not the result;
  // here the window count simply follows the widest scalar
  int nw = msm_windows_for_bits(max_bits);
  if (nw > kMsmFullWindows) nw = kMsmFullWindows;
  DBuf<pt_ext> part(c, msm_partials_count((int)nrows, (int)ncols, nw));
  DBuf<fq_t> oe(c, nrows * 4);
  if (c->world == 1) {
    launch_msm_rows(tab.p, nbases, 0, canon.p, 8, ncols, (int)nrows, (int)ncols, nw, 1, 0, part.p, oe.p, nullptr, nullptr, c->st);
  } else {
    // collective: every rank passed ITS shard of the terms; partial points are all-gathered and added
    // ("final bucket-sum reduce over NVLink" = gather-then-add, group addition is not an NCCL reduction)
    DBuf<uint32_t> raw(c, (size_t)(c->world + 1) * nrows * 32);
    uint32_t* mine = raw.p + (size_t)c->world * nrows * 32;
    launch_msm_rows(tab.p, nbases, 0, canon.p, 8, ncols, (int)nrows, (int)ncols, nw, 1, 0, part.p, nullptr, nullptr, mine, c->st);
    comm_allgather(c, mine, raw.p, nrows * 128);
    launch_sum_raw_points(raw.p, c->world, (int)nrows, nullptr, nullptr, oe.p, c->st);
  }
  LB_CUDA_CHECK(cudaMemcpyAsync(out_ext, oe.p, nrows * 128, cudaMemcpyDeviceToHost, c->st));
  c->sync();
}
// ---- one large MSM on device-resident inputs (msm_large.cu)
static lasso_msm_job* msm_job_make(Ctx* c, const uint64_t* bases_affine, size_t n_pool, const uint64_t* scalars, size_t n) {
  std::unique_ptr<lasso_msm_job> j(new lasso_msm_job());
  j->c = c;
  j->n = n;
  j->n_pool = n_pool;
  j->bases.alloc(c, n_pool * 2);
  j->scalars.alloc(c, n);
  j->niels.alloc(c, n);
  j->canon.alloc(c, n);
  j->scratch.alloc(c, msm_large_scratch_bytes(msm_large_plan(n, 253)));
  j->out_ext.alloc(c, 4);
  j->raw.alloc(c, (size_t)(c->world + 1) * 32);
  LB_CUDA_CHECK(cudaMemcpyAsync(j->bases.p, bases_affine, n_pool * 64, cudaMemcpyHostToDevice, c->st));
  LB_CUDA_CHECK(cudaMemcpyAsync(j->scalars.p, scalars, n * 32, cudaMemcpyHostToDevice, c->st));
  c->sync();
  return j.release();
}
// one MSM: prep (canonical scalars, niels bases, widest scalar) -> plan -> Pippenger; sharded: every rank's partial
// point is all-gathered and added ("final bucket-sum reduce over NVLink" = gather-then-add)
static void msm_job_once(lasso_msm_job* j) {
  Ctx* c = j->c;
  LB_CUDA_CHECK(cudaMemsetAsync(c->d_flag, 0, 4, c->st));
  launch_msm_large_prep(j->bases.p, j->scalars.p, j->n, j->n_pool == j->n ? 0 : j->n_pool, j->niels.p, j->canon.p, c->d_flag, c->st);
  unsigned max_bits = 0;
  c->d2h(&max_bits, c->d_flag, 4);
  // the reference's small-scalar shortcut (msm/mod.rs:95-106) only changes the schedule, not the result: here the
  // window count simply follows the widest scalar
  j->plan = msm_large_plan(j->n, max_bits);
  if (c->world == 1) {
    launch_msm_large(j->plan, j->niels.p, j->canon.p, j->scratch.p, j->out_ext.p, nullptr, c->st);
    return;
  }
  uint32_t* mine = j->raw.p + (size_t)c->world * 32;
  launch_msm_large(j->plan, j->niels.p, j->canon.p, j->scratch.p, nullptr, mine, c->st);
  comm_allgather(c, mine, j->raw.p, 128);
  launch_sum_raw_points(j->raw.p, c->world, 1, nullptr, nullptr, j->out_ext.p, c->st);
}
int lasso_msm_plan_info(size_t n, unsigned max_bits, int out[16]) {
  LB_TRY
  if (n == 0) return fail(LASSO_ERR_LENGTH, "msm plan: n >= 1");
  const MsmLargePlan p = msm_large_plan(n, max_bits);
  for (int i = 0; i < 16; i++) out[i] = 0;
  out[0] = p.c;
  out[1] = p.nw;
  out[2] = p.nbits;
  out[3] = (int)p.NB;
  out[4] = (int)p.S;
  out[5] = p.nlev;
  for (int k = 0; k < p.nlev && k < 8; k++) out[6 + k] = (int)p.lev_L[k];
  return 0;
  LB_CATCH
}
int lasso_msm_job_create(lasso_ctx* h, const uint64_t* bases_affine, size_t n_pool, const uint64_t* scalars, size_t n,
                         lasso_msm_job** out) {
  LB_TRY_CTX(h)
  *out = nullptr;
  if (n == 0 || n >= ((size_t)1 << 31) || n_pool == 0 || n_pool > n) return fail(LASSO_ERR_LENGTH, "msm job: 1 <= n_pool <= n < 2^31");
  *out = msm_job_make(h->c, bases_affine, n_pool, scalars, n);
  return 0;
  LB_CATCH
}
int lasso_msm_job_run(lasso_ctx* h, lasso_msm_job* j, int iters, double* avg_ms, uint64_t out_xytz[16], int info[8]) {
  LB_TRY_CTX(h)
  if (!j || j->c != h->c || iters < 1) return fail(LASSO_ERR_LENGTH, "msm job: bad arguments");
  Ctx* c = h->c;
  cudaEvent_t e0, e1;
  LB_CUDA_CHECK(cudaEventCreate(&e0));
  LB_CUDA_CHECK(cudaEventCreate(&e1));
  LB_CUDA_CHECK(cudaEventRecord(e0, c->st));
  for (int i = 0; i < iters; i++) msm_job_once(j);
  LB_CUDA_CHECK(cudaEventRecord(e1, c->st));
  LB_CUDA_CHECK(cudaEventSynchronize(e1));
  float ms = 0;
  LB_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (avg_ms) *avg_ms = ms / iters;
  if (out_xytz) {
    LB_CUDA_CHECK(cudaMemcpyAsync(out_xytz, j->out_ext.p, 128, cudaMemcpyDeviceToHost, c->st));
    c->sync();
  }
  if (info) {
    info[0] = j->plan.c;
    info[1] = j->plan.nw;
    info[2] = j->plan.nbits;
    info[3] = (int)j->plan.S;
    info[4] = (int)j->plan.lev_L[0];
    info[5] = j->plan.nlev;
    info[6] = c->world;
    info[7] = 0;
  }
  return 0;
  LB_CATCH
}
int lasso_msm_job_naive(lasso_ctx* h, lasso_msm_job* j, uint64_t out_xytz[16]) {
  LB_TRY_CTX(h)
  if (!j || j->c != h->c) return fail(LASSO_ERR_LENGTH, "msm job: bad arguments");
  Ctx* c = h->c;
  if (c->world > 1) return fail(LASSO_ERR_LENGTH, "msm job: the naive cross-check is single-GPU");
  if (!j->naive_part.p) j->naive_part.alloc(c, (size_t)kNumSMs * 8);
  launch_msm_naive(j->bases.p, j->scalars.p, j->n, j->n_pool == j->n ? 0 : j->n_pool, j->naive_part.p, j->out_ext.p, c->st);
  LB_CUDA_CHECK(cudaMemcpyAsync(out_xytz, j->out_ext.p, 128, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
  LB_CATCH
}
void lasso_msm_job_destroy(lasso_msm_job* j) {
  if (!j) return;
  cudaSetDevice(j->c->device);
  delete j;
}

int lasso_msm(lasso_ctx* h, const uint64_t* bases_affine, const uint64_t* scalars, size_t n, uint64_t out_xytz[16]) {
  LB_TRY_CTX(h)
  if (n == 0 || n > (1u << 30)) return fail(LASSO_ERR_LENGTH, "msm: 1 <= n <= 2^30");
  if (n >= kMsmLargeMin) {  // one large MSM: the large-window Pippenger (msm_large.cu); collective when sharded
    std::unique_ptr<lasso_msm_job> j(msm_job_make(h->c, bases_affine, n, scalars, n));
    msm_job_once(j.get());
    LB_CUDA_CHECK(cudaMemcpyAsync(out_xytz, j->out_ext.p, 128, cudaMemcpyDeviceToHost, h->c->st));
    h->c->sync();
    return 0;
  }
  msm_variable_base(h->c, bases_affine, n, scalars, 1, n, out_xytz);
  return 0;
  LB_CATCH
}
int lasso_commit_rows(lasso_ctx* h, const uint64_t* gens_affine, const uint64_t* Z, size_t L_size, size_t R_size,
                      uint64_t* out_points) {
  LB_TRY_CTX(h)
  if (!L_size || !R_size) return fail(LASSO_ERR_LENGTH, "commit_rows: empty matrix");
  // blind = 0 on this path, so the trailing generator h contributes nothing (commitments.rs:89-92)
  msm_variable_base(h->c, gens_affine, R_size, Z, L_size, R_size, out_points);
  return 0;
  LB_CATCH
}

size_t lasso_gens_points_needed(size_t c, size_t s, size_t num_memories, size_t log_m) {
  return gens_points_needed(c, s, num_memories, log_m);
}
int lasso_sample_generators(const char* label, size_t count, uint64_t* out_affine) {
  LB_TRY
  sample_generators(label, count, out_affine);
  return 0;
  LB_CATCH
}
int lasso_gens_create(lasso_ctx* h, const uint64_t* stream_affine, size_t n_points, size_t c, size_t s,
                      size_t num_memories, size_t log_m, lasso_gens** out) {
  LB_TRY_CTX(h)
  *out = nullptr;
  if (!is_pow2(s)) return fail(LASSO_ERR_NOT_POW2, "s must be a power of two");
  Gens* g = gens_create(h->c, stream_affine, n_points, c, s, num_memories, log_m);
  if (!g) return fail(LASSO_ERR_GENS, "generator stream shorter than lasso_gens_points_needed()");
  *out = new lasso_gens{g};
  return 0;
  LB_CATCH
}
void lasso_gens_destroy(lasso_gens* g) {
  if (!g) return;
  delete g->g;
  delete g;
}

int lasso_densify(lasso_ctx* h, const uint64_t* indices, size_t n_lookups, size_t C, size_t log_m, lasso_dense** out) {
  LB_TRY_CTX(h)
  *out = nullptr;
  Dense* d = timed(h->c->t_densify_ms, [&] { return densify(h->c, indices, n_lookups, C, log_m); });
  *out = new lasso_dense{d};
  return 0;
  LB_CATCH
}
int lasso_densify_device(lasso_ctx* h, const void* indices, size_t elem_bytes, size_t n_lookups, size_t C,
                         size_t row_stride, size_t col_stride, size_t log_m, void* stream, lasso_dense** out) {
  LB_TRY_CTX(h)
  *out = nullptr;
  Dense* d = timed(h->c->t_densify_ms, [&] {
    return densify_device(h->c, indices, elem_bytes, n_lookups, C, row_stride, col_stride, log_m,
                          static_cast<cudaStream_t>(stream));
  });
  *out = new lasso_dense{d};
  return 0;
  LB_CATCH
}
void lasso_dense_destroy(lasso_dense* d) {
  if (!d) return;
  delete d->d;
  delete d;
}
size_t lasso_dense_s(const lasso_dense* d) { return d->d->s; }
size_t lasso_dense_read(lasso_ctx* h, const lasso_dense* dd, int which, uint64_t* out, size_t cap) {
  try {
    const Dense& d = *dd->d;
    Ctx* c = h->c;
    LB_CUDA_CHECK(cudaSetDevice(c->device));
    if (c->world > 1) {  // the arrays hold this rank's low-bit shard only: the field views below do not apply
      g_err = "lasso_dense_read is not available on a sharded context";
      return 0;
    }
    size_t n = 0;
    if (which == 0) {
      n = d.C * d.s;
      if (n > cap) return 0;
      std::vector<uint32_t> tmp(n);
      c->d2h(tmp.data(), d.d_l_u32.p, n * 4);
      for (size_t i = 0; i < n; i++) out[i] = tmp[i];
      return n;
    }
    const fr_t* src = nullptr;
    switch (which) {
      case 1: src = d.d_l_fr.p; n = d.C * d.s; break;
      case 2: src = d.d_l_fr.p + d.C * d.s; n = d.C * d.s; break;
      case 3: src = d.d_m_fr.p; n = d.C * d.m; break;
      case 4: src = d.d_l_fr.p; n = (size_t)1 << d.nv_l; break;
      case 5: src = d.d_m_fr.p; n = (size_t)1 << d.nv_m; break;
      default: return 0;
    }
    if (n > cap) return 0;
    c->d2h(out, src, n * 32);
    return n;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 0;
  }
}

int lasso_commit(lasso_ctx* h, const lasso_dense* d, const lasso_gens* g, uint8_t* out, size_t cap, size_t* out_len) {
  LB_TRY_CTX(h)
  const std::vector<uint8_t> b = timed(h->c->t_commit_ms, [&] { return commit(h->c, *d->d, *g->g); });
  if (const int rc = out_room("commit", b.size(), out, cap, out_len)) return rc;
  return out_copy("commit", b, b.size(), out);
  LB_CATCH
}

// ---- caller-defined strategies
// Uploads a checked strategy: tables_u32 (integers, mirrored into Montgomery form on the device) or tables_fr
// (Montgomery, full width: no u32 copy), exactly one of them non-null.
static int strategy_upload(Ctx* c, CustomStrategy cs, const std::vector<CustomIns>& ins, const uint64_t* constants,
                           int n_constants, const uint32_t* const* tables_u32, const uint64_t* const* tables_fr,
                           lasso_strategy** out) {
  const size_t M = (size_t)1 << cs.log_m;
  std::unique_ptr<lasso_strategy> s(new lasso_strategy());
  s->c = c;
  s->ops.alloc(c, ins.size());
  s->consts.alloc(c, std::max(n_constants, 1));
  s->tables_fr.alloc(c, (size_t)cs.nsub * M);
  if (tables_u32) s->tables_u32.alloc(c, (size_t)cs.nsub * M);
  LB_CUDA_CHECK(cudaMemcpyAsync(s->ops.p, ins.data(), ins.size() * sizeof(CustomIns), cudaMemcpyHostToDevice, c->st));
  if (n_constants)
    LB_CUDA_CHECK(cudaMemcpyAsync(s->consts.p, constants, (size_t)n_constants * 32, cudaMemcpyHostToDevice, c->st));
  if (tables_u32) {
    for (int k = 0; k < cs.nsub; k++)
      LB_CUDA_CHECK(cudaMemcpyAsync(s->tables_u32.p + k * M, tables_u32[k], M * 4, cudaMemcpyHostToDevice, c->st));
    launch_from_u32(s->tables_u32.p, s->tables_fr.p, (size_t)cs.nsub * M, c->st);
  } else {
    for (int k = 0; k < cs.nsub; k++)
      LB_CUDA_CHECK(cudaMemcpyAsync(s->tables_fr.p + k * M, tables_fr[k], M * 32, cudaMemcpyHostToDevice, c->st));
  }
  c->sync();  // the sources are caller memory
  cs.d_ops = s->ops.p;
  cs.d_consts = s->consts.p;
  cs.d_tables_fr = s->tables_fr.p;
  cs.d_tables_u32 = s->tables_u32.p;
  s->cs = cs;
  *out = s.release();
  return 0;
}
int lasso_strategy_create(lasso_ctx* h, int C, int log_m, int num_subtables, const uint32_t* const* tables,
                          int num_memories, const int* mem_to_subtable, const int* mem_to_dimension,
                          const int32_t* program, int n_ops, const uint64_t* constants, int n_constants, int g_degree,
                          lasso_strategy** out) {
  CustomStrategy cs;
  std::vector<CustomIns> ins;
  if (const int rc = custom_check(C, log_m, num_subtables, num_memories, mem_to_subtable, mem_to_dimension, program,
                                  n_ops, constants, n_constants, g_degree, tables, out, cs, ins))
    return rc;
  const size_t M = (size_t)1 << log_m;
  uint32_t mx = 0;
  for (int k = 0; k < num_subtables; k++)
    for (size_t i = 0; i < M; i++) mx = std::max(mx, tables[k][i]);
  cs.tbits = mx ? 32u - (unsigned)__builtin_clz(mx) : 1u;
  LB_TRY_CTX(h)
  return strategy_upload(h->c, cs, ins, constants, n_constants, tables, nullptr, out);
  LB_CATCH
}
int lasso_strategy_create_fr(lasso_ctx* h, int C, int log_m, int num_subtables, const uint64_t* const* tables,
                             int num_memories, const int* mem_to_subtable, const int* mem_to_dimension,
                             const int32_t* program, int n_ops, const uint64_t* constants, int n_constants, int g_degree,
                             lasso_strategy** out) {
  CustomStrategy cs;
  std::vector<CustomIns> ins;
  if (const int rc = custom_check(C, log_m, num_subtables, num_memories, mem_to_subtable, mem_to_dimension, program,
                                  n_ops, constants, n_constants, g_degree, tables, out, cs, ins))
    return rc;
  const size_t M = (size_t)1 << log_m;
  // canonical values: every entry a canonical Montgomery residue; the widest one fixes the commitment's windows
  std::vector<uint32_t> small((size_t)num_subtables * M);
  unsigned bits = 1;
  for (int k = 0; k < num_subtables; k++)
    for (size_t i = 0; i < M; i++) {
      fr_t x;
      memcpy(x.v, tables[k] + 4 * i, 32);
      if (!fr_eq(fr_reduce_once(x.v), x)) return fail(LASSO_ERR_STRATEGY, "strategy: a table entry is not a canonical field element");
      const fr_t v = fr_to_canonical(x);
      for (int l = 7; l >= 0; l--)
        if (v.v[l]) {
          bits = std::max(bits, 32u * (unsigned)l + 32u - (unsigned)__builtin_clz(v.v[l]));
          break;
        }
      small[k * M + i] = v.v[0];
    }
  cs.tbits = bits;
  std::vector<const uint32_t*> rows(num_subtables);
  for (int k = 0; k < num_subtables; k++) rows[k] = small.data() + k * M;
  LB_TRY_CTX(h)
  // entries below 2^32: exactly the strategy lasso_strategy_create makes of those integers
  if (!cs.full_width()) return strategy_upload(h->c, cs, ins, constants, n_constants, rows.data(), nullptr, out);
  return strategy_upload(h->c, cs, ins, constants, n_constants, nullptr, tables, out);
  LB_CATCH
}
void lasso_strategy_destroy(lasso_strategy* s) {
  if (!s) return;
  cudaSetDevice(s->c->device);
  delete s;
}
int lasso_sumcheck_round_custom(lasso_ctx* h, const lasso_strategy* s, const uint64_t* const* polys, size_t len,
                                uint64_t* evals_out) {
  LB_TRY_CTX(h)
  if (!s || s->c != h->c) return fail(LASSO_ERR_STRATEGY, "strategy was created on another context");
  return sumcheck_round(h->c, s->S(), polys, len, evals_out);
  LB_CATCH
}
// ---- lookup proofs, on a caller's transcript and tape or on ones made from labels
static bool load_scalars(const uint64_t* s, size_t n, std::vector<fr_t>& out);
static int poly_ctx_check(lasso_ctx* h);
// The strategy of a built-in kind (strategy, log_R) or a custom one (s), checked against the context and the dense;
// every failure is LASSO_ERR_STRATEGY
static int strategy_for(lasso_ctx* h, int strategy, int log_R, const lasso_strategy* s, const lasso_dense* d,
                        Strategy& S) {
  auto bad = [](const std::string& why) { return fail(LASSO_ERR_STRATEGY, why); };
  if (!d) return bad("null densified representation");
  if (s) {
    if (s->c != h->c) return bad("strategy was created on another context");
    if ((size_t)s->cs.C != d->d->C || (size_t)s->cs.log_m != d->d->log_m)
      return bad("strategy (C, log_m) differ from the densified representation");
    S = s->S();
    return 0;
  }
  S = mkS(strategy, (int)d->d->C, (int)d->d->log_m, log_R);
  if (!S.valid()) return bad("unsupported strategy parameters");
  if (!S.provable())
    return bad("prove: " + std::to_string(2 * S.num_memories()) +
               " grand-product circuits exceed the batch limit of 32 (LT needs C <= 8)");
  return 0;
}
// The generators lasso_gens_create built for this (c, s, num_memories, log_m) (surge.rs:32-58), else LASSO_ERR_GENS.
// shared_gens: generators of another single-GPU context on the same device will do (lasso_prove lets such contexts
// share one set of read-only tables, many GB at 2^20 lookups); otherwise they must be the context's own
static int gens_check(lasso_ctx* h, const Strategy& S, const Dense& dense, const lasso_gens* g, bool shared_gens,
                      const char* what) {
  const size_t alpha = (size_t)S.num_memories();
  const Ctx* gc = g ? g->g->ctx : nullptr;
  const bool shareable = shared_gens && gc && gc->device == h->c->device && gc->world == 1 && h->c->world == 1;
  if (!g || (gc != h->c && !shareable))
    return fail(LASSO_ERR_GENS, std::string(what) + ": null generators, or generators of another context");
  const Gens& gg = *g->g;
  if (gg.c != dense.C || next_pow2(gg.s) != dense.s || gg.num_memories != alpha || gg.log_m != dense.log_m ||
      gg.nv_d != log2_exact_or_ceil(next_pow2(alpha * dense.s)) || gg.nv_l != dense.nv_l || gg.nv_m != dense.nv_m)
    return fail(LASSO_ERR_GENS, std::string(what) + ": generators built for another (c, s, num_memories, log_m)");
  return 0;
}
// shared_gens: as gens_check; generators of another single-GPU context on the same device will do (lasso_prove lets such contexts
// share one set of read-only tables, many GB at 2^20 lookups); otherwise they must be the context's own
static int prove_transcript(lasso_ctx* h, const Strategy& S, lasso_dense* d, const uint64_t* r, size_t r_len,
                            const lasso_gens* g, bool shared_gens, lasso_transcript* transcript, lasso_random_tape* tape,
                            uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t claimed_eval_out[4]) {
  const Dense& dense = *d->d;
  if (!transcript || !tape || !proof_len) return fail(LASSO_ERR_LENGTH, "prove: null transcript, random tape or proof_len");
  if (r_len != log2_exact_or_ceil(dense.s)) return fail(LASSO_ERR_LENGTH, "r.len() != log2(s)");  // surge.rs:131
  if (r_len && !r) return fail(LASSO_ERR_LENGTH, "prove: null point");
  if (const int rc = gens_check(h, S, dense, g, shared_gens, "prove")) return rc;
  const Gens& gg = *g->g;
  const size_t need = proof_bytes(S, dense, gg);
  if (const int rc = out_room("prove", need, proof_out, proof_cap, proof_len)) return rc;
  std::vector<fr_t> rv;
  if (!load_scalars(r, r_len, rv)) return fail(LASSO_ERR_VALUE, "prove: a coordinate of r is not a canonical residue");
  fr_t claimed;
  const std::vector<uint8_t> b =
      timed(h->c->t_prove_ms, [&] { return prove(h->c, S, *d->d, rv, gg, transcript->t, tape->t, &claimed); });
  if (const int rc = out_copy("prove", b, need, proof_out)) return rc;
  if (claimed_eval_out) memcpy(claimed_eval_out, claimed.v, 32);
  return 0;
}
// lasso_prove / lasso_prove_custom: prove_transcript on Transcript::new(transcript_label), which records every
// challenge it draws, and on RandomTape::new(tape_label) seeded with tape_seed
static int prove_labels(lasso_ctx* h, const Strategy& S, lasso_dense* d, const uint64_t* r, size_t r_len,
                        const lasso_gens* g, const char* transcript_label, const char* tape_label,
                        const uint64_t tape_seed[4], uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                        uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges) {
  if (!transcript_label || !tape_label || !tape_seed) return fail(LASSO_ERR_LENGTH, "prove: null label or tape seed");
  std::vector<fr_t> seed, trace;
  if (!load_scalars(tape_seed, 1, seed)) return fail(LASSO_ERR_VALUE, "prove: the tape seed is not a canonical residue");
  lasso_transcript transcript{Transcript(transcript_label)};
  transcript.t.trace = &trace;
  lasso_random_tape tape{RandomTape(tape_label, seed[0])};
  if (const int rc =
          prove_transcript(h, S, d, r, r_len, g, true, &transcript, &tape, proof_out, proof_cap, proof_len, nullptr))
    return rc;
  if (n_challenges) *n_challenges = trace.size();
  if (challenges_out)
    for (size_t i = 0; i < trace.size() && i < challenges_cap; i++) memcpy(challenges_out + 4 * i, trace[i].v, 32);
  return 0;
}
int lasso_prove(lasso_ctx* h, int strategy, int log_R, lasso_dense* d, const uint64_t* r, size_t r_len,
                const lasso_gens* g, const char* transcript_label, const char* tape_label, const uint64_t tape_seed[4],
                uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t* challenges_out,
                size_t challenges_cap, size_t* n_challenges) {
  LB_TRY_CTX(h)
  Strategy S{};
  if (const int rc = strategy_for(h, strategy, log_R, nullptr, d, S)) return rc;
  return prove_labels(h, S, d, r, r_len, g, transcript_label, tape_label, tape_seed, proof_out, proof_cap, proof_len,
                      challenges_out, challenges_cap, n_challenges);
  LB_CATCH
}
int lasso_prove_custom(lasso_ctx* h, const lasso_strategy* s, lasso_dense* d, const uint64_t* r, size_t r_len,
                       const lasso_gens* g, const char* transcript_label, const char* tape_label,
                       const uint64_t tape_seed[4], uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                       uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges) {
  LB_TRY_CTX(h)
  if (!s) return fail(LASSO_ERR_STRATEGY, "null strategy");
  Strategy S{};
  if (const int rc = strategy_for(h, 0, 0, s, d, S)) return rc;
  return prove_labels(h, S, d, r, r_len, g, transcript_label, tape_label, tape_seed, proof_out, proof_cap, proof_len,
                      challenges_out, challenges_cap, n_challenges);
  LB_CATCH
}
int lasso_prove_transcript(lasso_ctx* h, int strategy, int log_R, lasso_dense* d, const uint64_t* r, size_t r_len,
                           const lasso_gens* g, lasso_transcript* transcript, lasso_random_tape* random_tape,
                           uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t claimed_eval_out[4]) {
  LB_TRY_CTX(h)
  Strategy S{};
  if (const int rc = strategy_for(h, strategy, log_R, nullptr, d, S)) return rc;
  return prove_transcript(h, S, d, r, r_len, g, false, transcript, random_tape, proof_out, proof_cap, proof_len,
                          claimed_eval_out);
  LB_CATCH
}
int lasso_prove_custom_transcript(lasso_ctx* h, const lasso_strategy* s, lasso_dense* d, const uint64_t* r, size_t r_len,
                                  const lasso_gens* g, lasso_transcript* transcript, lasso_random_tape* random_tape,
                                  uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t claimed_eval_out[4]) {
  LB_TRY_CTX(h)
  if (!s) return fail(LASSO_ERR_STRATEGY, "null strategy");
  Strategy S{};
  if (const int rc = strategy_for(h, 0, 0, s, d, S)) return rc;
  return prove_transcript(h, S, d, r, r_len, g, false, transcript, random_tape, proof_out, proof_cap, proof_len,
                          claimed_eval_out);
  LB_CATCH
}
static int dense_outputs_checked(lasso_ctx* h, int strategy, int log_R, const lasso_strategy* s, const lasso_dense* d,
                                 lasso_poly** out) {
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!out) return fail(LASSO_ERR_LENGTH, "outputs: null output");
  Strategy S{};
  if (const int rc = strategy_for(h, strategy, log_R, s, d, S)) return rc;
  *out = new lasso_poly{dense_outputs(h->c, S, *d->d)};
  return 0;
}
int lasso_dense_outputs(lasso_ctx* h, int strategy, int log_R, const lasso_dense* d, lasso_poly** out) {
  LB_TRY_CTX(h)
  return dense_outputs_checked(h, strategy, log_R, nullptr, d, out);
  LB_CATCH
}
int lasso_dense_outputs_custom(lasso_ctx* h, const lasso_strategy* s, const lasso_dense* d, lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (!s) return fail(LASSO_ERR_STRATEGY, "outputs: null strategy");
  return dense_outputs_checked(h, 0, 0, s, d, out);
  LB_CATCH
}

// ---- memory checking inside a caller's protocol (single GPU): Subtables::new, the densified polynomials,
// MemoryCheckingProof::prove and GrandProducts::new over a caller's memory
static int lookup_polys_checked(lasso_ctx* h, int strategy, int log_R, const lasso_strategy* s, const lasso_dense* d,
                                lasso_poly** out, size_t n_out) {
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  Strategy S{};
  if (const int rc = strategy_for(h, strategy, log_R, s, d, S)) return rc;
  if (!out || n_out != (size_t)S.num_memories())
    return fail(LASSO_ERR_LENGTH, "lookup polys: null output, or n_out != num_memories (" +
                                      std::to_string(S.num_memories()) + ")");
  for (size_t i = 0; i < n_out; i++) out[i] = nullptr;
  const std::vector<Poly*> ps = lookup_polys(h->c, S, *d->d);
  for (size_t i = 0; i < n_out; i++) out[i] = new lasso_poly{ps[i]};
  return 0;
}
int lasso_lookup_polys(lasso_ctx* h, int strategy, int log_R, const lasso_dense* d, lasso_poly** out, size_t n_out) {
  LB_TRY_CTX(h)
  return lookup_polys_checked(h, strategy, log_R, nullptr, d, out, n_out);
  LB_CATCH
}
int lasso_lookup_polys_custom(lasso_ctx* h, const lasso_strategy* s, const lasso_dense* d, lasso_poly** out,
                              size_t n_out) {
  LB_TRY_CTX(h)
  if (!s) return fail(LASSO_ERR_STRATEGY, "lookup polys: null strategy");
  return lookup_polys_checked(h, 0, 0, s, d, out, n_out);
  LB_CATCH
}
int lasso_dense_poly(lasso_ctx* h, const lasso_dense* d, int which, size_t j, lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!d) return fail(LASSO_ERR_STRATEGY, "dense poly: null densified representation");
  if (!out) return fail(LASSO_ERR_LENGTH, "dense poly: null output");
  if (which < 1 || which > 3 || j >= d->d->C)
    return fail(LASSO_ERR_LENGTH, "dense poly: which must be 1 (dim), 2 (read) or 3 (final), and j < C");
  *out = new lasso_poly{dense_poly(h->c, *d->d, which, j)};
  return 0;
  LB_CATCH
}
static int memory_check_checked(lasso_ctx* h, int strategy, int log_R, const lasso_strategy* s, const lasso_dense* d,
                                const uint64_t gamma[4], const uint64_t tau[4], const lasso_gens* g,
                                lasso_transcript* transcript, lasso_random_tape* tape, uint8_t* proof_out,
                                size_t proof_cap, size_t* proof_len) {
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  Strategy S{};
  if (const int rc = strategy_for(h, strategy, log_R, s, d, S)) return rc;
  const Dense& dense = *d->d;
  if (!transcript || !tape || !proof_len || !gamma || !tau)
    return fail(LASSO_ERR_LENGTH, "memory check: null transcript, random tape, gamma, tau or proof_len");
  if (const int rc = gens_check(h, S, dense, g, false, "memory check")) return rc;
  const size_t need = memory_check_bytes(S, dense, *g->g);
  if (const int rc = out_room("memory check", need, proof_out, proof_cap, proof_len)) return rc;
  std::vector<fr_t> gv, tv;
  if (!load_scalars(gamma, 1, gv) || !load_scalars(tau, 1, tv))
    return fail(LASSO_ERR_VALUE, "memory check: gamma or tau is not a canonical residue");
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return memory_check_prove(h->c, S, dense, gv[0], tv[0], *g->g, transcript->t, tape->t);
  });
  return out_copy("memory check", b, need, proof_out);
}
int lasso_memory_check_prove(lasso_ctx* h, int strategy, int log_R, const lasso_dense* d, const uint64_t gamma[4],
                             const uint64_t tau[4], const lasso_gens* g, lasso_transcript* transcript,
                             lasso_random_tape* random_tape, uint8_t* proof_out, size_t proof_cap, size_t* proof_len) {
  LB_TRY_CTX(h)
  return memory_check_checked(h, strategy, log_R, nullptr, d, gamma, tau, g, transcript, random_tape, proof_out,
                              proof_cap, proof_len);
  LB_CATCH
}
int lasso_memory_check_prove_custom(lasso_ctx* h, const lasso_strategy* s, const lasso_dense* d,
                                    const uint64_t gamma[4], const uint64_t tau[4], const lasso_gens* g,
                                    lasso_transcript* transcript, lasso_random_tape* random_tape, uint8_t* proof_out,
                                    size_t proof_cap, size_t* proof_len) {
  LB_TRY_CTX(h)
  if (!s) return fail(LASSO_ERR_STRATEGY, "memory check: null strategy");
  return memory_check_checked(h, 0, 0, s, d, gamma, tau, g, transcript, random_tape, proof_out, proof_cap, proof_len);
  LB_CATCH
}
static int poly_array(lasso_ctx* h, const char* what, const lasso_poly* const* polys, size_t n, bool same_nv,
                      std::vector<const Poly*>& ps);
int lasso_memory_fingerprints(lasso_ctx* h, const lasso_poly* table, const lasso_poly* dim, const lasso_poly* read,
                              const lasso_poly* final_ts, const uint64_t gamma[4], const uint64_t tau[4],
                              lasso_poly* out[4]) {
  LB_TRY_CTX(h)
  if (out)
    for (int k = 0; k < 4; k++) out[k] = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  const lasso_poly* in[4] = {table, dim, read, final_ts};
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "fingerprints", in, 4, false, ps)) return rc;
  const Poly &T = *ps[0], &D = *ps[1], &R = *ps[2], &F = *ps[3];
  if (T.len != F.len || T.len < 2) return fail(LASSO_ERR_LENGTH, "fingerprints: table and final_ts must be of one length M >= 2");
  if (D.len != R.len || D.len < 2) return fail(LASSO_ERR_LENGTH, "fingerprints: dim and read must be of one length s >= 2");
  if (!out || !gamma || !tau) return fail(LASSO_ERR_LENGTH, "fingerprints: null gamma, tau or output");
  // dim.bits <= log2 M: every address is an integer below M, and dim has the u32 mirror the gather reads
  if (D.bits > T.nv || !D.d_u32.p) return fail(LASSO_ERR_INDEX_RANGE, "fingerprints: dim must hold integers below M");
  std::vector<fr_t> gv, tv;
  if (!load_scalars(gamma, 1, gv) || !load_scalars(tau, 1, tv))
    return fail(LASSO_ERR_VALUE, "fingerprints: gamma or tau is not a canonical residue");
  Poly* o[4];
  memory_fingerprints(h->c, T, D, R, F, gv[0], tv[0], o);
  for (int k = 0; k < 4; k++) out[k] = new lasso_poly{o[k]};
  return 0;
  LB_CATCH
}

// ---- transcripts and random tapes (host only: no context, no device)
#define LB_TRY_T(t) \
  try {             \
    if (!(t)) return fail(LASSO_ERR_LENGTH, "null transcript");
int lasso_transcript_create(const char* label, lasso_transcript** out) {
  LB_TRY
  if (!out || !label) return fail(LASSO_ERR_LENGTH, "transcript: null label or output");
  *out = new lasso_transcript{Transcript(label)};
  return 0;
  LB_CATCH
}
void lasso_transcript_destroy(lasso_transcript* t) { delete t; }
int lasso_transcript_append_message(lasso_transcript* t, const char* label, const uint8_t* msg, size_t len) {
  LB_TRY_T(t)
  if (len && !msg) return fail(LASSO_ERR_LENGTH, "transcript: null message");
  t->t.append_message(label, msg, len);
  return 0;
  LB_CATCH
}
int lasso_transcript_append_u64(lasso_transcript* t, const char* label, uint64_t x) {
  LB_TRY_T(t)
  t->t.append_u64(label, x);
  return 0;
  LB_CATCH
}
int lasso_transcript_append_protocol_name(lasso_transcript* t, const char* name) {
  LB_TRY_T(t)
  t->t.append_protocol_name(name);
  return 0;
  LB_CATCH
}
// the scalars of the caller are Montgomery limbs; a non-canonical one would serialise to another residue's bytes
static bool load_scalars(const uint64_t* s, size_t n, std::vector<fr_t>& out) {
  out.resize(n);
  for (size_t i = 0; i < n; i++) {
    memcpy(out[i].v, s + 4 * i, 32);
    if (!fr_eq(fr_reduce_once(out[i].v), out[i])) return false;
  }
  return true;
}
int lasso_transcript_append_scalar(lasso_transcript* t, const char* label, const uint64_t s[4]) {
  LB_TRY_T(t)
  std::vector<fr_t> v;
  if (!load_scalars(s, 1, v)) return fail(LASSO_ERR_VALUE, "transcript: the scalar is not a canonical residue");
  t->t.append_scalar(label, v[0]);
  return 0;
  LB_CATCH
}
int lasso_transcript_append_scalars(lasso_transcript* t, const char* label, const uint64_t* s, size_t n) {
  LB_TRY_T(t)
  std::vector<fr_t> v;
  if (n && !s) return fail(LASSO_ERR_LENGTH, "transcript: null scalars");
  if (!load_scalars(s, n, v)) return fail(LASSO_ERR_VALUE, "transcript: a scalar is not a canonical residue");
  t->t.append_scalars(label, v.data(), n);
  return 0;
  LB_CATCH
}
int lasso_transcript_append_point(lasso_transcript* t, const char* label, const uint8_t point[32]) {
  LB_TRY_T(t)
  t->t.append_point_compressed(label, point);
  return 0;
  LB_CATCH
}
int lasso_transcript_append_points(lasso_transcript* t, const char* label, const uint8_t* points, size_t n) {
  LB_TRY_T(t)
  if (n && !points) return fail(LASSO_ERR_LENGTH, "transcript: null points");
  t->t.append_message(label, std::string("begin_append_vector"));
  for (size_t i = 0; i < n; i++) t->t.append_point_compressed(label, points + 32 * i);
  t->t.append_message(label, std::string("end_append_vector"));
  return 0;
  LB_CATCH
}
int lasso_transcript_append_poly_commitment(lasso_transcript* t, const char* label, const uint8_t* bytes, size_t len) {
  LB_TRY_T(t)
  uint64_t n = 0;
  if (!bytes || len < 8) return fail(LASSO_ERR_LENGTH, "poly commitment: shorter than its count");
  memcpy(&n, bytes, 8);
  if (n > (len - 8) / 32 || len != 8 + 32 * n) return fail(LASSO_ERR_LENGTH, "poly commitment: length != 8 + 32 * count");
  t->t.append_message(label, std::string("poly_commitment_begin"));
  for (uint64_t i = 0; i < n; i++) t->t.append_point_compressed("poly_commitment_share", bytes + 8 + 32 * i);
  t->t.append_message(label, std::string("poly_commitment_end"));
  return 0;
  LB_CATCH
}
int lasso_transcript_append_sparse_commitment(lasso_transcript* t, const uint8_t* bytes, size_t len) {
  LB_TRY_T(t)
  if (!bytes && len) return fail(LASSO_ERR_LENGTH, "sparse commitment: null bytes");
  // lasso_commit's bytes: two (u64 count, 32 bytes per point) vectors, then s, log_m, m
  size_t at = 0, begin[2], count[2];
  for (int v = 0; v < 2; v++) {
    uint64_t n = 0;
    if (len - at < 8) return fail(LASSO_ERR_LENGTH, "sparse commitment: shorter than its counts");
    memcpy(&n, bytes + at, 8);
    at += 8;
    if (n > (len - at) / 32) return fail(LASSO_ERR_LENGTH, "sparse commitment: a count exceeds the bytes");
    begin[v] = at;
    count[v] = n;
    at += 32 * n;
  }
  if (len - at != 24) return fail(LASSO_ERR_LENGTH, "sparse commitment: not followed by exactly s, log_m, m");
  for (int v = 0; v < 2; v++)
    for (size_t i = 0; i < count[v]; i++)
      if (!h64::decompresses(bytes + begin[v] + 32 * i))
        return fail(LASSO_ERR_VALUE, "sparse commitment: a point does not decompress");
  // SparsePolynomialCommitment::append_to_transcript (surge.rs:70-82)
  static const char* const labels[2] = {"l_variate_polys_commitment", "log_m_variate_polys_commitment"};
  for (int v = 0; v < 2; v++) {
    t->t.append_message(labels[v], std::string("poly_commitment_begin"));
    for (size_t i = 0; i < count[v]; i++) t->t.append_point_compressed("poly_commitment_share", bytes + begin[v] + 32 * i);
    t->t.append_message(labels[v], std::string("poly_commitment_end"));
  }
  static const char* const fields[3] = {"s", "log_m", "m"};
  for (int k = 0; k < 3; k++) {
    uint64_t x;
    memcpy(&x, bytes + at + 8 * k, 8);
    t->t.append_u64(fields[k], x);
  }
  return 0;
  LB_CATCH
}
int lasso_transcript_append_combined_table_commitment(lasso_transcript* t, const char* label, const uint8_t* bytes,
                                                      size_t len) {
  LB_TRY_T(t)
  if (!label) return fail(LASSO_ERR_LENGTH, "combined table commitment: null label");
  uint64_t n = 0;
  if (!bytes || len < 8) return fail(LASSO_ERR_LENGTH, "combined table commitment: shorter than its count");
  memcpy(&n, bytes, 8);
  if (n > (len - 8) / 32 || len != 8 + 32 * n)
    return fail(LASSO_ERR_LENGTH, "combined table commitment: length != 8 + 32 * count");
  for (uint64_t i = 0; i < n; i++)
    if (!h64::decompresses(bytes + 8 + 32 * i))
      return fail(LASSO_ERR_VALUE, "combined table commitment: a point does not decompress");
  // CombinedTableCommitment::append_to_transcript (subtables/mod.rs:382-393)
  t->t.append_message("subtable_evals_commitment", std::string("begin_subtable_evals_commitment"));
  t->t.append_message(label, std::string("poly_commitment_begin"));
  for (uint64_t i = 0; i < n; i++) t->t.append_point_compressed("poly_commitment_share", bytes + 8 + 32 * i);
  t->t.append_message(label, std::string("poly_commitment_end"));
  t->t.append_message("subtable_evals_commitment", std::string("end_subtable_evals_commitment"));
  return 0;
  LB_CATCH
}
int lasso_transcript_challenge_scalar(lasso_transcript* t, const char* label, uint64_t out[4]) {
  LB_TRY_T(t)
  const fr_t c = t->t.challenge_scalar(label);
  memcpy(out, c.v, 32);
  return 0;
  LB_CATCH
}
int lasso_transcript_challenge_vector(lasso_transcript* t, const char* label, size_t n, uint64_t* out) {
  LB_TRY_T(t)
  if (n && !out) return fail(LASSO_ERR_LENGTH, "transcript: null output");
  for (size_t i = 0; i < n; i++) {
    const fr_t c = t->t.challenge_scalar(label);
    memcpy(out + 4 * i, c.v, 32);
  }
  return 0;
  LB_CATCH
}
int lasso_random_tape_create(const char* label, const uint64_t seed[4], lasso_random_tape** out) {
  LB_TRY
  if (!out || !label || !seed) return fail(LASSO_ERR_LENGTH, "random tape: null label, seed or output");
  std::vector<fr_t> s;
  if (!load_scalars(seed, 1, s)) return fail(LASSO_ERR_VALUE, "random tape: the seed is not a canonical residue");
  *out = new lasso_random_tape{RandomTape(label, s[0])};
  return 0;
  LB_CATCH
}
void lasso_random_tape_destroy(lasso_random_tape* t) { delete t; }
int lasso_random_tape_random_scalar(lasso_random_tape* t, const char* label, uint64_t out[4]) {
  return lasso_random_tape_random_vector(t, label, 1, out);
}
int lasso_random_tape_random_vector(lasso_random_tape* t, const char* label, size_t n, uint64_t* out) {
  LB_TRY_T(t)
  if (n && !out) return fail(LASSO_ERR_LENGTH, "random tape: null output");
  const std::vector<fr_t> v = t->t.random_vector(label, n);
  for (size_t i = 0; i < n; i++) memcpy(out + 4 * i, v[i].v, 32);
  return 0;
  LB_CATCH
}

// ---- dense polynomials of the caller
// Commitments, evaluations and openings are collective on a sharded context; the sumchecks, grand products and lookup
// outputs are not available there.
static int poly_ctx_check(lasso_ctx* h) {
  if (h->c->world > 1) return fail(LASSO_ERR_STRATEGY, "not available on a sharded context");
  return 0;
}
// a sharded context holds every row's columns on G ranks: R = poly_R(num_vars) >= G
static int poly_size_check(lasso_ctx* h, size_t num_vars) {
  if (!poly_fits(num_vars, h->c->world))
    return fail(LASSO_ERR_LENGTH, "poly: on a sharded context of G ranks, 2^(num_vars - num_vars/2) >= G");
  return 0;
}
size_t lasso_poly_gens_points_needed(size_t num_vars) { return poly_R(num_vars) + 2; }
int lasso_poly_gens_create(lasso_ctx* h, const uint64_t* stream_affine, size_t n_points, size_t num_vars,
                           lasso_poly_gens** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (!out || !stream_affine) return fail(LASSO_ERR_GENS, "poly gens: null stream or output");
  if (num_vars > 28) return fail(LASSO_ERR_LENGTH, "poly gens: num_vars <= 28");
  if (const int rc = poly_size_check(h, num_vars)) return rc;
  if (n_points < poly_R(num_vars) + 2) return fail(LASSO_ERR_GENS, "poly gens: stream shorter than lasso_poly_gens_points_needed()");
  Gens* g = poly_gens_create(h->c, stream_affine, n_points, num_vars);
  *out = new lasso_poly_gens{g, num_vars};
  return 0;
  LB_CATCH
}
void lasso_poly_gens_destroy(lasso_poly_gens* g) {
  if (!g) return;
  cudaSetDevice(g->g->ctx->device);
  delete g->g;
  delete g;
}
// DensePolynomial::new of a power-of-two length, or (padded) new_padded of any length, from the caller's rows
static int poly_new(lasso_ctx* h, const uint64_t* Z, size_t len, size_t row_stride, bool device, void* stream,
                    bool padded, lasso_poly** out) {
  if (out) *out = nullptr;
  if (!out) return fail(LASSO_ERR_LENGTH, "poly: null output");
  if (padded && len && !Z) return fail(LASSO_ERR_LENGTH, "poly padded: null evaluations");
  if (!padded && !is_pow2(len)) return fail(LASSO_ERR_NOT_POW2, "poly: the length must be a power of two (dense_mlpoly.rs:63-66)");
  if (len > kPolyMaxLen) return fail(LASSO_ERR_LENGTH, "poly: at most 2^28 evaluations after padding");
  if (const int rc = poly_size_check(h, log2_exact_or_ceil(next_pow2(std::max<size_t>(len, 1))))) return rc;
  if (row_stride < 4) return fail(LASSO_ERR_LENGTH, "poly: row_stride must be at least 4 u64");
  if (!device && len && !Z) return fail(LASSO_ERR_POINTER, "poly: null evaluations");
  *out = new lasso_poly{poly_create(h->c, Z, len, row_stride, device, static_cast<cudaStream_t>(stream))};
  return 0;
}
int lasso_poly_create(lasso_ctx* h, const uint64_t* Z, size_t len, lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_new(h, Z, len, 4, false, nullptr, false, out);
  LB_CATCH
}
int lasso_poly_create_device(lasso_ctx* h, const uint64_t* Z, size_t len, size_t row_stride, void* stream,
                             lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_new(h, Z, len, row_stride, true, stream, false, out);
  LB_CATCH
}
size_t lasso_poly_num_vars(const lasso_poly* p) { return p ? p->p->nv : 0; }
void lasso_poly_destroy(lasso_poly* p) {
  if (!p) return;
  cudaSetDevice(p->p->ctx->device);
  delete p->p;
  delete p;
}
// the checks every use of a polynomial shares: same context, and the generators' R equals the polynomial's
static int poly_use_check(lasso_ctx* h, const lasso_poly* p, const lasso_poly_gens* g) {
  if (!p || p->p->ctx != h->c) return fail(LASSO_ERR_STRATEGY, "poly: created on another context");
  if (g) {
    if (g->g->ctx != h->c) return fail(LASSO_ERR_GENS, "poly gens: created on another context");
    // commitments.rs:85 asserts gens.n == the row length
    if (poly_R(g->num_vars) != poly_R(p->p->nv)) return fail(LASSO_ERR_GENS, "poly gens: R differs from the polynomial's");
  }
  return 0;
}
int lasso_poly_commit(lasso_ctx* h, const lasso_poly* p, const lasso_poly_gens* g, uint8_t* out, size_t cap,
                      size_t* out_len) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, g)) return rc;
  if (!g) return fail(LASSO_ERR_GENS, "poly commit: null generators");
  const size_t need = poly_commitment_bytes(p->p->nv);
  if (const int rc = out_room("poly commit", need, out, cap, out_len)) return rc;
  const std::vector<uint8_t> b = timed(h->c->t_commit_ms, [&] { return poly_commit(h->c, *p->p, *g->g); });
  return out_copy("poly commit", b, need, out);
  LB_CATCH
}
int lasso_poly_commit_hiding(lasso_ctx* h, const lasso_poly* p, const lasso_poly_gens* g, lasso_random_tape* tape,
                             uint8_t* out, size_t cap, size_t* out_len, uint64_t* blinds_out, size_t blinds_cap) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, g)) return rc;
  if (!g) return fail(LASSO_ERR_GENS, "poly commit: null generators");
  if (!tape) return fail(LASSO_ERR_LENGTH, "poly commit: null random tape");
  const size_t L = (size_t)1 << (p->p->nv / 2), need = poly_commitment_bytes(p->p->nv);
  if (const int rc = out_room("poly commit", need, out, cap, out_len)) return rc;
  if (!blinds_out || blinds_cap < L) return fail(LASSO_ERR_LENGTH, "poly commit: room for fewer blinds than rows");
  std::vector<fr_t> blinds;
  const std::vector<uint8_t> b = timed(h->c->t_commit_ms, [&] {
    blinds = tape->t.random_vector("poly_blinds", L);  // dense_mlpoly.rs:165-170
    return poly_commit_hiding(h->c, *p->p, *g->g, blinds);
  });
  if (const int rc = out_copy("poly commit", b, need, out)) return rc;
  for (size_t i = 0; i < L; i++) memcpy(blinds_out + 4 * i, blinds[i].v, 32);
  return 0;
  LB_CATCH
}
static int load_point(const Poly& p, const uint64_t* r, size_t r_len, std::vector<fr_t>& rv) {
  if (r_len != p.nv) return fail(LASSO_ERR_LENGTH, "poly: r.len() != num_vars");
  if (r_len && !r) return fail(LASSO_ERR_LENGTH, "poly: null point");
  if (!load_scalars(r, r_len, rv)) return fail(LASSO_ERR_VALUE, "poly: a coordinate of r is not a canonical residue");
  return 0;
}
int lasso_poly_evaluate(lasso_ctx* h, const lasso_poly* p, const uint64_t* r, size_t r_len, uint64_t out[4]) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, nullptr)) return rc;
  std::vector<fr_t> rv;
  if (const int rc = load_point(*p->p, r, r_len, rv)) return rc;
  const fr_t v = poly_evaluate(h->c, *p->p, rv);
  memcpy(out, v.v, 32);
  return 0;
  LB_CATCH
}
int lasso_poly_eval_prove(lasso_ctx* h, const lasso_poly* p, const lasso_poly_gens* g, const uint64_t* r, size_t r_len,
                          const uint64_t Zr[4], lasso_transcript* transcript, lasso_random_tape* tape,
                          uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint8_t C_Zr_out[32]) {
  return lasso_poly_eval_prove_hiding(h, p, g, nullptr, 0, r, r_len, Zr, nullptr, transcript, tape, proof_out, proof_cap,
                                      proof_len, C_Zr_out);
}
int lasso_poly_eval_prove_hiding(lasso_ctx* h, const lasso_poly* p, const lasso_poly_gens* g, const uint64_t* blinds,
                                 size_t n_blinds, const uint64_t* r, size_t r_len, const uint64_t Zr[4],
                                 const uint64_t blind_Zr[4], lasso_transcript* transcript, lasso_random_tape* tape,
                                 uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint8_t C_Zr_out[32]) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, g)) return rc;
  if (!g) return fail(LASSO_ERR_GENS, "poly eval proof: null generators");
  if (!transcript || !tape) return fail(LASSO_ERR_LENGTH, "poly eval proof: null transcript or random tape");
  if (n_blinds != 0 && (n_blinds != ((size_t)1 << (p->p->nv / 2)) || !blinds))
    return fail(LASSO_ERR_LENGTH, "poly eval proof: n_blinds must be 0 (no blinds) or the commitment's row count");
  std::vector<fr_t> rv, zr, bl, bzr(1, fr_zero());
  if (const int rc = load_point(*p->p, r, r_len, rv)) return rc;
  if (!load_scalars(Zr, 1, zr)) return fail(LASSO_ERR_VALUE, "poly eval proof: Zr is not a canonical residue");
  if (!load_scalars(blinds, n_blinds, bl)) return fail(LASSO_ERR_VALUE, "poly eval proof: a blind is not a canonical residue");
  if (blind_Zr && !load_scalars(blind_Zr, 1, bzr))
    return fail(LASSO_ERR_VALUE, "poly eval proof: blind_Zr is not a canonical residue");
  const size_t need = dpl_bytes(p->p->nv);
  if (const int rc = out_room("poly eval proof", need, proof_out, proof_cap, proof_len)) return rc;
  uint8_t czr[32];
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return poly_eval_prove(h->c, *p->p, *g->g, rv, zr[0], transcript->t, tape->t, czr, bl, bzr[0]);
  });
  if (const int rc = out_copy("poly eval proof", b, need, proof_out)) return rc;
  if (C_Zr_out) memcpy(C_Zr_out, czr, 32);
  return 0;
  LB_CATCH
}
int lasso_poly_create_eq(lasso_ctx* h, const uint64_t* r, size_t r_len, lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (!out) return fail(LASSO_ERR_LENGTH, "eq poly: null output");
  if (r_len > 28) return fail(LASSO_ERR_LENGTH, "eq poly: at most 28 variables (2^28 evaluations)");
  if (const int rc = poly_size_check(h, r_len)) return rc;
  if (r_len && !r) return fail(LASSO_ERR_LENGTH, "eq poly: null point");
  std::vector<fr_t> rv;
  if (!load_scalars(r, r_len, rv)) return fail(LASSO_ERR_VALUE, "eq poly: a coordinate of r is not a canonical residue");
  *out = new lasso_poly{poly_create_eq(h->c, rv)};
  return 0;
  LB_CATCH
}

// ---- transforms of a caller's polynomial: binds, split, padding, read-back
static int poly_bind(lasso_ctx* h, const lasso_poly* p, const uint64_t* r, size_t k, lasso_poly** out, bool top) {
  if (out) *out = nullptr;
  if (const int rc = poly_use_check(h, p, nullptr)) return rc;
  if (!out || !r) return fail(LASSO_ERR_LENGTH, "poly bind: null point or output");
  if (k < 1 || k > p->p->nv) return fail(LASSO_ERR_LENGTH, "poly bind: k must be in 1..num_vars");
  if (const int rc = poly_size_check(h, p->p->nv - k)) return rc;
  std::vector<fr_t> rv;
  if (!load_scalars(r, k, rv)) return fail(LASSO_ERR_VALUE, "poly bind: a coordinate of r is not a canonical residue");
  *out = new lasso_poly{top ? poly_bind_top(h->c, *p->p, rv) : poly_bind_bot(h->c, *p->p, rv)};
  return 0;
}
int lasso_poly_bind_top(lasso_ctx* h, const lasso_poly* p, const uint64_t* r, size_t k, lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_bind(h, p, r, k, out, true);
  LB_CATCH
}
int lasso_poly_bind_bot(lasso_ctx* h, const lasso_poly* p, const uint64_t* r, size_t k, lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_bind(h, p, r, k, out, false);
  LB_CATCH
}
int lasso_poly_split(lasso_ctx* h, const lasso_poly* p, size_t idx, lasso_poly** lo_out, lasso_poly** hi_out) {
  LB_TRY_CTX(h)
  if (lo_out) *lo_out = nullptr;
  if (hi_out) *hi_out = nullptr;
  if (const int rc = poly_use_check(h, p, nullptr)) return rc;
  if (!lo_out || !hi_out) return fail(LASSO_ERR_LENGTH, "poly split: null output");
  if (!is_pow2(idx) || idx > p->p->len / 2) return fail(LASSO_ERR_LENGTH, "poly split: idx must be a power of two, 2 idx <= len");
  if (const int rc = poly_size_check(h, log2_exact_or_ceil(idx))) return rc;
  Poly *lo = nullptr, *hi = nullptr;
  poly_split(h->c, *p->p, idx, &lo, &hi);
  *lo_out = new lasso_poly{lo};
  *hi_out = new lasso_poly{hi};
  return 0;
  LB_CATCH
}
int lasso_poly_create_padded(lasso_ctx* h, const uint64_t* Z, size_t len, lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_new(h, Z, len, 4, false, nullptr, true, out);
  LB_CATCH
}
int lasso_poly_create_padded_device(lasso_ctx* h, const uint64_t* Z, size_t len, size_t row_stride, void* stream,
                                    lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_new(h, Z, len, row_stride, true, stream, true, out);
  LB_CATCH
}
int lasso_poly_read(lasso_ctx* h, const lasso_poly* p, uint64_t* out, size_t cap) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, nullptr)) return rc;
  if (!out || cap < p->p->len) return fail(LASSO_ERR_LENGTH, "poly read: room for fewer evaluations than the polynomial has");
  poly_read(h->c, *p->p, out);
  return 0;
  LB_CATCH
}
int lasso_poly_read_device(lasso_ctx* h, const lasso_poly* p, uint64_t* dst, size_t row_stride, void* stream) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, nullptr)) return rc;
  if (!dst) return fail(LASSO_ERR_LENGTH, "poly read: null destination");
  if (row_stride < 4) return fail(LASSO_ERR_LENGTH, "poly read: row_stride must be at least 4 u64");
  poly_read_device(h->c, *p->p, dst, row_stride, static_cast<cudaStream_t>(stream));
  return 0;
  LB_CATCH
}

// ---- many polynomials per call: merge, batched evaluation, one combined opening
// The n polynomials of one call: each of this context (LASSO_ERR_STRATEGY), then, with same_nv, all of one num_vars
// (LASSO_ERR_LENGTH).  ps receives them.
static int poly_array(lasso_ctx* h, const char* what, const lasso_poly* const* polys, size_t n, bool same_nv,
                      std::vector<const Poly*>& ps) {
  for (size_t j = 0; j < n; j++)
    if (const int rc = poly_use_check(h, polys[j], nullptr)) return rc;
  for (size_t j = 1; same_nv && j < n; j++)
    if (polys[j]->p->nv != polys[0]->p->nv)
      return fail(LASSO_ERR_LENGTH, std::string(what) + ": the polynomials have different num_vars");
  ps.resize(n);
  for (size_t j = 0; j < n; j++) ps[j] = polys[j]->p;
  return 0;
}
int lasso_poly_create_merge(lasso_ctx* h, const lasso_poly* const* polys, size_t n_polys, lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (!polys || n_polys == 0 || !out) return fail(LASSO_ERR_LENGTH, "merge: no polynomials, or a null output");
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "merge", polys, n_polys, false, ps)) return rc;
  size_t total = 0;
  for (const Poly* p : ps) {
    total += p->len;  // each len <= 2^28: the running sum cannot wrap before it passes the limit
    if (total > kPolyMaxLen) return fail(LASSO_ERR_LENGTH, "merge: at most 2^28 evaluations after padding");
  }
  *out = new lasso_poly{poly_merge(h->c, ps.data(), (int)n_polys)};
  return 0;
  LB_CATCH
}
int lasso_poly_evaluate_batch(lasso_ctx* h, const lasso_poly* const* polys, size_t n_polys, const uint64_t* r,
                              size_t r_len, uint64_t* out) {
  LB_TRY_CTX(h)
  if (!polys || n_polys == 0 || n_polys > (size_t)kDotMaxPolys || !out)
    return fail(LASSO_ERR_LENGTH, "evaluate batch: 1..64 polynomials and an output");
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "evaluate batch", polys, n_polys, true, ps)) return rc;
  std::vector<fr_t> rv;
  if (const int rc = load_point(*ps[0], r, r_len, rv)) return rc;
  const std::vector<fr_t> v = poly_evaluate_batch(h->c, ps.data(), (int)n_polys, rv);
  for (size_t j = 0; j < n_polys; j++) memcpy(out + 4 * j, v[j].v, 32);
  return 0;
  LB_CATCH
}
int lasso_combined_eval_prove(lasso_ctx* h, const lasso_poly* combined, const lasso_poly_gens* g, const uint64_t* evals,
                              size_t n_evals, const uint64_t* r, size_t r_len, lasso_transcript* transcript,
                              lasso_random_tape* tape, uint8_t* proof_out, size_t proof_cap, size_t* proof_len) {
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, combined, g)) return rc;
  if (!g) return fail(LASSO_ERR_GENS, "combined eval proof: null generators");
  if (n_evals == 0 || n_evals > kPolyMaxLen || !evals) return fail(LASSO_ERR_LENGTH, "combined eval proof: 1..2^28 evals");
  if (r_len && !r) return fail(LASSO_ERR_LENGTH, "combined eval proof: null point");
  // subtables/mod.rs:238-241: the joint polynomial has log2(#evals padded) variables more than r
  const size_t nv = combined->p->nv;
  if (nv != r_len + log2_exact_or_ceil(next_pow2(n_evals)))
    return fail(LASSO_ERR_LENGTH, "combined eval proof: num_vars != r.len() + log2(next_pow2(n_evals))");
  const size_t need = dpl_bytes(nv);  // the PolyEvalProof of lasso_poly_eval_prove at num_vars
  if (const int rc = out_room("combined eval proof", need, proof_out, proof_cap, proof_len)) return rc;
  if (!transcript || !tape) return fail(LASSO_ERR_LENGTH, "combined eval proof: null transcript or random tape");
  std::vector<fr_t> ev, rv;
  if (!load_scalars(evals, n_evals, ev)) return fail(LASSO_ERR_VALUE, "combined eval proof: an eval is not a canonical residue");
  if (!load_scalars(r, r_len, rv)) return fail(LASSO_ERR_VALUE, "combined eval proof: a coordinate of r is not a canonical residue");
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return combined_eval_prove(h->c, *combined->p, *g->g, ev, rv, transcript->t, tape->t);
  });
  return out_copy("combined eval proof", b, need, proof_out);
  LB_CATCH
}

// ---- sumchecks over a caller's polynomials
int lasso_comb_create(int n_inputs, const int32_t* program, int n_ops, const uint64_t* constants, int n_constants,
                      int degree, lasso_comb** out) {
  LB_TRY
  if (out) *out = nullptr;
  if (!out) return fail(LASSO_ERR_STRATEGY, "comb: null output");
  if (n_inputs < 1 || n_inputs > kCombMaxInputs) return fail(LASSO_ERR_STRATEGY, "comb: n_inputs must be in 1..16");
  if (!program) return fail(LASSO_ERR_STRATEGY, "comb: null program");
  Comb g;
  const std::string why = program_check(n_inputs, program, n_ops, constants, n_constants, degree, "degree", g.ins, &g.n_slots);
  if (!why.empty()) return fail(LASSO_ERR_STRATEGY, "comb: " + why);
  g.n_inputs = n_inputs;
  g.degree = degree;
  g.consts.resize(n_constants);
  if (n_constants) memcpy(g.consts.data(), constants, (size_t)n_constants * 32);
  *out = new lasso_comb{std::move(g)};
  return 0;
  LB_CATCH
}
void lasso_comb_destroy(lasso_comb* g) { delete g; }
int lasso_sumcheck_prove(lasso_ctx* h, const lasso_comb* g, const lasso_poly* const* polys, size_t n_polys,
                         size_t num_rounds, lasso_transcript* transcript, uint8_t* proof_out, size_t proof_cap,
                         size_t* proof_len, uint64_t* r_out, uint64_t* final_evals_out, uint64_t claim_out[4]) {
  LB_TRY_CTX(h)
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!g) return fail(LASSO_ERR_STRATEGY, "sumcheck: null combining function");
  if (!polys || n_polys != (size_t)g->g.n_inputs)
    return fail(LASSO_ERR_STRATEGY, "sumcheck: " + std::to_string(n_polys) + " polynomials for a combining function of " +
                                        std::to_string(g->g.n_inputs) + " inputs");
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "sumcheck", polys, n_polys, true, ps)) return rc;
  if (num_rounds < 1 || num_rounds > ps[0]->nv) return fail(LASSO_ERR_LENGTH, "sumcheck: num_rounds must be in 1..num_vars");
  const size_t need = sumcheck_bytes(num_rounds, (size_t)g->g.degree);
  if (const int rc = out_room("sumcheck", need, proof_out, proof_cap, proof_len)) return rc;
  if (!transcript || !r_out || !final_evals_out) return fail(LASSO_ERR_LENGTH, "sumcheck: null transcript or output");
  const SumcheckOut o = timed(h->c->t_prove_ms, [&] {
    return sumcheck_prove(h->c, g->g, ps.data(), (int)n_polys, num_rounds, transcript->t);
  });
  if (const int rc = out_copy("sumcheck", o.proof, need, proof_out)) return rc;
  for (size_t j = 0; j < num_rounds; j++) memcpy(r_out + 4 * j, o.r[j].v, 32);
  for (size_t j = 0; j < n_polys; j++) memcpy(final_evals_out + 4 * j, o.final_evals[j].v, 32);
  if (claim_out) memcpy(claim_out, o.claim.v, 32);
  return 0;
  LB_CATCH
}
int lasso_sumcheck_prove_cubic_batched(lasso_ctx* h, const lasso_poly* const* A, const lasso_poly* const* B, size_t n,
                                       const lasso_poly* C, const uint64_t* coeffs, const uint64_t claim[4],
                                       size_t num_rounds, lasso_transcript* transcript, uint8_t* proof_out,
                                       size_t proof_cap, size_t* proof_len, uint64_t* r_out, uint64_t* claims_A_out,
                                       uint64_t* claims_B_out, uint64_t claim_C_out[4]) {
  LB_TRY_CTX(h)
  if (n < 1 || n > 32) return fail(LASSO_ERR_STRATEGY, "cubic sumcheck: 1 <= n <= 32 pairs");
  if (!A || !B) return fail(LASSO_ERR_STRATEGY, "cubic sumcheck: null polynomial array");
  // A_0.., B_0.., C: one array for the checks
  std::vector<const lasso_poly*> all(A, A + n);
  all.insert(all.end(), B, B + n);
  all.push_back(C);
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "cubic sumcheck", all.data(), all.size(), true, ps)) return rc;
  if (num_rounds < 1 || num_rounds > ps[0]->nv) return fail(LASSO_ERR_LENGTH, "cubic sumcheck: num_rounds must be in 1..num_vars");
  const size_t need = sumcheck_bytes(num_rounds, 3);
  if (const int rc = out_room("cubic sumcheck", need, proof_out, proof_cap, proof_len)) return rc;
  if (!transcript || !coeffs || !claim || !r_out || !claims_A_out || !claims_B_out || !claim_C_out)
    return fail(LASSO_ERR_LENGTH, "cubic sumcheck: null transcript, input or output");
  std::vector<fr_t> cv, e;
  if (!load_scalars(coeffs, n, cv)) return fail(LASSO_ERR_VALUE, "cubic sumcheck: a coefficient is not a canonical residue");
  if (!load_scalars(claim, 1, e)) return fail(LASSO_ERR_VALUE, "cubic sumcheck: the claim is not a canonical residue");
  const CubicOut o = timed(h->c->t_prove_ms, [&] {
    return cubic_prove(h->c, ps.data(), ps.data() + n, (int)n, *ps[2 * n], cv, e[0], num_rounds, transcript->t);
  });
  if (const int rc = out_copy("cubic sumcheck", o.proof, need, proof_out)) return rc;
  for (size_t j = 0; j < num_rounds; j++) memcpy(r_out + 4 * j, o.r[j].v, 32);
  for (size_t k = 0; k < n; k++) {
    memcpy(claims_A_out + 4 * k, o.finals[k].v, 32);
    memcpy(claims_B_out + 4 * k, o.finals[n + k].v, 32);
  }
  memcpy(claim_C_out, o.finals[2 * n].v, 32);
  return 0;
  LB_CATCH
}
int lasso_poly_create_comb(lasso_ctx* h, const lasso_comb* g, const lasso_poly* const* polys, size_t n_polys,
                           lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (!g) return fail(LASSO_ERR_STRATEGY, "comb poly: null combining function");
  if (!polys || n_polys != (size_t)g->g.n_inputs)
    return fail(LASSO_ERR_STRATEGY, "comb poly: " + std::to_string(n_polys) + " polynomials for a combining function of " +
                                        std::to_string(g->g.n_inputs) + " inputs");
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "comb poly", polys, n_polys, true, ps)) return rc;
  if (const int rc = poly_size_check(h, ps[0]->nv)) return rc;
  if (!out) return fail(LASSO_ERR_LENGTH, "comb poly: null output");
  *out = new lasso_poly{poly_create_comb(h->c, g->g, ps.data(), (int)n_polys)};
  return 0;
  LB_CATCH
}

// ---- zero-knowledge sumchecks: MultiCommitGens, commitments, DotProductProof, ZKSumcheckInstanceProof
// Every call but lasso_zk_sumcheck_prove runs on a sharded context too: each rank computes alone, with no exchange.
int lasso_mc_gens_create(lasso_ctx* h, const uint64_t* G_affine, size_t n, const uint64_t h_affine[8],
                         lasso_mc_gens** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (!out || !G_affine || !h_affine) return fail(LASSO_ERR_GENS, "mc gens: null points or output");
  if (n < 1 || n > kMcMaxN) return fail(LASSO_ERR_LENGTH, "mc gens: n must be in 1..1024");
  *out = new lasso_mc_gens{mc_gens_create(h->c, G_affine, n, h_affine)};
  return 0;
  LB_CATCH
}
size_t lasso_mc_gens_n(const lasso_mc_gens* g) { return g ? g->g->n : 0; }
void lasso_mc_gens_destroy(lasso_mc_gens* g) {
  if (!g) return;
  cudaSetDevice(g->g->ctx->device);
  delete g->g;
  delete g;
}
// gens of this context with n points (n == 0: any n)
static int mc_gens_check(lasso_ctx* h, const char* what, const lasso_mc_gens* g, size_t n) {
  if (!g || g->g->ctx != h->c) return fail(LASSO_ERR_GENS, std::string(what) + ": null generators, or of another context");
  if (n && g->g->n != n)
    return fail(LASSO_ERR_GENS, std::string(what) + ": generators of n = " + std::to_string(g->g->n) + ", expected " +
                                    std::to_string(n));
  return 0;
}
int lasso_mc_commit(lasso_ctx* h, const lasso_mc_gens* g, const uint64_t* scalars, size_t n, const uint64_t blind[4],
                    uint8_t out[32]) {
  LB_TRY_CTX(h)
  if (const int rc = mc_gens_check(h, "mc commit", g, 0)) return rc;
  if (n != g->g->n) return fail(LASSO_ERR_GENS, "mc commit: n != gens.n (commitments.rs:85)");
  if (!scalars || !blind || !out) return fail(LASSO_ERR_LENGTH, "mc commit: null scalars, blind or output");
  std::vector<fr_t> s, b;
  if (!load_scalars(scalars, n, s) || !load_scalars(blind, 1, b))
    return fail(LASSO_ERR_VALUE, "mc commit: a scalar or the blind is not a canonical residue");
  timed(h->c->t_commit_ms, [&] {
    mc_commit(h->c, *g->g, s, b[0], out);
    return 0;
  });
  return 0;
  LB_CATCH
}
int lasso_dot_product_prove(lasso_ctx* h, const lasso_mc_gens* gens_1, const lasso_mc_gens* gens_n,
                            lasso_transcript* transcript, lasso_random_tape* tape, const uint64_t* x,
                            const uint64_t blind_x[4], const uint64_t* a, size_t n, const uint64_t y[4],
                            const uint64_t blind_y[4], uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                            uint8_t Cx_out[32], uint8_t Cy_out[32]) {
  LB_TRY_CTX(h)
  if (const int rc = mc_gens_check(h, "dot product proof", gens_1, 1)) return rc;
  if (const int rc = mc_gens_check(h, "dot product proof", gens_n, 0)) return rc;
  if (gens_n->g->n != n) return fail(LASSO_ERR_GENS, "dot product proof: gens_n.n != a.len() (dot_product.rs:50)");
  const size_t need = dot_product_bytes(n);
  if (const int rc = out_room("dot product proof", need, proof_out, proof_cap, proof_len)) return rc;
  if (!transcript || !tape || !x || !blind_x || !a || !y || !blind_y || !Cx_out || !Cy_out)
    return fail(LASSO_ERR_LENGTH, "dot product proof: null transcript, random tape, input or output");
  std::vector<fr_t> xv, av, bx, yv, by;
  if (!load_scalars(x, n, xv) || !load_scalars(a, n, av) || !load_scalars(blind_x, 1, bx) || !load_scalars(y, 1, yv) ||
      !load_scalars(blind_y, 1, by))
    return fail(LASSO_ERR_VALUE, "dot product proof: x, a, y or a blind is not a canonical residue");
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return dot_product_prove(h->c, *gens_1->g, *gens_n->g, transcript->t, tape->t, xv, bx[0], av, yv[0], by[0], Cx_out,
                             Cy_out);
  });
  return out_copy("dot product proof", b, need, proof_out);
  LB_CATCH
}
int lasso_zk_sumcheck_prove(lasso_ctx* h, const lasso_comb* g, const lasso_poly* const* polys, size_t n_polys,
                            size_t num_rounds, const uint64_t blind_claim[4], const lasso_mc_gens* gens_1,
                            const lasso_mc_gens* gens_n, lasso_transcript* transcript, lasso_random_tape* tape,
                            uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t* r_out,
                            uint64_t* final_evals_out, uint64_t claim_out[4], uint8_t comm_claim_out[32],
                            uint64_t blind_eval_out[4]) {
  LB_TRY_CTX(h)
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!g) return fail(LASSO_ERR_STRATEGY, "zk sumcheck: null combining function");
  if (!polys || n_polys != (size_t)g->g.n_inputs)
    return fail(LASSO_ERR_STRATEGY, "zk sumcheck: " + std::to_string(n_polys) + " polynomials for a combining function of " +
                                        std::to_string(g->g.n_inputs) + " inputs");
  std::vector<const Poly*> ps;
  if (const int rc = poly_array(h, "zk sumcheck", polys, n_polys, true, ps)) return rc;
  if (num_rounds < 1 || num_rounds > ps[0]->nv) return fail(LASSO_ERR_LENGTH, "zk sumcheck: num_rounds must be in 1..num_vars");
  if (const int rc = mc_gens_check(h, "zk sumcheck", gens_1, 1)) return rc;
  // sumcheck.rs:358: gens_n.n == degree_bound + 1
  if (const int rc = mc_gens_check(h, "zk sumcheck", gens_n, (size_t)g->g.degree + 1)) return rc;
  const size_t need = zk_sumcheck_bytes(num_rounds, (size_t)g->g.degree);
  if (const int rc = out_room("zk sumcheck", need, proof_out, proof_cap, proof_len)) return rc;
  if (!transcript || !tape || !blind_claim || !r_out || !final_evals_out)
    return fail(LASSO_ERR_LENGTH, "zk sumcheck: null transcript, random tape, blind_claim or output");
  std::vector<fr_t> bc;
  if (!load_scalars(blind_claim, 1, bc)) return fail(LASSO_ERR_VALUE, "zk sumcheck: blind_claim is not a canonical residue");
  const ZkSumcheckOut o = timed(h->c->t_prove_ms, [&] {
    return zk_sumcheck_prove(h->c, g->g, ps.data(), (int)n_polys, num_rounds, bc[0], *gens_1->g, *gens_n->g,
                             transcript->t, tape->t);
  });
  if (const int rc = out_copy("zk sumcheck", o.proof, need, proof_out)) return rc;
  for (size_t j = 0; j < num_rounds; j++) memcpy(r_out + 4 * j, o.r[j].v, 32);
  for (size_t j = 0; j < n_polys; j++) memcpy(final_evals_out + 4 * j, o.final_evals[j].v, 32);
  if (claim_out) memcpy(claim_out, o.claim.v, 32);
  if (comm_claim_out) memcpy(comm_claim_out, o.comm_claim, 32);
  if (blind_eval_out) memcpy(blind_eval_out, o.blind_eval.v, 32);
  return 0;
  LB_CATCH
}

// ---- Σ-protocols of committed scalars: KnowledgeProof, EqualityProof, ProductProof (subprotocols/zk.rs).  On a sharded
// context every rank computes alone, with no exchange.
// The shared checks, in the order of the other proofs: gens of this context with n == 1 (commitments.rs:79), then a null
// transcript, tape, scalar or output, then every scalar a canonical residue (into v, in order).
static int sigma_check(lasso_ctx* h, const char* what, const lasso_mc_gens* g, const void* transcript, const void* tape,
                       std::initializer_list<const uint64_t*> in, std::initializer_list<const void*> outs,
                       std::vector<fr_t>& v) {
  if (const int rc = mc_gens_check(h, what, g, 1)) return rc;
  bool null = !transcript || !tape;
  for (const uint64_t* p : in) null |= !p;
  for (const void* p : outs) null |= !p;
  if (null) return fail(LASSO_ERR_LENGTH, std::string(what) + ": null transcript, random tape, scalar or output");
  for (const uint64_t* p : in) {
    std::vector<fr_t> s;
    if (!load_scalars(p, 1, s)) return fail(LASSO_ERR_VALUE, std::string(what) + ": a value or blind is not a canonical residue");
    v.push_back(s[0]);
  }
  return 0;
}
int lasso_knowledge_prove(lasso_ctx* h, const lasso_mc_gens* gens, lasso_transcript* transcript, lasso_random_tape* tape,
                          const uint64_t x[4], const uint64_t r[4], uint8_t proof_out[96], uint8_t C_out[32]) {
  LB_TRY_CTX(h)
  std::vector<fr_t> v;
  if (const int rc = sigma_check(h, "knowledge proof", gens, transcript, tape, {x, r}, {proof_out, C_out}, v)) return rc;
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return knowledge_prove(h->c, *gens->g, transcript->t, tape->t, v[0], v[1], C_out);
  });
  return out_copy("knowledge proof", b, kKnowledgeProofBytes, proof_out);
  LB_CATCH
}
int lasso_equality_prove(lasso_ctx* h, const lasso_mc_gens* gens, lasso_transcript* transcript, lasso_random_tape* tape,
                         const uint64_t v1[4], const uint64_t s1[4], const uint64_t v2[4], const uint64_t s2[4],
                         uint8_t proof_out[64], uint8_t C1_out[32], uint8_t C2_out[32]) {
  LB_TRY_CTX(h)
  std::vector<fr_t> v;
  if (const int rc =
          sigma_check(h, "equality proof", gens, transcript, tape, {v1, s1, v2, s2}, {proof_out, C1_out, C2_out}, v))
    return rc;
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return equality_prove(h->c, *gens->g, transcript->t, tape->t, v[0], v[1], v[2], v[3], C1_out, C2_out);
  });
  return out_copy("equality proof", b, kEqualityProofBytes, proof_out);
  LB_CATCH
}
int lasso_product_prove(lasso_ctx* h, const lasso_mc_gens* gens, lasso_transcript* transcript, lasso_random_tape* tape,
                        const uint64_t x[4], const uint64_t rX[4], const uint64_t y[4], const uint64_t rY[4],
                        const uint64_t z[4], const uint64_t rZ[4], uint8_t proof_out[256], uint8_t X_out[32],
                        uint8_t Y_out[32], uint8_t Z_out[32]) {
  LB_TRY_CTX(h)
  std::vector<fr_t> v;
  if (const int rc = sigma_check(h, "product proof", gens, transcript, tape, {x, rX, y, rY, z, rZ},
                                 {proof_out, X_out, Y_out, Z_out}, v))
    return rc;
  const std::vector<uint8_t> b = timed(h->c->t_prove_ms, [&] {
    return product_prove(h->c, *gens->g, transcript->t, tape->t, v[0], v[1], v[2], v[3], v[4], v[5], X_out, Y_out, Z_out);
  });
  return out_copy("product proof", b, kProductProofBytes, proof_out);
  LB_CATCH
}

// ---- grand products over a caller's polynomials
int lasso_gp_circuit_create(lasso_ctx* h, const lasso_poly* p, lasso_gp_circuit** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (const int rc = poly_use_check(h, p, nullptr)) return rc;
  if (!out) return fail(LASSO_ERR_LENGTH, "grand product circuit: null output");
  if (p->p->nv < 1 || p->p->nv > 28)
    return fail(LASSO_ERR_LENGTH, "grand product circuit: num_vars must be in 1..28 (a single evaluation has no layers)");
  fr_t product;
  Circuit* ci = gp_circuit_create(h->c, *p->p, &product);
  *out = new lasso_gp_circuit{h->c, std::unique_ptr<Circuit>(ci), product, false};
  return 0;
  LB_CATCH
}
int lasso_gp_circuit_evaluate(const lasso_gp_circuit* gc, uint64_t out[4]) {
  if (!gc || !out) return fail(LASSO_ERR_LENGTH, "grand product circuit: null circuit or output");
  memcpy(out, gc->product.v, 32);
  return 0;
}
size_t lasso_gp_circuit_num_vars(const lasso_gp_circuit* gc) { return gc ? gc->ci->num_layers : 0; }
void lasso_gp_circuit_destroy(lasso_gp_circuit* gc) {
  if (!gc) return;
  cudaSetDevice(gc->c->device);
  delete gc;
}
int lasso_gp_prove(lasso_ctx* h, const lasso_gp_circuit* const* circuits, size_t n, lasso_transcript* transcript,
                   uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t* r_out, uint64_t* claims_out) {
  LB_TRY_CTX(h)
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!circuits || n == 0 || n > 32)
    return fail(LASSO_ERR_STRATEGY, "grand product: 1..32 circuits per batch (CubicCoeffs, TreePtrs)");
  for (size_t k = 0; k < n; k++) {
    if (!circuits[k] || circuits[k]->c != h->c) return fail(LASSO_ERR_STRATEGY, "grand product: a circuit of another context");
    if (circuits[k]->proven) return fail(LASSO_ERR_STRATEGY, "grand product: a circuit can be proven once (its layers are bound)");
    for (size_t j = 0; j < k; j++)
      if (circuits[j] == circuits[k]) return fail(LASSO_ERR_STRATEGY, "grand product: the same circuit twice in one batch");
  }
  const size_t v = circuits[0]->ci->num_layers;
  for (size_t k = 1; k < n; k++)
    if (circuits[k]->ci->num_layers != v) return fail(LASSO_ERR_LENGTH, "grand product: the circuits have different num_vars");
  const size_t need = gpa_bytes(n, v);
  if (const int rc = out_room("grand product", need, proof_out, proof_cap, proof_len)) return rc;
  if (!transcript || !r_out || !claims_out) return fail(LASSO_ERR_LENGTH, "grand product: null transcript or output");
  std::vector<Circuit*> cs(n);
  std::vector<fr_t> products(n);
  for (size_t k = 0; k < n; k++) {
    cs[k] = circuits[k]->ci.get();
    products[k] = circuits[k]->product;
    circuits[k]->proven = true;
  }
  const GrandProductOut o = timed(h->c->t_prove_ms, [&] { return gp_prove(h->c, cs, products, transcript->t); });
  if (const int rc = out_copy("grand product", o.proof, need, proof_out)) return rc;
  for (size_t j = 0; j < v; j++) memcpy(r_out + 4 * j, o.r[j].v, 32);
  for (size_t k = 0; k < n; k++) memcpy(claims_out + 4 * k, o.claims[k].v, 32);
  return 0;
  LB_CATCH
}

unsigned long long lasso_launch_count(const lasso_ctx*) { return g_launches.load(); }
void lasso_last_timings(const lasso_ctx* h, double out_ms[3]) {
  out_ms[0] = h->c->t_densify_ms;
  out_ms[1] = h->c->t_commit_ms;
  out_ms[2] = h->c->t_prove_ms;
}
size_t lasso_spans(const lasso_ctx* h, char* buf, size_t cap) {
  std::string s;
  for (auto& kv : h->c->spans) s += kv.first + "=" + std::to_string(kv.second) + ";";
  if (buf && cap) {
    size_t n = std::min(cap - 1, s.size());
    memcpy(buf, s.data(), n);
    buf[n] = 0;
  }
  h->c->spans.clear();
  return s.size();
}

int lasso_bench_bind(lasso_ctx* h, size_t len, int npolys, int iters, double* avg_ms) {
  LB_TRY_CTX(h)
  if (!is_pow2(len) || len < 2 || npolys < 1) return fail(LASSO_ERR_NOT_POW2, "bench_bind: bad shape");
  Ctx* c = h->c;
  DBuf<fr_t> d(c, len * npolys);
  // fill with pseudo-random canonical residues: eq table of a fixed point, replicated
  FrVec rv;
  int ell = 0;
  while (((size_t)1 << ell) < len) ell++;
  for (int i = 0; i < ell; i++) rv.v[i] = fr_from_u64(0x9e3779b97f4a7c15ull * (i + 1));
  for (int k = 0; k < npolys; k++) launch_eq_evals(rv, ell, d.p + (size_t)k * len, c->d_eq_scratch, c->st);
  fr_t r = fr_from_u64(0xdeadbeefcafef00dull);
  cudaEvent_t e0, e1;
  LB_CUDA_CHECK(cudaEventCreate(&e0));
  LB_CUDA_CHECK(cudaEventCreate(&e1));
  for (int w = 0; w < 3; w++) launch_bind_top(d.p, len, npolys, len / 2, r, c->st);
  c->sync();
  LB_CUDA_CHECK(cudaEventRecord(e0, c->st));
  for (int i = 0; i < iters; i++) launch_bind_top(d.p, len, npolys, len / 2, r, c->st);
  LB_CUDA_CHECK(cudaEventRecord(e1, c->st));
  LB_CUDA_CHECK(cudaEventSynchronize(e1));
  float ms = 0;
  LB_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  *avg_ms = ms / iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
  LB_CATCH
}

}  // extern "C"
