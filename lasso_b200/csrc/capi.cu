// lasso_b200 — extern "C" boundary (include/lasso_b200.h).  Plain pointers and sizes only; every entry
// point states the reference item it replaces in the header.
#include "../../include/lasso_b200.h"

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
  catch (const std::exception& e) {               \
    return fail(-1, e.what());                    \
  }

static bool is_pow2(size_t x) { return x && !(x & (x - 1)); }
static constexpr size_t kMsmLargeMin = 1 << 14;  // below this the row kernels (c = 8, buckets in shared memory) win
static Strategy mkS(int kind, int C, int log_M, int log_R) { return Strategy{kind, C, log_M, log_R}; }

// Checks a custom strategy's descriptor (everything but the tables' contents) and fills cs with its shape, the degree
// of g and the instructions with SSA slots mapped to physical slots.  "" = valid, else the reason.
static std::string custom_check(int C, int log_m, int nsub, int alpha, const int* sub, const int* dim, const int32_t* prog,
                                int n_ops, const uint64_t* consts, int n_consts, int degree, CustomStrategy& cs,
                                std::vector<CustomIns>& ins) {
  if (C < 1 || C > 16) return "C must be in 1..16";
  if (log_m < 2 || log_m > 24) return "log_m must be in 2..24";
  if (alpha < 1 || alpha > kCustomMaxMemories) return "num_memories must be in 1..16";
  if (nsub < 1 || nsub > alpha) return "num_subtables must be in 1..num_memories";
  if (!sub || !dim || !prog) return "null map or program";
  for (int i = 0; i < alpha; i++) {
    if (sub[i] < 0 || sub[i] >= nsub) return "memory_to_subtable_index out of range";
    if (dim[i] < 0 || dim[i] >= C) return "memory_to_dimension_index out of range";
  }
  int n_slots = 0;
  const std::string why = program_check(alpha, prog, n_ops, consts, n_consts, degree, "g_poly_degree", ins, &n_slots);
  if (!why.empty()) return why;
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
  return "";
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

int lasso_bind_top(lasso_ctx* h, uint64_t* Z, size_t len, const uint64_t r[4]) {
  LB_TRY_CTX(h)
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "bind_top: len must be a power of two >= 2");
  Ctx* c = h->c;
  DBuf<fr_t> d(c, len);
  LB_CUDA_CHECK(cudaMemcpyAsync(d.p, Z, len * 32, cudaMemcpyHostToDevice, c->st));
  fr_t rr;
  memcpy(rr.v, r, 32);
  launch_bind_top(d.p, 0, 1, len / 2, rr, c->st);
  LB_CUDA_CHECK(cudaMemcpyAsync(Z, d.p, (len / 2) * 32, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
  LB_CATCH
}
int lasso_bind_bot(lasso_ctx* h, uint64_t* Z, size_t len, const uint64_t r[4]) {
  LB_TRY_CTX(h)
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "bind_bot: len must be a power of two >= 2");
  Ctx* c = h->c;
  DBuf<fr_t> d(c, len), o(c, len / 2);
  LB_CUDA_CHECK(cudaMemcpyAsync(d.p, Z, len * 32, cudaMemcpyHostToDevice, c->st));
  fr_t rr;
  memcpy(rr.v, r, 32);
  launch_bind_bot(d.p, o.p, len / 2, rr, c->st);
  LB_CUDA_CHECK(cudaMemcpyAsync(Z, o.p, (len / 2) * 32, cudaMemcpyDeviceToHost, c->st));
  c->sync();
  return 0;
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
int lasso_sumcheck_round_arbitrary(lasso_ctx* h, int strategy, int C, int log_M, int log_R,
                                   const uint64_t* const* polys, size_t len, uint64_t* evals_out) {
  LB_TRY_CTX(h)
  Strategy S = mkS(strategy, C, log_M, log_R);
  if (!S.valid()) return fail(LASSO_ERR_STRATEGY, "unsupported strategy parameters");
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "len must be a power of two >= 2");
  Ctx* c = h->c;
  int np = S.num_memories() + 1, npts = S.sumcheck_poly_degree() + 1;
  DBuf<fr_t> d(c, (size_t)np * len);
  for (int k = 0; k < np; k++)
    LB_CUDA_CHECK(cudaMemcpyAsync(d.p + (size_t)k * len, polys[k], len * 32, cudaMemcpyHostToDevice, c->st));
  const Finalize f = c->fin_begin();
  launch_sumcheck_eval_arbitrary(S, d.p, len, len / 2, f, c->st);
  c->fin_wait(f, (fr_t*)evals_out, npts);
  return 0;
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
  auto t0 = std::chrono::steady_clock::now();
  int err = 0;
  Dense* d = densify(h->c, indices, n_lookups, C, log_m, &err);
  if (!d) return fail(err == 3 ? LASSO_ERR_INDEX_RANGE : LASSO_ERR_STRATEGY, "densify: invalid input");
  h->c->t_densify_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  *out = new lasso_dense{d};
  return 0;
  LB_CATCH
}
int lasso_densify_device(lasso_ctx* h, const void* indices, size_t elem_bytes, size_t n_lookups, size_t C,
                         size_t row_stride, size_t col_stride, size_t log_m, void* stream, lasso_dense** out) {
  LB_TRY_CTX(h)
  *out = nullptr;
  auto t0 = std::chrono::steady_clock::now();
  int err = 0;
  Dense* d = densify_device(h->c, indices, elem_bytes, n_lookups, C, row_stride, col_stride, log_m,
                            static_cast<cudaStream_t>(stream), &err);
  if (err == 3) return fail(LASSO_ERR_INDEX_RANGE, "densify_device: an index is >= m");
  if (err == 7) return fail(LASSO_ERR_POINTER, "densify_device: the indices are not device memory of the context's GPU");
  if (!d) return fail(LASSO_ERR_STRATEGY, "densify_device: invalid input");
  h->c->t_densify_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
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
  auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> b = commit(h->c, *d->d, *g->g);
  h->c->t_commit_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  *out_len = b.size();
  if (b.size() > cap) return fail(LASSO_ERR_LENGTH, "commit: output buffer too small");
  memcpy(out, b.data(), b.size());
  return 0;
  LB_CATCH
}

}  // extern "C"

// lasso_prove / lasso_prove_custom after the strategy has been checked
static int prove_checked(lasso_ctx* h, const Strategy& S, lasso_dense* d, const uint64_t* r, size_t r_len,
                         const lasso_gens* g, const char* transcript_label, const char* tape_label,
                         const uint64_t tape_seed[4], uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                         uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges) {
  // assert_eq!(r.len(), log2(dense.s))  surge.rs:131
  if (r_len != log2_exact_or_ceil(d->d->s)) return fail(LASSO_ERR_LENGTH, "r.len() != log2(s)");
  std::vector<fr_t> rv(r_len);
  for (size_t i = 0; i < r_len; i++) memcpy(rv[i].v, r + 4 * i, 32);
  fr_t seed;
  memcpy(seed.v, tape_seed, 32);
  std::vector<fr_t> trace;
  auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> b;
  try {
    b = prove(h->c, S, *d->d, rv, *g->g, transcript_label, tape_label, seed, &trace);
  } catch (const std::runtime_error& e) {
    if (std::string(e.what()).find("multiset") != std::string::npos) return fail(LASSO_ERR_MULTISET, e.what());
    throw;
  }
  h->c->t_prove_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  *proof_len = b.size();
  if (n_challenges) *n_challenges = trace.size();
  if (challenges_out)
    for (size_t i = 0; i < trace.size() && i < challenges_cap; i++) memcpy(challenges_out + 4 * i, trace[i].v, 32);
  if (b.size() > proof_cap) return fail(LASSO_ERR_LENGTH, "prove: output buffer too small");
  memcpy(proof_out, b.data(), b.size());
  return 0;
}

extern "C" {

int lasso_prove(lasso_ctx* h, int strategy, int log_R, lasso_dense* d, const uint64_t* r, size_t r_len,
                const lasso_gens* g, const char* transcript_label, const char* tape_label, const uint64_t tape_seed[4],
                uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t* challenges_out,
                size_t challenges_cap, size_t* n_challenges) {
  LB_TRY_CTX(h)
  Strategy S = mkS(strategy, (int)d->d->C, (int)d->d->log_m, log_R);
  if (!S.valid()) return fail(LASSO_ERR_STRATEGY, "unsupported strategy parameters");
  if (!S.provable())
    return fail(LASSO_ERR_STRATEGY, "prove: " + std::to_string(2 * S.num_memories()) +
                                        " grand-product circuits exceed the batch limit of 32 (LT needs C <= 8)");
  return prove_checked(h, S, d, r, r_len, g, transcript_label, tape_label, tape_seed, proof_out, proof_cap, proof_len,
                       challenges_out, challenges_cap, n_challenges);
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
  if (out) *out = nullptr;
  CustomStrategy cs;
  std::vector<CustomIns> ins;
  const std::string why = custom_check(C, log_m, num_subtables, num_memories, mem_to_subtable, mem_to_dimension, program,
                                       n_ops, constants, n_constants, g_degree, cs, ins);
  if (!why.empty()) return fail(LASSO_ERR_STRATEGY, "strategy: " + why);
  if (!out || !tables) return fail(LASSO_ERR_STRATEGY, "strategy: null tables or output");
  for (int k = 0; k < num_subtables; k++)
    if (!tables[k]) return fail(LASSO_ERR_STRATEGY, "strategy: null table");
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
  if (out) *out = nullptr;
  CustomStrategy cs;
  std::vector<CustomIns> ins;
  const std::string why = custom_check(C, log_m, num_subtables, num_memories, mem_to_subtable, mem_to_dimension, program,
                                       n_ops, constants, n_constants, g_degree, cs, ins);
  if (!why.empty()) return fail(LASSO_ERR_STRATEGY, "strategy: " + why);
  if (!out || !tables) return fail(LASSO_ERR_STRATEGY, "strategy: null tables or output");
  for (int k = 0; k < num_subtables; k++)
    if (!tables[k]) return fail(LASSO_ERR_STRATEGY, "strategy: null table");
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
  if (!is_pow2(len) || len < 2) return fail(LASSO_ERR_NOT_POW2, "len must be a power of two >= 2");
  Ctx* c = h->c;
  const Strategy S = s->S();
  const int np = S.num_memories() + 1, npts = S.sumcheck_poly_degree() + 1;
  DBuf<fr_t> d(c, (size_t)np * len);
  for (int k = 0; k < np; k++)
    LB_CUDA_CHECK(cudaMemcpyAsync(d.p + (size_t)k * len, polys[k], len * 32, cudaMemcpyHostToDevice, c->st));
  const Finalize f = c->fin_begin();
  launch_sumcheck_eval_arbitrary(S, d.p, len, len / 2, f, c->st);
  c->fin_wait(f, (fr_t*)evals_out, npts);
  return 0;
  LB_CATCH
}
int lasso_prove_custom(lasso_ctx* h, const lasso_strategy* s, lasso_dense* d, const uint64_t* r, size_t r_len,
                       const lasso_gens* g, const char* transcript_label, const char* tape_label,
                       const uint64_t tape_seed[4], uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                       uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges) {
  LB_TRY_CTX(h)
  if (!s || s->c != h->c) return fail(LASSO_ERR_STRATEGY, "strategy was created on another context");
  if ((size_t)s->cs.C != d->d->C || (size_t)s->cs.log_m != d->d->log_m)
    return fail(LASSO_ERR_STRATEGY, "strategy (C, log_m) differ from the densified representation");
  return prove_checked(h, s->S(), d, r, r_len, g, transcript_label, tape_label, tape_seed, proof_out, proof_cap, proof_len,
                       challenges_out, challenges_cap, n_challenges);
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
static int poly_ctx_check(lasso_ctx* h) {
  if (h->c->world > 1) return fail(LASSO_ERR_STRATEGY, "dense polynomials are not available on a sharded context");
  return 0;
}
size_t lasso_poly_gens_points_needed(size_t num_vars) { return poly_R(num_vars) + 2; }
int lasso_poly_gens_create(lasso_ctx* h, const uint64_t* stream_affine, size_t n_points, size_t num_vars,
                           lasso_poly_gens** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!out || !stream_affine) return fail(LASSO_ERR_GENS, "poly gens: null stream or output");
  if (num_vars > 28) return fail(LASSO_ERR_LENGTH, "poly gens: num_vars <= 28");
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
static int poly_new(lasso_ctx* h, const uint64_t* Z, size_t len, size_t row_stride, bool device, void* stream,
                    lasso_poly** out) {
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!out) return fail(LASSO_ERR_LENGTH, "poly: null output");
  if (!is_pow2(len)) return fail(LASSO_ERR_NOT_POW2, "poly: the length must be a power of two (dense_mlpoly.rs:63-66)");
  if (len > kPolyMaxLen) return fail(LASSO_ERR_LENGTH, "poly: at most 2^28 evaluations");
  if (row_stride < 4) return fail(LASSO_ERR_LENGTH, "poly: row_stride must be at least 4 u64");
  if (!device && !Z) return fail(LASSO_ERR_POINTER, "poly: null evaluations");
  int err = 0;
  Poly* p = poly_create(h->c, Z, len, row_stride, device, static_cast<cudaStream_t>(stream), &err);
  if (err == 7) return fail(LASSO_ERR_POINTER, "poly: the evaluations are not device memory of the context's GPU");
  if (err == 8) return fail(LASSO_ERR_VALUE, "poly: an evaluation is not a canonical Montgomery residue");
  *out = new lasso_poly{p};
  return 0;
}
int lasso_poly_create(lasso_ctx* h, const uint64_t* Z, size_t len, lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_new(h, Z, len, 4, false, nullptr, out);
  LB_CATCH
}
int lasso_poly_create_device(lasso_ctx* h, const uint64_t* Z, size_t len, size_t row_stride, void* stream,
                             lasso_poly** out) {
  LB_TRY_CTX(h)
  return poly_new(h, Z, len, row_stride, true, stream, out);
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
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
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
  const size_t need = 8 + 32 * ((size_t)1 << (p->p->nv / 2));
  if (out_len) *out_len = need;
  if (!out || cap < need) return fail(LASSO_ERR_LENGTH, "poly commit: output buffer too small");
  auto t0 = std::chrono::steady_clock::now();
  const std::vector<uint8_t> b = poly_commit(h->c, *p->p, *g->g);
  h->c->t_commit_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  memcpy(out, b.data(), b.size());
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
  LB_TRY_CTX(h)
  if (const int rc = poly_use_check(h, p, g)) return rc;
  if (!g) return fail(LASSO_ERR_GENS, "poly eval proof: null generators");
  if (!transcript || !tape) return fail(LASSO_ERR_LENGTH, "poly eval proof: null transcript or random tape");
  std::vector<fr_t> rv, zr;
  if (const int rc = load_point(*p->p, r, r_len, rv)) return rc;
  if (!load_scalars(Zr, 1, zr)) return fail(LASSO_ERR_VALUE, "poly eval proof: Zr is not a canonical residue");
  // the proof's size is fixed by num_vars: L_vec and R_vec of log2(R) points, delta, beta, z1, z2
  const size_t lg = p->p->nv - p->p->nv / 2, need = 2 * (8 + 32 * lg) + 4 * 32;
  if (proof_len) *proof_len = need;
  if (!proof_out || proof_cap < need) return fail(LASSO_ERR_LENGTH, "poly eval proof: output buffer too small");
  auto t0 = std::chrono::steady_clock::now();
  uint8_t czr[32];
  const std::vector<uint8_t> b = poly_eval_prove(h->c, *p->p, *g->g, rv, zr[0], transcript->t, tape->t, czr);
  h->c->t_prove_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (b.size() != need) return fail(-1, "poly eval proof: unexpected proof size");
  memcpy(proof_out, b.data(), b.size());
  if (C_Zr_out) memcpy(C_Zr_out, czr, 32);
  return 0;
  LB_CATCH
}
int lasso_poly_create_eq(lasso_ctx* h, const uint64_t* r, size_t r_len, lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!out) return fail(LASSO_ERR_LENGTH, "eq poly: null output");
  if (r_len > 28) return fail(LASSO_ERR_LENGTH, "eq poly: at most 28 variables (2^28 evaluations)");
  if (r_len && !r) return fail(LASSO_ERR_LENGTH, "eq poly: null point");
  std::vector<fr_t> rv;
  if (!load_scalars(r, r_len, rv)) return fail(LASSO_ERR_VALUE, "eq poly: a coordinate of r is not a canonical residue");
  *out = new lasso_poly{poly_create_eq(h->c, rv)};
  return 0;
  LB_CATCH
}

// ---- many polynomials per call: merge, batched evaluation, one combined opening
int lasso_poly_create_merge(lasso_ctx* h, const lasso_poly* const* polys, size_t n_polys, lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!polys || n_polys == 0 || !out) return fail(LASSO_ERR_LENGTH, "merge: no polynomials, or a null output");
  for (size_t j = 0; j < n_polys; j++)
    if (const int rc = poly_use_check(h, polys[j], nullptr)) return rc;
  size_t total = 0;
  for (size_t j = 0; j < n_polys; j++) {
    total += polys[j]->p->len;  // each len <= 2^28: the running sum cannot wrap before it passes the limit
    if (total > kPolyMaxLen) return fail(LASSO_ERR_LENGTH, "merge: at most 2^28 evaluations after padding");
  }
  std::vector<const Poly*> ps(n_polys);
  for (size_t j = 0; j < n_polys; j++) ps[j] = polys[j]->p;
  *out = new lasso_poly{poly_merge(h->c, ps.data(), (int)n_polys)};
  return 0;
  LB_CATCH
}
int lasso_poly_evaluate_batch(lasso_ctx* h, const lasso_poly* const* polys, size_t n_polys, const uint64_t* r,
                              size_t r_len, uint64_t* out) {
  LB_TRY_CTX(h)
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!polys || n_polys == 0 || n_polys > (size_t)kDotMaxPolys || !out)
    return fail(LASSO_ERR_LENGTH, "evaluate batch: 1..64 polynomials and an output");
  for (size_t j = 0; j < n_polys; j++)
    if (const int rc = poly_use_check(h, polys[j], nullptr)) return rc;
  for (size_t j = 1; j < n_polys; j++)
    if (polys[j]->p->nv != polys[0]->p->nv) return fail(LASSO_ERR_LENGTH, "evaluate batch: the polynomials have different num_vars");
  std::vector<fr_t> rv;
  if (const int rc = load_point(*polys[0]->p, r, r_len, rv)) return rc;
  std::vector<const Poly*> ps(n_polys);
  for (size_t j = 0; j < n_polys; j++) ps[j] = polys[j]->p;
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
  // the PolyEvalProof of lasso_poly_eval_prove at num_vars
  const size_t lg = nv - nv / 2, need = 2 * (8 + 32 * lg) + 4 * 32;
  if (proof_len) *proof_len = need;
  if (!proof_out || proof_cap < need) return fail(LASSO_ERR_LENGTH, "combined eval proof: output buffer too small");
  if (!transcript || !tape) return fail(LASSO_ERR_LENGTH, "combined eval proof: null transcript or random tape");
  std::vector<fr_t> ev, rv;
  if (!load_scalars(evals, n_evals, ev)) return fail(LASSO_ERR_VALUE, "combined eval proof: an eval is not a canonical residue");
  if (!load_scalars(r, r_len, rv)) return fail(LASSO_ERR_VALUE, "combined eval proof: a coordinate of r is not a canonical residue");
  auto t0 = std::chrono::steady_clock::now();
  const std::vector<uint8_t> b = combined_eval_prove(h->c, *combined->p, *g->g, ev, rv, transcript->t, tape->t);
  h->c->t_prove_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (b.size() != need) return fail(-1, "combined eval proof: unexpected proof size");
  memcpy(proof_out, b.data(), b.size());
  return 0;
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
  for (size_t j = 0; j < n_polys; j++)
    if (const int rc = poly_use_check(h, polys[j], nullptr)) return rc;
  const size_t nv = polys[0]->p->nv;
  for (size_t j = 1; j < n_polys; j++)
    if (polys[j]->p->nv != nv) return fail(LASSO_ERR_LENGTH, "sumcheck: the polynomials have different num_vars");
  if (num_rounds < 1 || num_rounds > nv) return fail(LASSO_ERR_LENGTH, "sumcheck: num_rounds must be in 1..num_vars");
  // SumcheckInstanceProof: a u64 count, then per round a u64 length and the degree coefficients except the linear one
  const size_t need = 8 + num_rounds * (8 + 32 * (size_t)g->g.degree);
  if (proof_len) *proof_len = need;
  if (!proof_out || proof_cap < need) return fail(LASSO_ERR_LENGTH, "sumcheck: output buffer too small");
  if (!transcript || !r_out || !final_evals_out) return fail(LASSO_ERR_LENGTH, "sumcheck: null transcript or output");
  std::vector<const Poly*> ps(n_polys);
  for (size_t j = 0; j < n_polys; j++) ps[j] = polys[j]->p;
  auto t0 = std::chrono::steady_clock::now();
  const SumcheckOut o = sumcheck_prove(h->c, g->g, ps.data(), (int)n_polys, num_rounds, transcript->t);
  h->c->t_prove_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (o.proof.size() != need) return fail(-1, "sumcheck: unexpected proof size");
  memcpy(proof_out, o.proof.data(), need);
  for (size_t j = 0; j < num_rounds; j++) memcpy(r_out + 4 * j, o.r[j].v, 32);
  for (size_t j = 0; j < n_polys; j++) memcpy(final_evals_out + 4 * j, o.final_evals[j].v, 32);
  if (claim_out) memcpy(claim_out, o.claim.v, 32);
  return 0;
  LB_CATCH
}
int lasso_poly_create_comb(lasso_ctx* h, const lasso_comb* g, const lasso_poly* const* polys, size_t n_polys,
                           lasso_poly** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
  if (poly_ctx_check(h)) return LASSO_ERR_STRATEGY;
  if (!g) return fail(LASSO_ERR_STRATEGY, "comb poly: null combining function");
  if (!polys || n_polys != (size_t)g->g.n_inputs)
    return fail(LASSO_ERR_STRATEGY, "comb poly: " + std::to_string(n_polys) + " polynomials for a combining function of " +
                                        std::to_string(g->g.n_inputs) + " inputs");
  for (size_t j = 0; j < n_polys; j++)
    if (const int rc = poly_use_check(h, polys[j], nullptr)) return rc;
  for (size_t j = 1; j < n_polys; j++)
    if (polys[j]->p->nv != polys[0]->p->nv) return fail(LASSO_ERR_LENGTH, "comb poly: the polynomials have different num_vars");
  if (!out) return fail(LASSO_ERR_LENGTH, "comb poly: null output");
  std::vector<const Poly*> ps(n_polys);
  for (size_t j = 0; j < n_polys; j++) ps[j] = polys[j]->p;
  *out = new lasso_poly{poly_create_comb(h->c, g->g, ps.data(), (int)n_polys)};
  return 0;
  LB_CATCH
}

// ---- grand products over a caller's polynomials
int lasso_gp_circuit_create(lasso_ctx* h, const lasso_poly* p, lasso_gp_circuit** out) {
  LB_TRY_CTX(h)
  if (out) *out = nullptr;
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
  // per layer i < v: a sumcheck of i cubic rounds (8 + 8 + 104 i) and two vectors of n claims (2 (8 + 32 n))
  const size_t need = 8 + v * (24 + 64 * n) + 52 * v * (v - 1);
  if (proof_len) *proof_len = need;
  if (!proof_out || proof_cap < need) return fail(LASSO_ERR_LENGTH, "grand product: output buffer too small");
  if (!transcript || !r_out || !claims_out) return fail(LASSO_ERR_LENGTH, "grand product: null transcript or output");
  std::vector<Circuit*> cs(n);
  std::vector<fr_t> products(n);
  for (size_t k = 0; k < n; k++) {
    cs[k] = circuits[k]->ci.get();
    products[k] = circuits[k]->product;
    circuits[k]->proven = true;
  }
  auto t0 = std::chrono::steady_clock::now();
  const GrandProductOut o = gp_prove(h->c, cs, products, transcript->t);
  h->c->t_prove_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (o.proof.size() != need) return fail(-1, "grand product: unexpected proof size");
  memcpy(proof_out, o.proof.data(), need);
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
