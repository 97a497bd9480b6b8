// lasso_b200 — host-side prover objects: context, device buffers, generator tables, the
// densified representation and the proof byte writer.  The prover logic is in prover.cu.
#pragma once
#include <sched.h>

#include <atomic>
#include <chrono>
#include <map>
#include <memory>
#include <stdexcept>
#include <vector>

#include "../../include/lasso_b200.h"
#include "host_transcript.hpp"
#include "kernels.cuh"
#include "msm.cuh"

namespace lb {

// A failure of the caller's input that the C boundary returns as its own LASSO_ERR_* code; any other exception is -1
struct LbError : std::runtime_error {
  int code;
  LbError(int code, const std::string& msg) : std::runtime_error(msg), code(code) {}
};

struct Ctx {
  int device = 0;
  cudaStream_t st = nullptr;
  uint8_t* h_pin = nullptr;  // pinned staging for small device->host results
  size_t h_pin_bytes = 0;
  fr_t* d_partial = nullptr;  // block partial sums / bound chunks
  size_t partial_elems = 0;
  fr_t* d_small = nullptr;  // small results (<= 64K elements)
  size_t small_elems = 0;
  fr_t* d_eq_scratch = nullptr;
  unsigned* d_flag = nullptr;
  uint32_t* h_stage = nullptr;  // pinned staging for the densified integer arrays (grown on demand, reused)
  size_t h_stage_elems = 0;
  uint32_t* stage(size_t elems) {
    if (elems > h_stage_elems) {
      if (h_stage) cudaFreeHost(h_stage);
      h_stage = nullptr;
      h_stage_elems = 0;  // a failed allocation below must not leave a stale size behind
      LB_CUDA_CHECK(cudaMallocHost((void**)&h_stage, elems * sizeof(uint32_t)));
      h_stage_elems = elems;
    }
    return h_stage;
  }
  // ---- single proof sharded over `world` GPUs (comm.cu); world == 1: everything below is inert
  int world = 1, rank = 0, lg_world = 0;
  void* xchg = nullptr;  // comm.cu: shared host segments + peer exchange buffers
  bool h_pub_owned = false;
  fr_t* d_gather = nullptr;  // all-gather landing zone
  size_t gather_elems = 0;
  double t_densify_ms = 0, t_commit_ms = 0, t_prove_ms = 0;
  std::map<std::string, double> spans;  // filled when LASSO_B200_SPANS=1 (forces syncs)
  bool span_sync = false;

  void sync() { LB_CUDA_CHECK(cudaStreamSynchronize(st)); }
  // Small results (<= 4 KiB) that are not round messages: a one-warp kernel copies the result into mapped pinned
  // host memory and then raises a sequence flag (system-scope fence); the host spins on the flag instead of paying
  // for cudaMemcpyAsync + cudaStreamSynchronize.
  uint32_t* h_mapped = nullptr;  // [0..1024) payload words, [1024] flag
  uint32_t* d_mapped = nullptr;
  uint32_t mapped_seq = 0;
  static constexpr size_t kMappedBytes = 8192;
  // Tagged publication of round messages and MSM points (common.cuh PubDst): this process's receive buffer
  // [writer][region][element][kPubSlotWords] and the device view of every reader's buffer (world == 1: only its
  // own, plain cudaHostAlloc; world > 1: shared pinned host segments mapped by every process, comm.cu)
  unsigned long long* h_pub = nullptr;
  unsigned long long* d_pub_reader[kPubMaxReaders] = {};
  // messages so far to this process only [0] and to every process [1]: the next region of each ring, and its tag.
  // Each ring counts its own messages, so that a rank's private messages (their number may depend on the tables
  // its GPU holds) never shift the tags of the messages every rank of a sharded context exchanges.
  uint32_t pub_ring[2] = {0, 0};
  static constexpr size_t kPubBytes = (size_t)kPubMaxReaders * kPubRegions * kPubElems * kPubSlotWords * 8;  // 1 MiB
  cudaEvent_t ev_aux = nullptr;  // marks a device->host copy that overlaps later launches on the same stream
  cudaEvent_t ev_caller = nullptr;  // densify_device: the caller's stream up to the call (the index matrix is ready)
  cudaEvent_t ev_stage = nullptr;  // recorded after the last upload out of h_stage (the buffer is reused by the next densify)
  bool stage_busy = false;
  // host-thread placement (bind_host_threads): the CPUs the library's helper threads may use
  cpu_set_t helper_mask;
  bool have_helper_mask = false;
  void helper_thread_enter() const {
    if (have_helper_mask) sched_setaffinity(0, sizeof helper_mask, &helper_mask);
  }
  void d2h_small(void* dst, const void* src, size_t bytes);  // prover.cu
  void wait_flag(uint32_t seq);                               // prover.cu
  // next message: `all` = every rank stores into every reader's buffer and the readers add the G residues
  // (the per-round exchange of a sharded proof); otherwise the message goes to this process only
  PubDst pub_begin(bool all) {
    PubDst p;
    p.ndst = 0;
    p.tag = 0;
    p.region = 0;
    p.all = 0;
    for (int i = 0; i < kPubMaxReaders; i++) p.dst[i] = nullptr;
    p.all = (all && world > 1) ? 1 : 0;
    // A peer reads this writer's message to every process before it launches its next one, so in a peer's buffer a
    // region is free again two such messages later.  Messages to this process only take no peer with them: were they
    // to advance the same ring, a writer running ahead through them would reuse a region a peer has not read yet.
    const uint32_t seq = pub_ring[p.all]++;
    p.region = (int)(seq % kPubRegions);
    p.tag = 1 + seq % kPubTagMod;
    const size_t off = ((size_t)rank * kPubRegions + p.region) * kPubElems * kPubSlotWords;
    if (p.all) {
      for (int r = 0; r < world; r++) p.dst[p.ndst++] = d_pub_reader[r] + off;
    } else {
      p.dst[p.ndst++] = d_pub_reader[rank] + off;
    }
    return p;
  }
  // count elements of 8 x u32 words from one writer's region; blocks until every word carries the tag
  void pub_wait_raw(const PubDst& p, int writer, int count, uint32_t* out);  // prover.cu
  // a round message produced by a single launch (common.cuh Finalize): results land directly in the mapped host
  // buffer(s); reduce = sum over the ranks of a sharded proof
  Finalize fin_begin(bool reduce = false) {
    Finalize f;
    f.partial = d_partial;
    f.counter = d_flag + 4;
    f.pub = pub_begin(reduce);
    return f;
  }
  void fin_wait(const Finalize& f, fr_t* dst, int count);  // prover.cu (adds the residues of all ranks when f.pub.all)
  // npoints x (X, Y, Z) canonical Fq limbs published by msm_finish_quad_kernel
  void wait_points(const PubDst& p, int npoints, uint32_t* xyz /* npoints x 24 words */);
  // device -> host through the pinned buffer (small) or directly (large)
  void d2h(void* dst, const void* src, size_t bytes) {
    if (bytes <= 4096) {
      d2h_small(dst, src, bytes);
      return;
    }
    if (bytes <= h_pin_bytes) {
      LB_CUDA_CHECK(cudaMemcpyAsync(h_pin, src, bytes, cudaMemcpyDeviceToHost, st));
      sync();
      memcpy(dst, h_pin, bytes);
    } else {
      LB_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
      sync();
    }
  }
  void h2d(void* dst, const void* src, size_t bytes) {
    LB_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
    sync();  // the source may be a stack / pageable buffer
  }
};

// While helper threads are being CREATED the calling thread widens its own affinity to the helper CPUs: a new thread
// inherits its creator's mask, and a creator pinned to one core that goes on to spin there would leave its children
// waiting for that very core before they can even move themselves (milliseconds).  Restored on scope exit.
struct HelperSpawnScope {
  cpu_set_t saved;
  bool active = false;
  HelperSpawnScope(const Ctx* c, bool spawning) {
    if (spawning && c->have_helper_mask && sched_getaffinity(0, sizeof saved, &saved) == 0)
      active = sched_setaffinity(0, sizeof c->helper_mask, &c->helper_mask) == 0;
  }
  ~HelperSpawnScope() {
    if (active) sched_setaffinity(0, sizeof saved, &saved);
  }
};

// stream-ordered device buffer
template <class T>
struct DBuf {
  T* p = nullptr;
  size_t n = 0;
  Ctx* c = nullptr;
  DBuf() {}
  DBuf(Ctx* ctx, size_t count) { alloc(ctx, count); }
  void alloc(Ctx* ctx, size_t count) {
    release();
    c = ctx;
    n = count;
    if (count) LB_CUDA_CHECK(cudaMallocAsync((void**)&p, count * sizeof(T), ctx->st));
  }
  void release() {
    if (p) cudaFreeAsync(p, c->st);
    p = nullptr;
    n = 0;
  }
  ~DBuf() { release(); }
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  DBuf(DBuf&& o) noexcept : p(o.p), n(o.n), c(o.c) { o.p = nullptr; }
  DBuf& operator=(DBuf&& o) noexcept {
    release();
    p = o.p;
    n = o.n;
    c = o.c;
    o.p = nullptr;
    return *this;
  }
};

struct SpanTimer {
  Ctx* c;
  const char* name;
  std::chrono::steady_clock::time_point t0;
  SpanTimer(Ctx* ctx, const char* n) : c(ctx), name(n) {
    if (c->span_sync) {
      c->sync();
      t0 = std::chrono::steady_clock::now();
    }
  }
  ~SpanTimer() {
    if (c->span_sync) {
      c->sync();
      c->spans[name] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
  }
};

// SparsePolyCommitmentGens<G> (lasso/surge.rs:25-58): one generator stream, three (n, Q, h) views
struct Gens {
  Ctx* ctx = nullptr;
  size_t n_points = 0;
  size_t c = 0, s = 0, num_memories = 0, log_m = 0;
  size_t nv_l = 0, nv_m = 0, nv_d = 0;  // num_vars of the three committed polynomials
  DBuf<fq_t> d_bases_ark;               // n_points x (x, y)
  DBuf<pt_niels> d_table;               // kMsmFullWindows x n_points, T[w][j] = 2^(8w) G_j
  // multiples M[w][j][d-1] = d * T[w][j] (d = 1..128) of the first n_direct generators: the bucket-free MSM of
  // the opening proofs (msm_kernels.cu).  Single-GPU contexts only; empty -> the bucket MSM is used.
  DBuf<pt_niels> d_multiples;
  size_t n_direct = 0;
  // 16-bit multiples M16[j][d-1] = d * G_j (d = 1..32768) of the first n_direct16 generators: the Hyrax row
  // commitments of integer-valued polynomials (3 MB per generator; LASSO_B200_TABLE_GB caps it, default 64)
  DBuf<pt_niels> d_multiples16;
  size_t n_direct16 = 0;
  DBuf<pt_ext> d_centre;  // centring constants 2^15 * sum_{j < R} G_j for R = 2^k, k = 0 .. 31 (entry k; msm_kernels.cu)
};

// DensifiedRepresentation<F, C> (lasso/densified.rs:8-18), device resident
struct Dense {
  Ctx* ctx = nullptr;
  size_t C = 0, s = 0, log_m = 0, m = 0, nv_l = 0, nv_m = 0;
  size_t s_loc = 0, m_loc = 0;  // this rank's share (s / G, m / G): element i' is global element i'*G + rank
  DBuf<uint32_t> d_l_u32;  // (2^nv_l)/G: dim_0..dim_{C-1} | read_0..read_{C-1} | 0..   (dim_usize = first C*s_loc)
  DBuf<uint32_t> d_m_u32;  // (2^nv_m)/G: final_0..final_{C-1} | 0..
  DBuf<fr_t> d_l_fr;       // combined_l_variate_polys (this rank's low-bit shard)
  DBuf<fr_t> d_m_fr;       // combined_log_m_variate_polys
  const uint32_t* nz() const { return d_l_u32.p; }
  const fr_t* dim(size_t i) const { return d_l_fr.p + i * s_loc; }
  const fr_t* read(size_t i) const { return d_l_fr.p + (C + i) * s_loc; }
  const fr_t* fin(size_t i) const { return d_m_fr.p + i * m_loc; }
};

// DensePolynomial<Fr> (poly/dense_mlpoly.rs:13-18) of a caller, device resident: the library's own copy of its
// evaluations, checked canonical on the way in (dense_poly_kernels.cu)
// On a sharded context every rank holds its low-bit shard, as Dense does: element i' is global element i'*G + rank, so
// for every one of the L rows the R/G columns congruent to the rank (poly_R(nv) >= G, poly_fits).
struct Poly {
  Ctx* ctx = nullptr;
  size_t len = 0, nv = 0;  // the whole polynomial
  size_t len_loc = 0;      // this rank's share, len / G: the length of d_fr and d_u32
  unsigned bits = 0;     // bit width of the widest value as an integer (0: the zero polynomial)
  DBuf<fr_t> d_fr;       // Montgomery form
  DBuf<uint32_t> d_u32;  // the same values as integers when bits <= 32 (commit_u32 / bound_u32), else empty
};

// GrandProductCircuit (grand_product.rs:14-66): layer k is one contiguous array of N/2^k elements,
// left_vec[k] = first half, right_vec[k] = second half; layer k+1[i] = layer k[i] * layer k[i + N/2^(k+1)].
// Sharded: layers with N/2^k >= G are held as low-bit shards (local length N/(2^k G)); the layer of global
// length G is all-gathered and the few layers above it are kept replicated on every rank.
// A caller's circuit (single GPU) has an external layer 0, the caller's polynomial, which is only read: `tree` holds
// layers 1.. (N - 2 elements), and the prover binds layer 0 out of place into layer 1's storage.
struct Circuit {
  DBuf<fr_t> tree;   // local shards: layer 0 at 0 (N/G elements), layer 1 after it, ...  (ext0: layer 1 at 0)
  fr_t* ext0 = nullptr;   // layer 0 when it is a caller's buffer, else null
  fr_t* rtree = nullptr;  // replicated top: layer k_rep (G elements), k_rep + 1, ... (2G slots in a shared allocation; G > 1)
  size_t N = 0, num_layers = 0;
  int G = 1;
  size_t k_rep = 0;  // first replicated layer: N >> k_rep == G
  bool layer_is_sharded(size_t k) const { return G == 1 || (N >> k) >= 2 * (size_t)G; }
  size_t layer_len_global(size_t k) const { return N >> k; }
  fr_t* layer_local(size_t k) const {  // valid for (N >> k) >= G
    if (ext0 && k == 0) return ext0;
    size_t off = 0, len = N / G;
    for (size_t i = 0; i < k; i++) {
      off += len;
      len /= 2;
    }
    return tree.p + (ext0 ? off - N : off);  // ext0: layer 0 is not stored
  }
  fr_t* layer_rep(size_t k) const {  // valid for k >= k_rep (G > 1)
    size_t off = 0, len = (size_t)G;
    for (size_t i = k_rep; i < k; i++) {
      off += len;
      len /= 2;
    }
    return rtree + off;
  }
};

// ark-serialize (compressed) writer
struct ByteWriter {
  std::vector<uint8_t> b;
  void u64(uint64_t v) {
    for (int i = 0; i < 8; i++) b.push_back((uint8_t)(v >> (8 * i)));
  }
  void fr(const fr_t& f) {
    uint8_t t[32];
    fr_to_bytes(f, t);
    b.insert(b.end(), t, t + 32);
  }
  void raw(const void* p, size_t n) { b.insert(b.end(), (const uint8_t*)p, (const uint8_t*)p + n); }
  void vec_fr(const std::vector<fr_t>& v) {
    u64(v.size());
    for (auto& f : v) fr(f);
  }
  void arr_fr(const std::vector<fr_t>& v) {
    for (auto& f : v) fr(f);
  }
  void vec_pts(const std::vector<uint8_t>& comp) {  // comp = 32 B per point
    u64(comp.size() / 32);
    raw(comp.data(), comp.size());
  }
};

inline size_t log2_exact_or_ceil(size_t x) {  // utils/math.rs:27-35 Math::log_2
  if ((x & (x - 1)) == 0) return (size_t)__builtin_ctzll((unsigned long long)x);
  return 64 - (size_t)__builtin_clzll((unsigned long long)x);
}
inline size_t next_pow2(size_t x) {
  size_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

// entry points implemented in prover.cu
int bind_host_threads(int device, cpu_set_t* helper_mask, bool* have_helper_mask);  // -> NUMA node or -1
Ctx* ctx_create(int device);
void ctx_destroy(Ctx*);
Gens* gens_create(Ctx*, const uint64_t* stream_affine, size_t n_points, size_t c, size_t s, size_t num_memories,
                  size_t log_m);
size_t gens_points_needed(size_t c, size_t s, size_t num_memories, size_t log_m);
// Both throw LbError: LASSO_ERR_INDEX_RANGE for an entry >= m, LASSO_ERR_STRATEGY for a bad shape or elem_bytes,
// LASSO_ERR_POINTER when the matrix is not device memory of the context's GPU.  Sharded: every rank throws together.
Dense* densify(Ctx*, const uint64_t* indices, size_t n_lookups, size_t C, size_t log_m);
Dense* densify_device(Ctx*, const void* indices, size_t elem_bytes, size_t n_lookups, size_t C, size_t row_stride,
                      size_t col_stride, size_t log_m, cudaStream_t caller);
std::vector<uint8_t> commit(Ctx*, const Dense&, const Gens&);
// SparsePolynomialEvaluationProof::prove (surge.rs:118-211) on the caller's transcript and tape, advanced in place.
// Throws before the first transcript write when S or g do not fit the dense; the working memory is reserved in the
// context's pool before it too.  *claimed_evaluation (may be null): the primary sumcheck's claim.  A failed multiset
// check throws LbError(LASSO_ERR_MULTISET) after the transcript has moved.
std::vector<uint8_t> prove(Ctx*, const Strategy& S, Dense&, const std::vector<fr_t>& r, const Gens&, Transcript&,
                           RandomTape&, fr_t* claimed_evaluation);
// Serialised sizes, fixed by the shapes.  prove's output (S and g fit dense):
size_t proof_bytes(const Strategy& S, const Dense&, const Gens&);
// the MemoryCheckingProof that ends prove's output and memory_check_prove's (S and g fit dense)
size_t memory_check_bytes(const Strategy& S, const Dense&, const Gens&);
// a PolyEvalProof at nv variables: L_vec and R_vec of nv - nv/2 points, delta, beta, z1, z2
size_t dpl_bytes(size_t nv);
// a BatchedGrandProductArgument over n circuits of v variables: layer j has j cubic rounds
size_t gpa_bytes(size_t n, size_t v);
// a SumcheckInstanceProof: a u64 count, then per round a u64 length and the degree coefficients except the linear one
size_t sumcheck_bytes(size_t rounds, size_t degree);
// a PolyCommitment at num_vars: a u64 count, then one point per row, 2^(num_vars/2) rows
size_t poly_commitment_bytes(size_t num_vars);
// The lookup outputs v[k] = combine_lookups(E_0[k], .., E_{alpha-1}[k]) for k < s as a new polynomial of log2(s)
// variables, with a u32 mirror when every value is below 2^32.  Single-GPU contexts (the caller checks).
Poly* dense_outputs(Ctx*, const Strategy& S, const Dense&);
void sample_generators(const std::string& label, size_t count, uint64_t* out_affine);

// Memory checking inside a caller's protocol (single GPU; the caller checks)
// Subtables::new (subtables/mod.rs:116-129): the alpha lookup polynomials E_i[j] = T_sub(i)[dim_i[j]] in memory order,
// each of log2(s) variables with storage of its own, bits = the tables' width, a u32 mirror when that is <= 32
std::vector<Poly*> lookup_polys(Ctx*, const Strategy& S, const Dense&);
// MemoryCheckingProof::prove (memory_checking.rs:56-83) at (gamma, tau) on the caller's transcript and tape, advanced in
// place; the lookup polynomials are rebuilt from (S, dense).  Throws before the first transcript write when S or g do
// not fit the dense, with the working memory reserved before it too; a failed multiset check throws
// LbError(LASSO_ERR_MULTISET) after the transcript has moved.
std::vector<uint8_t> memory_check_prove(Ctx*, const Strategy& S, const Dense&, const fr_t& gamma, const fr_t& tau,
                                        const Gens&, Transcript&, RandomTape&);
// dim_j, read_j or final_j (which = 1, 2, 3; j < C) as a new polynomial with its u32 mirror
Poly* dense_poly(Ctx*, const Dense&, int which, size_t j);
// GrandProducts::new (memory_checking.rs:175-310) with dim as dim_usize: out = init, read, write, final, full-width
// polynomials with hash(a, v, t) = t gamma^2 + v gamma + a - tau.  T.len == fin.len >= 2, dim.len == read.len >= 2,
// dim has a u32 mirror with every entry below T.len (the caller checks).
void memory_fingerprints(Ctx*, const Poly& T, const Poly& dim, const Poly& read, const Poly& fin, const fr_t& gamma,
                         const fr_t& tau, Poly* out[4]);

// dense polynomials of a caller (prover.cu): PolyCommitmentGens, DensePolynomial::{new, commit, evaluate},
// PolyEvalProof::prove.  On a sharded context the calls are collective: every rank calls them with the same arguments
// and gets the same results.  cubic_prove is collective too; the other sumchecks and the grand products below are
// single-GPU only.
static constexpr size_t kPolyMaxLen = (size_t)1 << 28;
inline size_t poly_R(size_t num_vars) { return (size_t)1 << (num_vars - num_vars / 2); }
// a polynomial of num_vars variables can be held on `world` ranks: every rank has at least one column of every row,
// R = 2^(num_vars - num_vars/2) >= world, i.e. num_vars >= 2 log2(world) - 1
inline bool poly_fits(size_t num_vars, int world) { return poly_R(num_vars) >= (size_t)world; }
// PolyCommitmentGens::new (dense_mlpoly.rs:38-45) from an explicit stream: G_0..G_{R-1}, Q = stream[R], h = stream[R+1];
// nullptr when n_points < R + 2
Gens* poly_gens_create(Ctx*, const uint64_t* stream_affine, size_t n_points, size_t num_vars);
// Z: len rows of 4 u64 Montgomery limbs, row_stride u64 apart; host memory, or device memory of the context's GPU
// (device != 0, read in the order of `caller`).  Throws LbError: LASSO_ERR_VALUE for an entry that is not a canonical
// residue, LASSO_ERR_POINTER for rows that are not device memory of the context's GPU.
// Any len: zero-padded to next_pow2(max(len, 1)) evaluations (DensePolynomial::new_padded, dense_mlpoly.rs:75-87).
// Sharded: every rank passes the whole polynomial and reads its rows; the verdict and the width are agreed by all ranks.
Poly* poly_create(Ctx*, const uint64_t* Z, size_t len, size_t row_stride, bool device, cudaStream_t caller);
std::vector<uint8_t> poly_commit(Ctx*, const Poly&, const Gens&);  // serialised PolyCommitment
// the hiding PolyCommitment of the same size: row i is committed with blinds[i] on h (blinds.size() == L)
std::vector<uint8_t> poly_commit_hiding(Ctx*, const Poly&, const Gens&, const std::vector<fr_t>& blinds);
fr_t poly_evaluate(Ctx*, const Poly&, const std::vector<fr_t>& r);
// serialised PolyEvalProof; C_Zr receives the compressed commitment to Zr the reference returns alongside it,
// Zr * Q + blind_Zr * h.  blinds: the commitment's L row blinds, or empty for None (zero blinds)
std::vector<uint8_t> poly_eval_prove(Ctx*, const Poly&, const Gens&, const std::vector<fr_t>& r, const fr_t& Zr,
                                     Transcript&, RandomTape&, uint8_t C_Zr[32], const std::vector<fr_t>& blinds = {},
                                     const fr_t& blind_Zr = fr_zero());
// EqPolynomial::new(r).evals() (eq_poly.rs:21-38) as a full-width polynomial (no u32 mirror); r.size() <= 28
Poly* poly_create_eq(Ctx*, const std::vector<fr_t>& r);
// DensePolynomial::merge (dense_mlpoly.rs:251-261) of k >= 1 polynomials (the caller checks the merged length): a new
// polynomial of its own, with a u32 mirror iff every input has one
Poly* poly_merge(Ctx*, const Poly* const* polys, int k);
// P_j(r) for 1 <= k <= kDotMaxPolys polynomials of one num_vars == r.size() (the caller checks), one eq table
std::vector<fr_t> poly_evaluate_batch(Ctx*, const Poly* const* polys, int k, const std::vector<fr_t>& r);
// CombinedTableEvalProof::prove (subtables/mod.rs:284-313) without blinds: the serialised PolyEvalProof at
// (challenges || r); p.nv == r.size() + log2(next_pow2(evals.size())) (the caller checks)
std::vector<uint8_t> combined_eval_prove(Ctx*, const Poly& p, const Gens& g, const std::vector<fr_t>& evals,
                                         const std::vector<fr_t>& r, Transcript&, RandomTape&);

// Transforms (DESIGN §3.14): new full-width polynomials, or copies, with storage of their own; the input is only read.
// Collective on a sharded context.  The caller checks 1 <= r.size() <= nv and poly_fits of the result.
// bound_poly_var_top with r[0], r[1], .. in turn (dense_mlpoly.rs:209-216)
Poly* poly_bind_top(Ctx*, const Poly&, const std::vector<fr_t>& r);
// bound_poly_var_bot with r[0], r[1], .. in turn (dense_mlpoly.rs:218-225): r[0] binds the lowest variable
Poly* poly_bind_bot(Ctx*, const Poly&, const std::vector<fr_t>& r);
// split(idx) (dense_mlpoly.rs:101-107), idx a power of two, 2 idx <= len: the parent's bits and u32 mirror, halved
void poly_split(Ctx*, const Poly&, size_t idx, Poly** lo, Poly** hi);
// the len evaluations in natural order, 4 Montgomery limbs each: to host memory, or (poly_read_device) to device
// memory of the context's GPU, row i at dst + i * row_stride, in the order of `caller`; LbError(LASSO_ERR_POINTER) when
// dst is not such memory
void poly_read(Ctx*, const Poly&, uint64_t* out);
void poly_read_device(Ctx*, const Poly&, uint64_t* dst, size_t row_stride, cudaStream_t caller);

// A combining function g(x_0..x_{n_inputs-1}) of SumcheckInstanceProof::prove_arbitrary: a checked program (capi.cu)
// with its slots allocated, and the declared combined_degree.  Host only.
struct Comb {
  int n_inputs = 0, degree = 0, n_slots = 0;
  std::vector<CustomIns> ins;
  std::vector<fr_t> consts;
};
struct SumcheckOut {
  std::vector<uint8_t> proof;  // ark-serialize (compressed) SumcheckInstanceProof
  std::vector<fr_t> r, final_evals;
  fr_t claim;  // e_0 + e_1 of the first round: the sum over the hypercube
};
// SumcheckInstanceProof::prove_arbitrary (sumcheck.rs:149-260) over polys[0..k), k == g.n_inputs, all of one num_vars,
// 1 <= num_rounds <= num_vars (the caller checks).  The polynomials are not modified: the first bind writes into a
// workspace of k x 2^(num_vars-1) elements, allocated before the transcript is touched.
SumcheckOut sumcheck_prove(Ctx*, const Comb& g, const Poly* const* polys, int k, size_t num_rounds, Transcript&);
// Q(x) = g(polys[0](x), .., polys[k-1](x)) at every point, k == g.n_inputs, all of one num_vars (the caller checks): a
// full-width polynomial like poly_create_eq
Poly* poly_create_comb(Ctx*, const Comb& g, const Poly* const* polys, int k);
struct CubicOut {
  std::vector<uint8_t> proof;  // ark-serialize (compressed) SumcheckInstanceProof
  std::vector<fr_t> r, finals;  // finals: A_0(..), .., A_{n-1}, B_0, .., B_{n-1}, C at (r || 0..0)
};
// SumcheckInstanceProof::prove_cubic_batched (sumcheck.rs:26-135) of claim = sum_x C(x) sum_k coeffs[k] A[k](x) B[k](x)
// over 1 <= n <= 32 pairs and C, all of one num_vars, 1 <= num_rounds <= num_vars (the caller checks).  The polynomials
// are not modified: the first bind writes a workspace, allocated before the transcript is touched.  Collective on a
// sharded context.
CubicOut cubic_prove(Ctx*, const Poly* const* A, const Poly* const* B, int n, const Poly& C,
                     const std::vector<fr_t>& coeffs, const fr_t& claim, size_t num_rounds, Transcript&);

// Zero-knowledge sumchecks (DESIGN §3.16)
// MultiCommitGens { n, G, h } (poly/commitments.rs:14-70) on the device: the 8-bit digit-multiples table of its n + 1
// points G_0..G_{n-1}, h (the layout of Gens::d_multiples), always built.  1 <= n <= kMcMaxN (the caller checks).
static constexpr size_t kMcMaxN = 1024;
struct McGens {
  Ctx* ctx = nullptr;
  size_t n = 0;
  DBuf<pt_niels> d_multiples;  // kMsmFullWindows x (n + 1) x 128
};
// G_affine: n points, h_affine: one, 64-byte affine layout (sample_generators)
McGens* mc_gens_create(Ctx*, const uint64_t* G_affine, size_t n, const uint64_t* h_affine);
// Commitments::batch_commit (commitments.rs:84-93), commit when n == 1: <scalars, G> + blind h, compressed
void mc_commit(Ctx*, const McGens&, const std::vector<fr_t>& scalars, const fr_t& blind, uint8_t out[32]);
// a DotProductProof of n elements: delta, beta, z (u64 count + n), z_delta, z_beta
inline size_t dot_product_bytes(size_t n) { return 136 + 32 * n; }
// DotProductProof::prove (subprotocols/dot_product.rs:31-93) on the caller's transcript and tape; gens_1.n == 1,
// gens_n.n == x.size() == a.size() (the caller checks).  Cx, Cy: the commitments the reference returns alongside.
std::vector<uint8_t> dot_product_prove(Ctx*, const McGens& gens_1, const McGens& gens_n, Transcript&, RandomTape&,
                                       const std::vector<fr_t>& x, const fr_t& blind_x, const std::vector<fr_t>& a,
                                       const fr_t& y, const fr_t& blind_y, uint8_t Cx[32], uint8_t Cy[32]);
// a ZKSumcheckInstanceProof of R rounds of degree d: comm_polys, comm_evals (u64 count + R points each), R proofs
inline size_t zk_sumcheck_bytes(size_t rounds, size_t degree) { return 24 + rounds * (200 + 32 * (degree + 1)); }
struct ZkSumcheckOut : SumcheckOut {
  uint8_t comm_claim[32];  // claim G_1 + blind_claim h_1
  fr_t blind_eval;         // the blind of the last comm_eval
};
// The prover of ZKSumcheckInstanceProof (verifier: subprotocols/sumcheck.rs:331-447) over the rounds of sumcheck_prove,
// the tape drawn up front: blinds_poly (R), blinds_evals (R), then every round's d_vec / r_delta / r_beta.
// gens_1.n == 1, gens_n.n == g.degree + 1, the rest as sumcheck_prove (the caller checks).
ZkSumcheckOut zk_sumcheck_prove(Ctx*, const Comb& g, const Poly* const* polys, int k, size_t num_rounds,
                                const fr_t& blind_claim, const McGens& gens_1, const McGens& gens_n, Transcript&,
                                RandomTape&);

// Σ-protocols of committed scalars (subprotocols/zk.rs, DESIGN §3.17) on the caller's transcript and tape; gens.n == 1
// (the caller checks).  Each is one short MSM of its 2, 3 or 6 rows and one host wait.  The proof bytes are
// ark-serialize compressed; the commitments are the points the reference returns alongside.
static constexpr size_t kKnowledgeProofBytes = 96;  // alpha, z1, z2
static constexpr size_t kEqualityProofBytes = 64;   // alpha, z
static constexpr size_t kProductProofBytes = 256;   // alpha, beta, delta, z[5]
std::vector<uint8_t> knowledge_prove(Ctx*, const McGens&, Transcript&, RandomTape&, const fr_t& x, const fr_t& r,
                                     uint8_t C[32]);
std::vector<uint8_t> equality_prove(Ctx*, const McGens&, Transcript&, RandomTape&, const fr_t& v1, const fr_t& s1,
                                    const fr_t& v2, const fr_t& s2, uint8_t C1[32], uint8_t C2[32]);
std::vector<uint8_t> product_prove(Ctx*, const McGens&, Transcript&, RandomTape&, const fr_t& x, const fr_t& rX,
                                   const fr_t& y, const fr_t& rY, const fr_t& z, const fr_t& rZ, uint8_t X[32],
                                   uint8_t Y[32], uint8_t Z[32]);

// grand products over a caller's polynomials (single GPU)
// GrandProductCircuit::new (grand_product.rs:38-58) with p as layer 0 (p.nv >= 1; p is only read and must outlive the
// circuit); *product receives evaluate() (grand_product.rs:60-65)
Circuit* gp_circuit_create(Ctx*, const Poly& p, fr_t* product);
struct GrandProductOut {
  std::vector<uint8_t> proof;   // ark-serialize (compressed) BatchedGrandProductArgument
  std::vector<fr_t> r, claims;  // rand and the final claims_to_verify (P_k(rand))
};
// BatchedGrandProductArgument::prove (grand_product.rs:100-201) on the caller's transcript; products[k] = evaluate() of
// circuits[k], all of one num_vars, at most 32.  The stored layers are bound in place, so a circuit is proven once.
GrandProductOut gp_prove(Ctx*, std::vector<Circuit*>& circuits, const std::vector<fr_t>& products, Transcript&);

// comm.cu
void comm_unique_id(uint8_t out[128]);
void comm_init(Ctx*, const uint8_t id[128], int rank, int world);
void comm_destroy(Ctx*);
void comm_allgather(Ctx*, const void* d_send, void* d_recv, size_t bytes_per_rank);
// every rank holds the low-bit shard (n_loc elements) of a vector; d_out <- the whole vector (n_loc * G), on every rank
void comm_gather_vector(Ctx*, const fr_t* d_shard, size_t n_loc, fr_t* d_scratch, fr_t* d_out);
// every rank holds a vector of m elements (a multiple of G); d_out (m / G) <- this rank's low-bit shard of their sum
void comm_sum_shard(Ctx*, const fr_t* d_vec, size_t m, fr_t* d_out);
// every rank holds one element per polynomial (ptrs[k][0], or base[k*stride] when ptrs == null);
// d_out[k*G + g] <- rank g's element of polynomial k
// `extra` (may be null): one more single-element polynomial, gathered as polynomial number npolys
void comm_gather_heads(Ctx*, fr_t* const* d_ptrs, const fr_t* base, size_t stride, int npolys, const fr_t* extra, fr_t* d_out);
void pack_heads(Ctx*, fr_t* const* d_ptrs, const fr_t* base, size_t stride, int npolys, fr_t* d_out);

}  // namespace lb
