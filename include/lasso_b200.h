/* lasso_b200 — C ABI of the H100-native Lasso prover hot path.
 *
 * This is the drop-in boundary for a16z/Lasso's
 *   DensifiedRepresentation::from_lookup_indices -> commit -> SparsePolynomialEvaluationProof::prove
 * path (SURVEY.md §8b).  The reference has no FFI of its own (it is three Rust generics); each entry
 * point below names the reference item it replaces (file:line relative to the reference's src/),
 * which is where a Rust maintainer would bind it (see INTEGRATION.md for the extern "C" shim).
 *
 * Conventions
 *  - field elements (curve25519 Fr) are 4 x uint64_t little-endian limbs in ark-ff Montgomery form
 *    (a * 2^256 mod l): a Rust `&[Fr]` can be passed as `*const u64` without conversion;
 *  - affine points are (x, y) = 2 x 4 x uint64_t Fq Montgomery limbs (ark_ec TE `Affine`, 64 B);
 *    extended points are (x, y, t, z) = 4 x 4 x uint64_t (ark_ec TE `Projective`, 128 B);
 *  - every call is blocking; buffers are caller-owned HOST memory unless a name says otherwise;
 *  - return value 0 = ok; > 0 = the reference's panic / Err condition; < 0 = CUDA / internal error
 *    (lasso_last_error() gives the text).  There is no CPU fallback: without a CUDA device
 *    lasso_ctx_create fails and nothing else can be called.
 */
#ifndef LASSO_B200_H
#define LASSO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lasso_ctx lasso_ctx;
typedef struct lasso_gens lasso_gens;   /* SparsePolyCommitmentGens<G>        lasso/surge.rs:25-58  */
typedef struct lasso_dense lasso_dense; /* DensifiedRepresentation<F, C>      lasso/densified.rs:8-18 */

/* SubtableStrategy impls (subtables/{and,or,xor,lt,range_check}.rs) */
enum { LASSO_AND = 0, LASSO_OR = 1, LASSO_XOR = 2, LASSO_LT = 3, LASSO_RANGE_CHECK = 4 };

/* error codes > 0 mirror the reference's panics */
enum {
  LASSO_OK = 0,
  LASSO_ERR_LENGTH = 1,      /* assert_eq!(r.len(), log2(s)) surge.rs:131; msm Err(min_len) msm/mod.rs:36-40 */
  LASSO_ERR_NOT_POW2 = 2,    /* DensePolynomial::new on a non power of two  poly/dense_mlpoly.rs:63-66 */
  LASSO_ERR_INDEX_RANGE = 3, /* debug_assert!(memory_address < m)           lasso/densified.rs:46 */
  LASSO_ERR_STRATEGY = 4,    /* unknown / unsupported strategy parameters */
  LASSO_ERR_GENS = 5,        /* generator set too small for the polynomial  poly/commitments.rs:85 */
  LASSO_ERR_MULTISET = 6,    /* assert_eq!(hash_init*hash_write, hash_read*hash_final) memory_checking.rs:689 */
  LASSO_ERR_POINTER = 7,     /* a buffer that must be device memory of the context's GPU is not */
  LASSO_ERR_VALUE = 8        /* a field element that is not a canonical Montgomery residue (< l) */
};

const char* lasso_last_error(void);

/* One context per GPU: owns the device, stream, memory pool and scratch. */
int lasso_ctx_create(lasso_ctx** out, int device_id);
void lasso_ctx_destroy(lasso_ctx* ctx);

/* One proof sharded over `world` ranks of ONE node (one process per GPU, world a power of two <= 8; several ranks
 * may also share a GPU): rank 0 obtains an id with lasso_comm_unique_id, every rank receives it out of band (e.g.
 * torch.distributed broadcast) and calls lasso_ctx_init_comm before any other call.  Afterwards lasso_densify /
 * lasso_commit / lasso_prove are collective: every rank passes the SAME arguments, holds the low-index-bit shard
 * of every polynomial, and receives the same (bit-identical to single-GPU) commitment and proof bytes.
 * Exchanges (DESIGN.md section 6): per sumcheck round every GPU stores its three partial sums into the shared
 * pinned host segment of every process (no collective, no extra launch); the few bulk hand-overs (partial points
 * of a row-MSM, heads of the polynomials, the LZ vector of an opening) are all-gathers written as one kernel of
 * peer-memory stores over NVLink (CUDA IPC), or ncclAllGather under LASSO_B200_XCHG=nccl. */
int lasso_comm_unique_id(uint8_t out[128]);
int lasso_ctx_init_comm(lasso_ctx*, const uint8_t id[128], int rank, int world);
/* Optional host-thread placement for one process per GPU on a multi-socket node (sysfs; returns the NUMA node of the
 * context's GPU, or -1 if the topology is not exposed): the CALLING thread — the one that will call lasso_prove and
 * spin on the round messages — is pinned to a dedicated physical core of that node (a different one for every GPU
 * of the node), the library's helper threads (staging of the index matrix) get the rest of the node.  Call it from
 * the proving thread after the process has created its other threads (they keep their affinity). */
int lasso_ctx_bind_host_threads(lasso_ctx*);

/* ---------------------------------------------------------------- per-loop entry points (host buffers) */

/* DensePolynomial::bound_poly_var_top  poly/dense_mlpoly.rs:209-216.  Z has `len` elements; the first
 * len/2 are overwritten with the bound polynomial. */
int lasso_bind_top(lasso_ctx*, uint64_t* Z, size_t len, const uint64_t r[4]);
/* DensePolynomial::bound_poly_var_bot  poly/dense_mlpoly.rs:218-225 */
int lasso_bind_bot(lasso_ctx*, uint64_t* Z, size_t len, const uint64_t r[4]);
/* EqPolynomial::evals  poly/eq_poly.rs:21-38.  out has 2^ell elements; r[0] binds the MSB. */
int lasso_eq_evals(lasso_ctx*, const uint64_t* r, int ell, uint64_t* out);
/* One round of SumcheckInstanceProof::prove_arbitrary's evaluation loop  subprotocols/sumcheck.rs:179-237
 * with comb_func = S::combine_lookups_eq.  polys = (NUM_MEMORIES+1) arrays of `len` elements, the last
 * one the eq polynomial.  evals_out receives sumcheck_poly_degree()+1 elements (t = 0..deg). */
int lasso_sumcheck_round_arbitrary(lasso_ctx*, int strategy, int C, int log_M, int log_R,
                                   const uint64_t* const* polys, size_t len, uint64_t* evals_out);
/* The step between two rounds of prove_arbitrary as the prover runs it: bind every polynomial's top variable to r
 * (subprotocols/sumcheck.rs:247-253, in place: polys[k][0 .. len/2) are overwritten), then evaluate the next
 * round over the bound polynomials (sumcheck.rs:179-237).  One fused pass for the strategies with a linear g.
 * len >= 4. */
int lasso_sumcheck_bind_round_arbitrary(lasso_ctx*, int strategy, int C, int log_M, int log_R, uint64_t* const* polys,
                                        size_t len, const uint64_t r[4], uint64_t* evals_out);
/* One round of prove_cubic_batched's evaluation loop  subprotocols/sumcheck.rs:49-93:
 * e0e2e3_out[3k..3k+3) = sum_i A_k B_k Ceq at t = 0, 2, 3. */
int lasso_sumcheck_round_cubic(lasso_ctx*, int n_circuits, const uint64_t* const* A, const uint64_t* const* B,
                               const uint64_t* Ceq, size_t len, uint64_t* e0e2e3_out);
/* SubtableStrategy::materialize_subtables  subtables/{and.rs:16-28,or.rs,xor.rs:16-27,lt.rs:16-30,
 * range_check.rs:15-34}.  tables_out[k] has M = 2^log_M elements, k < NUM_SUBTABLES. */
int lasso_materialize_subtables(lasso_ctx*, int strategy, int C, int log_M, int log_R, uint64_t* const* tables_out);
/* SubtableStrategy::to_lookup_polys  subtables/mod.rs:78-92.  nz[d] = lookup indices of dimension d
 * (s entries, `usize` = u64); E_out[k] receives s elements, k < NUM_MEMORIES. */
int lasso_gather_lookup_polys(lasso_ctx*, int strategy, int C, int log_M, int log_R, const uint64_t* const* nz,
                              size_t s, uint64_t* const* E_out);
/* VariableBaseMSM::msm  msm/mod.rs:36-40 (bases: n affine points, scalars: n Fr) -> one extended point,
 * normalised (z = 1).  Same group element as the reference's msm_bigint_wnaf.  After lasso_ctx_init_comm this
 * (and lasso_commit_rows) is collective: each rank passes ITS SHARD of the terms (any split), partial points are
 * all-gathered over NCCL and added, every rank receives the full sum. */
int lasso_msm(lasso_ctx*, const uint64_t* bases_affine, const uint64_t* scalars, size_t n, uint64_t out_xytz[16]);
/* BASELINE config 5 — the same VariableBaseMSM::msm on DEVICE-RESIDENT inputs, as a reusable job: `n` terms, term i
 * uses base i % n_pool (n_pool == n: one base per term; smaller: a pool of distinct points tiled, for benchmarks).
 * lasso_msm_job_run runs the whole MSM (scalars -> canonical integers, bases -> internal form, Pippenger with the
 * reference's window rule, msm/mod.rs:91-164) `iters` times between two CUDA events on the context's stream and
 * returns the average ms and the normalised point; info (may be null) = {window bits c, windows, widest scalar bits,
 * unit size, L, T2, world, 0}.  On a sharded context every rank passes ITS terms and the call is collective.
 * lasso_msm_job_naive evaluates the same sum by per-term double-and-add + a tree sum (an independent cross-check
 * for sizes the CPU oracle cannot reach). */
typedef struct lasso_msm_job lasso_msm_job;
/* The schedule the large MSM would use for n terms whose widest scalar has max_bits bits (no GPU needed): out = {window
 * bits c (the reference's rule, msm/mod.rs:112-116, capped at 17), windows, scalar bits, buckets per window 2^(c-1), unit
 * size, reduction levels, group size of level 0.., zero padded}. */
int lasso_msm_plan_info(size_t n, unsigned max_bits, int out[16]);
int lasso_msm_job_create(lasso_ctx*, const uint64_t* bases_affine, size_t n_pool, const uint64_t* scalars, size_t n,
                         lasso_msm_job** out);
int lasso_msm_job_run(lasso_ctx*, lasso_msm_job*, int iters, double* avg_ms, uint64_t out_xytz[16], int info[8]);
int lasso_msm_job_naive(lasso_ctx*, lasso_msm_job*, uint64_t out_xytz[16]);
void lasso_msm_job_destroy(lasso_msm_job*);
/* DensePolynomial::commit_inner  poly/dense_mlpoly.rs:109-128 (+ Commitments::batch_commit
 * poly/commitments.rs:84-93 with blind = 0): Z viewed as L_size rows of R_size; gens_affine holds the
 * R_size generators followed by h.  out_points = L_size extended points (z = 1). */
int lasso_commit_rows(lasso_ctx*, const uint64_t* gens_affine, const uint64_t* Z, size_t L_size, size_t R_size,
                      uint64_t* out_points);

/* ---------------------------------------------------------------- the whole path, device-resident */

/* Number of generator-stream points SparsePolyCommitmentGens::new(label, c, s, num_memories, log_m)
 * needs (the widest PolyCommitmentGens: n + 2).  lasso/surge.rs:32-58, subprotocols/dot_product.rs:146-149 */
size_t lasso_gens_points_needed(size_t c, size_t s, size_t num_memories, size_t log_m);
/* MultiCommitGens::new's sampling (poly/commitments.rs:22-44): Shake256(label || compressed generator)
 * -> ChaCha20Rng -> G::rand, `count` affine points.  Deterministic; see DESIGN.md on what is unpinned. */
int lasso_sample_generators(const char* label, size_t count, uint64_t* out_affine);
/* SparsePolyCommitmentGens from an explicit generator stream (the parity contract passes generators in):
 * stream[0..n) = G, stream[n] = gens_1.G[0], stream[n+1] = h for each of the three PolyCommitmentGens.
 * Also expands the stream into the fixed-base window table and — on a single-GPU context — the digit-multiples
 * tables of the opening / commitment generators (DESIGN.md section 2: ~14 GB of HBM at 2^20 lookups;
 * LASSO_B200_NO_MULTIPLES=1 disables them, LASSO_B200_TABLE_GB caps the 16-bit one).  Outputs do not depend on it. */
int lasso_gens_create(lasso_ctx*, const uint64_t* stream_affine, size_t n_points, size_t c, size_t s,
                      size_t num_memories, size_t log_m, lasso_gens** out);
void lasso_gens_destroy(lasso_gens*);

/* DensifiedRepresentation::from_lookup_indices  lasso/densified.rs:21-75.
 * indices: n_lookups x C row-major `usize` (the reference's &Vec<[usize; C]>). */
int lasso_densify(lasso_ctx*, const uint64_t* indices, size_t n_lookups, size_t C, size_t log_m, lasso_dense** out);
/* DensifiedRepresentation::from_lookup_indices with the index matrix in DEVICE memory of the context's GPU (e.g. a
 * torch CUDA tensor, or lookups a kernel of the caller wrote): no host narrowing, no upload, the GPU sort at every size.
 *  - entry (k, i), k < n_lookups, i < C, is indices[k * row_stride + i * col_stride] (strides in elements, so
 *    transposed and sliced views need no copy), an UNSIGNED integer of elem_bytes = 4 or 8.  It is compared with m in
 *    its full width: an entry >= m (a signed -1 included) returns LASSO_ERR_INDEX_RANGE, creates no dense and leaves
 *    the context usable;
 *  - the addresses of the first and the last entry must both be device memory of the context's device
 *    (cudaPointerGetAttributes); otherwise (host, pinned, managed or another GPU's memory) LASSO_ERR_POINTER, before
 *    any launch;
 *  - elem_bytes not 4 or 8, and the n_lookups, C, log_m lasso_densify rejects, return LASSO_ERR_STRATEGY;
 *  - stream (a cudaStream_t of the context's device, NULL = the legacy default stream): the matrix is read only after
 *    all work enqueued on `stream` before the call, and work enqueued on `stream` after the call returns is ordered
 *    after those reads (a caching allocator may free or reuse the matrix in stream order).  The call returns once
 *    the range verdict is known; the sort may still run, stream-ordered like lasso_densify's;
 *  - on a sharded context the call is collective like lasso_densify: every rank passes the WHOLE matrix, on its own
 *    GPU, checks all of it (so every rank reaches the same verdict without an exchange), sorts it and keeps its shard;
 *  - lasso_last_timings reports its wall time as the densify time. */
int lasso_densify_device(lasso_ctx*, const void* indices, size_t elem_bytes, size_t n_lookups, size_t C,
                         size_t row_stride, size_t col_stride, size_t log_m, void* stream, lasso_dense** out);
void lasso_dense_destroy(lasso_dense*);
size_t lasso_dense_s(const lasso_dense*);
/* copies of the public fields (densified.rs:8-18) back to the host, for inspection / tests:
 * which = 0 dim_usize (C*s u64), 1 dim (C*s Fr), 2 read (C*s Fr), 3 final (C*m Fr),
 *         4 combined_l_variate_polys (Fr), 5 combined_log_m_variate_polys (Fr).  Returns element count. */
size_t lasso_dense_read(lasso_ctx*, const lasso_dense*, int which, uint64_t* out, size_t cap_elems);

/* DensifiedRepresentation::commit  lasso/densified.rs:77-96 -> SparsePolynomialCommitment serialised with
 * ark-serialize (compressed): Vec<G> l_variate, Vec<G> log_m_variate, s, log_m, m (surge.rs:61-68). */
int lasso_commit(lasso_ctx*, const lasso_dense*, const lasso_gens*, uint8_t* out, size_t cap, size_t* out_len);

/* SparsePolynomialEvaluationProof::<G, C, M, S>::prove  lasso/surge.rs:118-211.
 * r: log2(s) Fr elements.  transcript_label: Transcript::new(label) (b"example" in bench.rs:59);
 * tape_label / tape_seed: RandomTape::new(b"proof") seeded with an explicit scalar (the reference draws it
 * from ark_std::test_rng()).  proof_out receives the ark-serialize (compressed) bytes of the proof struct.
 * challenges_out (optional) receives every Fiat-Shamir challenge in order (4 limbs each).
 * This is lasso_prove_transcript (below) on a transcript and a tape made from the labels and the seed: the same
 * bytes, and the same errors, each returned before any launch.  LASSO_ERR_STRATEGY for the parameters
 * lasso_sumcheck_round_arbitrary rejects and for LT with C > 8: its 2C memories make 4C grand-product circuits,
 * above the 32 that one batched grand product holds.  The per-loop entry points above accept LT up to C = 16.
 * LASSO_ERR_LENGTH for r_len != log2(s), a null label, tape seed or proof_len, or proof_cap too small (*proof_len
 * receives the size the proof needs); LASSO_ERR_GENS for generators built for another (c, s, num_memories, log_m),
 * or of another context unless both are single-GPU contexts of one device (such contexts may share one generator
 * set: its tables are only read); LASSO_ERR_VALUE for a coordinate of r or a tape seed that is not a canonical
 * residue. */
int lasso_prove(lasso_ctx*, int strategy, int log_R, lasso_dense*, const uint64_t* r, size_t r_len,
                const lasso_gens*, const char* transcript_label, const char* tape_label, const uint64_t tape_seed[4],
                uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t* challenges_out,
                size_t challenges_cap, size_t* n_challenges);

/* ---------------------------------------------------------------- caller-defined strategies
 *
 * A SubtableStrategy (subtables/mod.rs:31-93) given as data instead of one of the built-in kinds above:
 *  - C, log_m: the const generics, 1 <= C <= 16, 2 <= log_m <= 24 (log_m may be odd);
 *  - tables[k], k < num_subtables: materialize_subtables() as M = 2^log_m u32 values each (integers below 2^32;
 *    lasso_strategy_create_fr below takes tables of arbitrary field elements);
 *  - mem_to_subtable[i], mem_to_dimension[i], i < num_memories (alpha): memory_to_subtable_index /
 *    memory_to_dimension_index; 1 <= num_subtables <= alpha <= 16 (2 alpha grand-product circuits in one batch);
 *  - program (n_ops instructions of 3 int32 {op, a, b}): combine_lookups in SSA form.  Slots 0..alpha-1 hold the
 *    memory values, instruction j writes slot alpha + j, the last instruction's slot is g.  Operands name earlier
 *    slots; for MULK / ADDK b indexes `constants` (n_constants Fr, 4 Montgomery limbs each).  1 <= n_ops <= 128,
 *    n_constants <= 64, at most 16 intermediate values live at once;
 *  - g_degree: g_poly_degree(), 1..16, at least the program's degree (an input has degree 1, ADD / SUB / ADDK take the
 *    larger operand degree, MUL the sum, MULK its operand's).  It sets the number of evaluation points, so proofs
 *    match a Rust strategy that declares the same value.
 * Any malformed part fails with LASSO_ERR_STRATEGY before a CUDA call.  The tables (u32 and Montgomery form) and the
 * program are uploaded to the context's device once; destroy the strategy before its context.  On a sharded context
 * every rank creates the same strategy (the tables are replicated). */
typedef struct lasso_strategy lasso_strategy;
enum { LASSO_OP_ADD = 0, LASSO_OP_SUB = 1, LASSO_OP_MUL = 2, LASSO_OP_MULK = 3, LASSO_OP_ADDK = 4 };
int lasso_strategy_create(lasso_ctx*, int C, int log_m, int num_subtables, const uint32_t* const* tables,
                          int num_memories, const int* mem_to_subtable, const int* mem_to_dimension,
                          const int32_t* program, int n_ops, const uint64_t* constants, int n_constants,
                          int g_degree, lasso_strategy** out);
/* The same with tables of arbitrary field elements: tables[k] holds M Fr values, 4 Montgomery limbs each (a Rust
 * caller passes materialize_subtables()[k].as_ptr() as it is).  Every other parameter and check as above; an entry that
 * is not a canonical Montgomery residue also fails with LASSO_ERR_STRATEGY before a CUDA call.  When every entry is
 * below 2^32 the strategy is the one lasso_strategy_create makes of those integers.  Otherwise it is full-width: only
 * the Montgomery tables are uploaded, and the lookup values are committed with ceil((w + 2) / 8) signed 8-bit windows,
 * w the bit width of the widest entry.  An entry l - k costs the full width: it is committed as the canonical integer
 * it is, never as -k, since the generators may carry a torsion component. */
int lasso_strategy_create_fr(lasso_ctx*, int C, int log_m, int num_subtables, const uint64_t* const* tables,
                             int num_memories, const int* mem_to_subtable, const int* mem_to_dimension,
                             const int32_t* program, int n_ops, const uint64_t* constants, int n_constants,
                             int g_degree, lasso_strategy** out);
void lasso_strategy_destroy(lasso_strategy*);
/* lasso_sumcheck_round_arbitrary for a custom strategy: polys = num_memories + 1 arrays of `len` elements (the last
 * one eq); evals_out receives g_degree + 2 elements. */
int lasso_sumcheck_round_custom(lasso_ctx*, const lasso_strategy*, const uint64_t* const* polys, size_t len,
                                uint64_t* evals_out);
/* lasso_prove with a custom strategy: the same semantics, outputs, errors and collectiveness.  LASSO_ERR_STRATEGY
 * for a null strategy, one of another context, or one whose (C, log_m) differ from the densified representation's. */
int lasso_prove_custom(lasso_ctx*, const lasso_strategy*, lasso_dense*, const uint64_t* r, size_t r_len,
                       const lasso_gens*, const char* transcript_label, const char* tape_label,
                       const uint64_t tape_seed[4], uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                       uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges);

/* ---------------------------------------------------------------- transcripts and dense polynomials
 *
 * For a caller that composes Lasso into a larger protocol: its own multilinear polynomials committed and opened on the
 * GPU, bound by one Fiat-Shamir transcript the caller holds across calls.
 *
 * ProofTranscript (utils/transcript.rs:6-72) over merlin, and RandomTape (utils/random.rs:9-39).  Host objects: they
 * need no context and no GPU.  Labels are NUL-terminated; scalars are 4 Montgomery limbs and must be canonical
 * residues (LASSO_ERR_VALUE otherwise); points are 32-byte ark-serialize compressed encodings, absorbed as given.
 * append_scalars / append_points frame the vector with the begin/end markers of the reference. */
typedef struct lasso_transcript lasso_transcript;
typedef struct lasso_random_tape lasso_random_tape;
int lasso_transcript_create(const char* label, lasso_transcript** out); /* Transcript::new(label) */
void lasso_transcript_destroy(lasso_transcript*);
int lasso_transcript_append_message(lasso_transcript*, const char* label, const uint8_t* msg, size_t len);
int lasso_transcript_append_u64(lasso_transcript*, const char* label, uint64_t x);
int lasso_transcript_append_protocol_name(lasso_transcript*, const char* name);
int lasso_transcript_append_scalar(lasso_transcript*, const char* label, const uint64_t s[4]);
int lasso_transcript_append_scalars(lasso_transcript*, const char* label, const uint64_t* s, size_t n);
int lasso_transcript_append_point(lasso_transcript*, const char* label, const uint8_t point[32]);
int lasso_transcript_append_points(lasso_transcript*, const char* label, const uint8_t* points, size_t n);
/* PolyCommitment::append_to_transcript (poly/dense_mlpoly.rs:281-289) of serialised commitment bytes (lasso_poly_commit's
 * output: a u64 count, then 32 bytes per point); LASSO_ERR_LENGTH when len != 8 + 32 * count */
int lasso_transcript_append_poly_commitment(lasso_transcript*, const char* label, const uint8_t* bytes, size_t len);
int lasso_transcript_challenge_scalar(lasso_transcript*, const char* label, uint64_t out[4]);
int lasso_transcript_challenge_vector(lasso_transcript*, const char* label, size_t n, uint64_t* out);
/* RandomTape::new(label) seeded with an explicit scalar, as lasso_prove's tape is */
int lasso_random_tape_create(const char* label, const uint64_t seed[4], lasso_random_tape** out);
void lasso_random_tape_destroy(lasso_random_tape*);
int lasso_random_tape_random_scalar(lasso_random_tape*, const char* label, uint64_t out[4]);
int lasso_random_tape_random_vector(lasso_random_tape*, const char* label, size_t n, uint64_t* out);

/* PolyCommitmentGens (poly/dense_mlpoly.rs:31-45) from an explicit generator stream: with R = 2^(num_vars - num_vars/2),
 * G_0..G_{R-1} = stream[0..R), Q = stream[R], h = stream[R+1] (poly/commitments.rs:21-44, dot_product.rs:146-149).
 * Its own type: it cannot be passed to lasso_commit or lasso_prove.  Builds the same device tables a lasso_gens of the
 * same R builds (window table, digit-multiples tables; LASSO_B200_NO_MULTIPLES and LASSO_B200_TABLE_GB apply): about
 * 14 GB of HBM at R = 2^12.  LASSO_ERR_GENS when n_points < R + 2, LASSO_ERR_LENGTH when num_vars > 28.
 *
 * Sharded contexts (lasso_ctx_init_comm over G ranks): the lasso_poly_* calls below, lasso_poly_gens_create and
 * lasso_combined_eval_prove are COLLECTIVE, like lasso_commit and lasso_prove: every rank calls them in the same order
 * with the same arguments (the same kind of pointer too: host or device), device inputs on its own GPU, transcripts and
 * tapes in the same state.  Every rank returns the same bytes, values and error code, and its handles end in the same
 * state; the outputs are those of a single-GPU context, byte for byte.  A polynomial is held as its low-bit shard (rank
 * g holds evaluations i * G + g: the R/G columns congruent to g of every row), so on G ranks a polynomial, or the
 * generators, of num_vars variables needs R = 2^(num_vars - num_vars/2) >= G, i.e. num_vars >= 2 log2(G) - 1:
 * otherwise LASSO_ERR_LENGTH before any launch (lasso_poly_gens_create, lasso_poly_create[_device], lasso_poly_create_eq,
 * lasso_poly_create_comb).  Commitments make one all-gather of the row partials; evaluations add the ranks' partial
 * values in one message to every process; openings gather L.Z and run the Bulletproofs rounds replicated.
 * lasso_sumcheck_prove_cubic_batched is collective too.  lasso_sumcheck_prove, lasso_gp_circuit_create, lasso_gp_prove,
 * lasso_dense_outputs[_custom] and the memory-checking calls (lasso_lookup_polys[_custom], lasso_dense_poly,
 * lasso_memory_check_prove[_custom], lasso_memory_fingerprints) are not available on a sharded context: they return
 * LASSO_ERR_STRATEGY before any work. */
typedef struct lasso_poly_gens lasso_poly_gens;
typedef struct lasso_poly lasso_poly;
size_t lasso_poly_gens_points_needed(size_t num_vars); /* R + 2 */
int lasso_poly_gens_create(lasso_ctx*, const uint64_t* stream_affine, size_t n_points, size_t num_vars,
                           lasso_poly_gens** out);
void lasso_poly_gens_destroy(lasso_poly_gens*);
/* DensePolynomial::new (poly/dense_mlpoly.rs:62-71): a device-resident copy of `len` evaluations, 4 Montgomery limbs
 * each.  len must be a power of two (LASSO_ERR_NOT_POW2, 0 included) and at most 2^28 (LASSO_ERR_LENGTH).  Every
 * evaluation must be a canonical residue: otherwise LASSO_ERR_VALUE, found by the ingest pass on the device (the one
 * error reported after a launch; no polynomial is made and the context stays usable).  A polynomial whose values are
 * all integers below 2^32 is committed and opened through the 16-bit digit tables, a wider one with ceil((w + 2) / 8)
 * signed 8-bit windows, w the bit width of its widest value; both give the same bytes.
 * lasso_poly_create reads host memory (len x 4 u64, contiguous).  lasso_poly_create_device reads DEVICE memory of the
 * context's GPU: row i at Z + i * row_stride (row_stride in u64, >= 4, else LASSO_ERR_LENGTH), limbs contiguous.  The
 * first and the last row must be device memory of the context's device, otherwise LASSO_ERR_POINTER before any launch;
 * the rows are read after the work enqueued on `stream` (NULL = the legacy default stream) before the call, and later
 * work on `stream` is ordered after those reads.  The library keeps its own copy: the caller may free Z on return.
 * On a sharded context every rank passes the WHOLE polynomial, as lasso_densify takes the whole index matrix, and reads
 * only its rows i * G + g (host rows are staged and uploaded by each rank, 1/G of the PCIe bytes); the ranks agree on the
 * verdict and on the widest value in one exchange, so a non-canonical evaluation in any rank's rows gives
 * LASSO_ERR_VALUE on every rank, and the context stays usable for the next collective call. */
int lasso_poly_create(lasso_ctx*, const uint64_t* Z, size_t len, lasso_poly** out);
int lasso_poly_create_device(lasso_ctx*, const uint64_t* Z, size_t len, size_t row_stride, void* stream,
                             lasso_poly** out);
size_t lasso_poly_num_vars(const lasso_poly*);
void lasso_poly_destroy(lasso_poly*);
/* DensePolynomial::commit (poly/dense_mlpoly.rs:152-181) without blinds (with them: lasso_poly_commit_hiding) ->
 * PolyCommitment { C: Vec<G> } serialised with ark-serialize (compressed): a u64 count L = 2^(num_vars/2), then 32
 * bytes per row.  *out_len receives the size
 * (also when cap is too small: LASSO_ERR_LENGTH).  LASSO_ERR_GENS when the generators' R differs from the
 * polynomial's (poly/commitments.rs:85). */
int lasso_poly_commit(lasso_ctx*, const lasso_poly*, const lasso_poly_gens*, uint8_t* out, size_t cap, size_t* out_len);
/* DensePolynomial::evaluate (poly/dense_mlpoly.rs:229-235): Z(r), r_len == num_vars (LASSO_ERR_LENGTH otherwise) */
int lasso_poly_evaluate(lasso_ctx*, const lasso_poly*, const uint64_t* r, size_t r_len, uint64_t out[4]);
/* PolyEvalProof::prove (poly/dense_mlpoly.rs:301-359) without blinds: proof_out receives the ark-serialize (compressed)
 * PolyEvalProof, C_Zr_out (may be null) the compressed C_Zr_prime returned alongside it.  The transcript and the tape
 * are advanced in place, so later calls continue them.  Errors as lasso_poly_commit and lasso_poly_evaluate. */
int lasso_poly_eval_prove(lasso_ctx*, const lasso_poly*, const lasso_poly_gens*, const uint64_t* r, size_t r_len,
                          const uint64_t Zr[4], lasso_transcript* transcript, lasso_random_tape* random_tape,
                          uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint8_t C_Zr_out[32]);
/* Hiding commitments and openings (collective on a sharded context, like every lasso_poly_* call: every rank draws the
 * same blinds from its tape and returns the same bytes).
 * lasso_poly_commit_hiding is DensePolynomial::commit(gens, Some(random_tape)) (poly/dense_mlpoly.rs:152-181): it draws
 * L = 2^(num_vars/2) blinds from the tape as random_vector("poly_blinds", L), writes the hiding PolyCommitment (row i is
 * <row_i, G> + blinds[i] * h; same format and size as lasso_poly_commit) to out and the L blinds (L x 4 Montgomery limbs)
 * to blinds_out, which has room for blinds_cap of them.
 * lasso_poly_eval_prove_hiding is PolyEvalProof::prove(poly, blinds_opt, r, Zr, blind_Zr_opt, ...)
 * (poly/dense_mlpoly.rs:301-359): blinds (n_blinds == L, the commitment's blinds) or None (n_blinds == 0); blind_Zr
 * or None (NULL).  Same proof size as lasso_poly_eval_prove; C_Zr_out (may be null) is Zr * Q + blind_Zr * h.  With no
 * blinds and no blind_Zr it is lasso_poly_eval_prove, byte for byte.
 * Both check everything before any launch and before the tape or the transcript moves: LASSO_ERR_LENGTH for out / cap
 * or blinds_out / blinds_cap too small (*out_len / *proof_len receive the size needed), a null tape or transcript, or
 * n_blinds other than 0 or L; LASSO_ERR_VALUE for a blind, blind_Zr, Zr or coordinate of r that is not a canonical
 * residue; LASSO_ERR_GENS and LASSO_ERR_STRATEGY as lasso_poly_commit / lasso_poly_eval_prove. */
int lasso_poly_commit_hiding(lasso_ctx*, const lasso_poly*, const lasso_poly_gens*, lasso_random_tape*,
                             uint8_t* out, size_t cap, size_t* out_len, uint64_t* blinds_out, size_t blinds_cap);
int lasso_poly_eval_prove_hiding(lasso_ctx*, const lasso_poly*, const lasso_poly_gens*, const uint64_t* blinds,
                                 size_t n_blinds, const uint64_t* r, size_t r_len, const uint64_t Zr[4],
                                 const uint64_t blind_Zr[4], lasso_transcript*, lasso_random_tape*, uint8_t* proof_out,
                                 size_t proof_cap, size_t* proof_len, uint8_t C_Zr_out[32]);
/* EqPolynomial::new(r).evals() (poly/eq_poly.rs:21-38) as a polynomial of the context, r[0] the most significant
 * variable: 2^r_len evaluations, r_len <= 28 (LASSO_ERR_LENGTH), each coordinate a canonical residue (LASSO_ERR_VALUE). */
int lasso_poly_create_eq(lasso_ctx*, const uint64_t* r, size_t r_len, lasso_poly** out);

/* ---------------------------------------------------------------- deriving polynomials and reading them back
 *
 * None of these calls modifies its input.  Each result is a new polynomial with storage of its own (a grand-product
 * circuit may hold the input as its layer 0), to be destroyed with lasso_poly_destroy.  Collective on a sharded context
 * like every lasso_poly_* call: every rank passes the same arguments and gets the single-GPU result.  Every error is
 * returned before any launch, exchange or allocation: LASSO_ERR_LENGTH for a null pointer, k outside 1..num_vars, a
 * result that a sharded context cannot hold (2^(nv - nv/2) >= G for the result's nv), cap too small, or more than 2^28
 * evaluations after padding; LASSO_ERR_VALUE for a coordinate of r or an evaluation that is not a canonical residue
 * (an evaluation is found by the ingest pass, as in lasso_poly_create); LASSO_ERR_STRATEGY for a polynomial of another
 * context; LASSO_ERR_POINTER for device memory of another GPU.
 *
 * lasso_poly_bind_top: k calls of DensePolynomial::bound_poly_var_top (poly/dense_mlpoly.rs:209-216), r[0] first:
 * P(r_0, .., r_{k-1}, x), num_vars - k variables.  Up to 8 variables per pass over the data (the first pass reads the
 * 4-byte integer form of a polynomial whose values are below 2^32), so a sumcheck stopped after k rounds continues on
 * the result without a host round trip.
 * lasso_poly_bind_bot: k calls of bound_poly_var_bot (:218-225) in the order given, r[0] binding the lowest variable:
 * P(x, r_{k-1}, .., r_0).  The reference's own callers pass their challenges last first (subtables/mod.rs:256): to get
 * their result, pass r reversed.
 * Both results are full width: committed through the Fr windows, like lasso_poly_create_eq.
 * lasso_poly_split: split(idx) (:101-107): lo = Z[0..idx), hi = Z[idx..2 idx); idx a power of two with 2 idx <= len.
 * Both keep the parent's width (the 16-bit commitment path when its values are below 2^32).
 * lasso_poly_create_padded[_device]: DensePolynomial::new_padded (:75-87): len evaluations of any length (the forms and
 * rules of lasso_poly_create / lasso_poly_create_device), zero-padded up to the next power of two.  As in the
 * reference, whose utils::is_power_of_two(0) is false, len = 0 gives the polynomial of one zero evaluation (num_vars 0).
 * lasso_poly_read: the 2^num_vars evaluations in natural order, 4 Montgomery limbs each (the layout lasso_poly_create
 * takes), into out, which has room for cap of them.  lasso_poly_read_device writes them into DEVICE memory of the
 * context's GPU, row i at dst + i * row_stride (row_stride in u64, >= 4), as a copy on `stream` (NULL = the legacy
 * default stream) ordered after the library's work on the polynomial.  Sharded: every rank receives the whole
 * polynomial. */
int lasso_poly_bind_top(lasso_ctx*, const lasso_poly*, const uint64_t* r, size_t k, lasso_poly** out);
int lasso_poly_bind_bot(lasso_ctx*, const lasso_poly*, const uint64_t* r, size_t k, lasso_poly** out);
int lasso_poly_split(lasso_ctx*, const lasso_poly*, size_t idx, lasso_poly** lo_out, lasso_poly** hi_out);
int lasso_poly_create_padded(lasso_ctx*, const uint64_t* Z, size_t len, lasso_poly** out);
int lasso_poly_create_padded_device(lasso_ctx*, const uint64_t* Z, size_t len, size_t row_stride, void* stream,
                                    lasso_poly** out);
int lasso_poly_read(lasso_ctx*, const lasso_poly*, uint64_t* out, size_t cap);
int lasso_poly_read_device(lasso_ctx*, const lasso_poly*, uint64_t* dst, size_t row_stride, void* stream);

/* ---------------------------------------------------------------- lookups inside a caller's protocol
 *
 * SparsePolynomialEvaluationProof::prove (lasso/surge.rs:118-211) on the caller's transcript and tape, both advanced in
 * place: the reference's signature prove(dense, r, gens, transcript, random_tape) one to one.  lasso_prove is this call on
 * Transcript::new(transcript_label) and a fresh tape, with the same bytes.  proof_out receives the ark-serialize
 * (compressed) proof, whose size is fixed by the strategy, s, log_m and the generators (*proof_len receives it, also when
 * proof_cap is too small); claimed_eval_out (may be NULL) PrimarySumcheck::claimed_evaluation, the sum over k of
 * eq(r, k) combine_lookups(E_0(k), ..).  Collective on a sharded context like lasso_prove: every rank passes its own
 * transcript and tape in the same state, and every rank's handles end in the same state.
 * Errors, each returned before any launch and before the transcript or the tape is touched: LASSO_ERR_STRATEGY for
 * the strategies lasso_prove / lasso_prove_custom reject (LT with C > 8 included), a strategy of another context, or
 * (C, log_m) that differ from the dense's; LASSO_ERR_LENGTH for r_len != log2(s), proof_cap too small, or a null
 * transcript, tape or proof_len; LASSO_ERR_GENS for generators of another context or built for another
 * (c, s, num_memories, log_m); LASSO_ERR_VALUE for a coordinate of r that is not a canonical residue.  The proof's
 * working memory is reserved in the context's pool before the first transcript write.  LASSO_ERR_MULTISET, as the
 * reference's panic, can only be raised after the transcript and the tape have moved. */
int lasso_prove_transcript(lasso_ctx*, int strategy, int log_R, lasso_dense*, const uint64_t* r, size_t r_len,
                           const lasso_gens*, lasso_transcript* transcript, lasso_random_tape* random_tape,
                           uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t claimed_eval_out[4]);
int lasso_prove_custom_transcript(lasso_ctx*, const lasso_strategy*, lasso_dense*, const uint64_t* r, size_t r_len,
                                  const lasso_gens*, lasso_transcript* transcript, lasso_random_tape* random_tape,
                                  uint8_t* proof_out, size_t proof_cap, size_t* proof_len, uint64_t claimed_eval_out[4]);
/* SparsePolynomialCommitment::append_to_transcript (lasso/surge.rs:70-82) of lasso_commit's output bytes: both
 * PolyCommitments with their begin / end markers, then s, log_m and m as u64.  Host only: no context.  LASSO_ERR_LENGTH
 * when the bytes do not parse as that struct (a count beyond the bytes, missing or trailing bytes); LASSO_ERR_VALUE for a
 * point that does not decompress; nothing is absorbed in either case. */
int lasso_transcript_append_sparse_commitment(lasso_transcript*, const uint8_t* bytes, size_t len);
/* The lookup outputs v[k] = combine_lookups(T_sub(0)[dim_usize(0)[k]], ..) for k < s, padded lookups included (their
 * indices are 0, densified.rs:37), as a polynomial of log2(s) variables.  Its MLE at r is the claimed evaluation of a
 * proof at r, so a caller can commit to v (lasso_poly_commit) and open it at r (lasso_poly_eval_prove) to tie the proof
 * to its own commitments.  One pass over the indices on the GPU; built-in entries are computed from the index, custom
 * ones read from the strategy's tables.  When every value is below 2^32, v has the u32 mirror (the 16-bit commitment
 * path).  LASSO_ERR_STRATEGY for the strategies lasso_prove rejects, a strategy of another context or other (C, log_m),
 * and on a sharded context; LASSO_ERR_LENGTH for a null output. */
int lasso_dense_outputs(lasso_ctx*, int strategy, int log_R, const lasso_dense*, lasso_poly** out);
int lasso_dense_outputs_custom(lasso_ctx*, const lasso_strategy*, const lasso_dense*, lasso_poly** out);

/* ---------------------------------------------------------------- memory checking inside a caller's protocol
 *
 * The pieces of SparsePolynomialEvaluationProof::prove (lasso/surge.rs:119-211) around the primary sumcheck, so that a
 * caller can run its own sumcheck over the lookup polynomials and still prove the memory check, and offline memory
 * checking of a caller's own memory (Spark's eq(r_x) table read at addresses dim, say).  Single GPU only: on a sharded
 * context each call returns LASSO_ERR_STRATEGY before any work.
 *
 * lasso_lookup_polys[_custom]: Subtables::new's lookup_polys (subtables/mod.rs:116-129), E_i[j] = T_sub(i)[dim_i[j]] for
 * the alpha = num_memories memories in memory order, each a new polynomial of log2(s) variables with storage of its own.
 * Their width is the strategy's table width, with the u32 mirror when that is <= 32, so that
 * lasso_poly_create_merge(E) committed with the proof's derefs generators gives the proof's comm_derefs.  One table
 * materialisation (built-in strategies) and one gather.  LASSO_ERR_STRATEGY as lasso_dense_outputs; LASSO_ERR_LENGTH
 * for a null out or n_out != alpha. */
int lasso_lookup_polys(lasso_ctx*, int strategy, int log_R, const lasso_dense*, lasso_poly** out, size_t n_out);
int lasso_lookup_polys_custom(lasso_ctx*, const lasso_strategy*, const lasso_dense*, lasso_poly** out, size_t n_out);
/* DensifiedRepresentation's dim_j, read_j or final_j (lasso/densified.rs:8-18) as a new polynomial: which takes
 * lasso_dense_read's numbers (1 = dim, 2 = read, 3 = final), j < C (LASSO_ERR_LENGTH otherwise).  s evaluations (m for
 * final), all integers, with the u32 mirror.  LASSO_ERR_STRATEGY for a null dense or a sharded context. */
int lasso_dense_poly(lasso_ctx*, const lasso_dense*, int which, size_t j, lasso_poly** out);
/* MemoryCheckingProof::prove (subtables/memory_checking.rs:56-83) at (gamma, tau) on the caller's transcript and tape,
 * both advanced in place.  The reference's `subtables` argument is rebuilt from (strategy, dense): identical by
 * construction, at the cost of one gather.  proof_out receives the ark-serialize (compressed) MemoryCheckingProof, the
 * product layer then the hash layer, 4*32*alpha + gpa(2 alpha, log m) + gpa(2 alpha, log s) + 32 (3C + alpha) + three
 * PolyEvalProofs at the generators' (nv_l, nv_m, nv_d); *proof_len receives that size, also when proof_cap is too small.
 * Inside lasso_prove_transcript this is what follows challenge_vector("challenge_r_hash", 2) = (gamma, tau).
 * Errors, each before any launch and before the transcript or the tape moves: LASSO_ERR_STRATEGY as lasso_prove;
 * LASSO_ERR_LENGTH for a null transcript, tape, gamma, tau or proof_len, or proof_cap too small; LASSO_ERR_GENS for
 * generators of another context or shape; LASSO_ERR_VALUE for a gamma or tau that is not a canonical residue.  The
 * working memory is reserved in the context's pool before the first transcript write.  LASSO_ERR_MULTISET, as the
 * reference's panic, can only be raised after the transcript has moved. */
int lasso_memory_check_prove(lasso_ctx*, int strategy, int log_R, const lasso_dense*, const uint64_t gamma[4],
                             const uint64_t tau[4], const lasso_gens*, lasso_transcript* transcript,
                             lasso_random_tape* random_tape, uint8_t* proof_out, size_t proof_cap, size_t* proof_len);
int lasso_memory_check_prove_custom(lasso_ctx*, const lasso_strategy*, const lasso_dense*, const uint64_t gamma[4],
                                    const uint64_t tau[4], const lasso_gens*, lasso_transcript* transcript,
                                    lasso_random_tape* random_tape, uint8_t* proof_out, size_t proof_cap,
                                    size_t* proof_len);
/* GrandProducts::new(eval_table, dim, dim_usize, read, final, (gamma, tau)) (subtables/memory_checking.rs:175-310)
 * over a caller's memory, with dim doubling as dim_usize as in every reference caller: out receives four new
 * full-width polynomials in the reference's field order, with hash(a, v, t) = t gamma^2 + v gamma + a - tau:
 *   init[i] = hash(i, T[i], 0), final[i] = hash(i, T[i], final_ts[i])                    for i < M = table's length,
 *   read[j] = hash(dim[j], T[dim[j]], read[j]), write[j] = hash(dim[j], T[dim[j]], read[j] + 1)   for j < s.
 * read and write come from one pass that gathers T[dim[j]] (never stored); read and final_ts may be any field elements.
 * Errors, each before any launch: LASSO_ERR_LENGTH when table and final_ts are not of one length M >= 2, dim and read
 * not of one length s >= 2, or gamma, tau or out is null; LASSO_ERR_INDEX_RANGE when dim does not hold integers below M
 * (its bit width, known without a device pass, exceeds log2 M); LASSO_ERR_VALUE for a gamma or tau that is not a
 * canonical residue; LASSO_ERR_STRATEGY for a polynomial of another context or a sharded context.  Grand-product circuits
 * over the results (lasso_gp_circuit_create) give the reference's GrandProducts. */
int lasso_memory_fingerprints(lasso_ctx*, const lasso_poly* table, const lasso_poly* dim, const lasso_poly* read,
                              const lasso_poly* final_ts, const uint64_t gamma[4], const uint64_t tau[4],
                              lasso_poly* out[4]);
/* CombinedTableCommitment::append_to_transcript (subtables/mod.rs:382-393) of PolyCommitment bytes (lasso_poly_commit's
 * format): the begin / end subtable_evals_commitment messages around PolyCommitment::append_to_transcript under label.
 * Host only.  LASSO_ERR_LENGTH for a null label or bytes that do not parse; LASSO_ERR_VALUE for a point that does not
 * decompress; nothing is absorbed in either case. */
int lasso_transcript_append_combined_table_commitment(lasso_transcript*, const char* label, const uint8_t* bytes,
                                                      size_t len);

/* ---------------------------------------------------------------- many polynomials per call
 *
 * DensePolynomial::merge (poly/dense_mlpoly.rs:251-261): a new polynomial holding the evaluations of polys[0..n_polys) one
 * after another, zero-padded to the next power of two.  Inputs may have different num_vars and may repeat; they are not
 * modified, and the result owns its own copy, so they may be destroyed afterwards.  It has a u32 mirror (is committed and
 * opened through the 16-bit tables) iff every input has one, i.e. iff every value is an integer below 2^32.  Copies only:
 * no kernel is launched.  Errors, before any copy: LASSO_ERR_LENGTH for n_polys == 0, a null array or output, or more
 * than 2^28 evaluations after padding; LASSO_ERR_STRATEGY for a polynomial of another context.  Sharded: every input's
 * length is a multiple of G, so each rank concatenates its shards of the inputs, with no exchange. */
int lasso_poly_create_merge(lasso_ctx*, const lasso_poly* const* polys, size_t n_polys, lasso_poly** out);
/* DensePolynomial::evaluate (poly/dense_mlpoly.rs:229-235) of n_polys polynomials of one num_vars at one point r: out
 * receives n_polys x 4 limbs, P_j(r) at out + 4 j.  One eq table serves every polynomial, and the dot kernel reads each of
 * its elements once per group of 8 inputs.  1 <= n_polys <= 64: the inputs travel as one kernel parameter of 64 pointers,
 * and the per-input block partials of one launch fill at most 8 x 528 elements of the context's scratch.  Integer and
 * full-width polynomials may be mixed.  Errors, before any launch: LASSO_ERR_LENGTH for different num_vars,
 * r_len != num_vars, n_polys outside 1..64, or a null array or output; LASSO_ERR_VALUE for a non-canonical coordinate;
 * LASSO_ERR_STRATEGY for a polynomial of another context.  Collective on a sharded context. */
int lasso_poly_evaluate_batch(lasso_ctx*, const lasso_poly* const* polys, size_t n_polys, const uint64_t* r, size_t r_len,
                              uint64_t* out);
/* CombinedTableEvalProof::prove (subtables/mod.rs:229-313) without blinds: opens the merged polynomial `combined` at r for
 * the n_evals claims `evals` with ONE PolyEvalProof.  The protocol name "Lasso CombinedTableEvalProof" is appended, evals
 * are zero-padded to a power of two and appended as "evals_ops_val", log2 of that many challenges are drawn
 * ("challenge_combine_n_to_one"), the padded evals are folded with them (bound_poly_var_bot, last challenge first) into
 * "joint_claim_eval", and the polynomial is opened at (challenges || r).  proof_out receives the ark-serialize
 * (compressed) CombinedTableEvalProof, which is its PolyEvalProof alone: the size lasso_poly_eval_prove gives at
 * combined's num_vars (*proof_len receives it, also when proof_cap is too small).  The transcript and the tape advance in
 * place.
 * As in the reference, evals are the caller's claims and are not checked: a wrong one gives a proof the verifier rejects.
 * For combined = lasso_poly_create_merge(P_0..P_{k-1}) the claim evals[i] = P_i(r) is about block i of combined only when
 * every P_i has num_vars == r_len (equal sizes); with unequal sizes block i is not component i.
 * Errors, each returned before any launch and before the transcript or the tape is touched: LASSO_ERR_LENGTH for
 * num_vars != r_len + log2(next_pow2(n_evals)), n_evals == 0, a too small proof_cap, or a null transcript, tape, evals or
 * output; LASSO_ERR_GENS for generators whose R differs from the polynomial's; LASSO_ERR_VALUE for a non-canonical eval or
 * coordinate; LASSO_ERR_STRATEGY for another context.  The opening's working memory is reserved in the context's memory
 * pool before the first transcript write.  Collective on a sharded context. */
int lasso_combined_eval_prove(lasso_ctx*, const lasso_poly* combined, const lasso_poly_gens*, const uint64_t* evals,
                              size_t n_evals, const uint64_t* r, size_t r_len, lasso_transcript*, lasso_random_tape*,
                              uint8_t* proof_out, size_t proof_cap, size_t* proof_len);

/* ---------------------------------------------------------------- sumchecks over a caller's polynomials
 *
 * A combining function g(x_0..x_{n_inputs-1}) in the program format of lasso_strategy_create (slots 0..n_inputs-1 are
 * the inputs, instruction j writes slot n_inputs + j, the last instruction's slot is g), its constants, and the declared
 * combined_degree.  The rules of lasso_strategy_create apply: 1 <= n_inputs <= 16, 1 <= n_ops <= 128, at most 64
 * constants, each a canonical residue, operands name earlier slots, at most 16 intermediate values live at once,
 * 1 <= degree <= 16 and at least the program's degree; LASSO_ERR_STRATEGY otherwise.  A host object: it needs no context
 * and no GPU. */
typedef struct lasso_comb lasso_comb;
int lasso_comb_create(int n_inputs, const int32_t* program, int n_ops, const uint64_t* constants, int n_constants,
                      int degree, lasso_comb** out);
void lasso_comb_destroy(lasso_comb*);
/* SumcheckInstanceProof::prove_arbitrary (subprotocols/sumcheck.rs:149-260): num_rounds rounds of the sumcheck of
 * sum_x g(polys[0](x), .., polys[n_polys-1](x)) on the caller's transcript, which is advanced in place.  The caller's
 * polynomials are NOT modified (the reference binds them in place): they can be opened at r afterwards.  The same
 * polynomial may appear several times.
 *  - proof_out: the ark-serialize bytes of SumcheckInstanceProof, 8 + num_rounds * (8 + 32 * degree) bytes (*proof_len
 *    receives the size, also when proof_cap is too small);
 *  - r_out: the num_rounds challenges; final_evals_out: n_polys values, element 0 of each polynomial after the binds
 *    (its evaluation at r when num_rounds == num_vars);
 *  - claim_out (may be NULL): e_0 + e_1 of the first round, i.e. the sum over the hypercube.
 * Errors, each returned before any launch and before the transcript is touched: LASSO_ERR_STRATEGY for n_polys !=
 * n_inputs, a polynomial of another context or a sharded context; LASSO_ERR_LENGTH for polynomials of different
 * num_vars, num_rounds outside 1..num_vars, proof_cap too small, or a null transcript or output.  The working memory
 * (n_polys x 2^(num_vars-1) elements when num_rounds >= 2) is allocated before the first transcript write. */
int lasso_sumcheck_prove(lasso_ctx*, const lasso_comb*, const lasso_poly* const* polys, size_t n_polys,
                         size_t num_rounds, lasso_transcript*, uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
                         uint64_t* r_out, uint64_t* final_evals_out, uint64_t claim_out[4]);
/* SumcheckInstanceProof::prove_cubic_batched (subprotocols/sumcheck.rs:26-135): num_rounds rounds of the sumcheck of
 * claim = sum_x C(x) * sum_k coeffs[k] * A[k](x) * B[k](x) over 1 <= n <= 32 pairs, top variable first, on the
 * caller's transcript, which is advanced in place.  Round j appends the cubic through [e0, e - e0, e2, e3], e starting
 * at the caller's claim, which is not checked (as in the reference: a wrong claim gives a proof the verifier rejects).
 * The caller's polynomials are NOT modified, and the same polynomial may appear several times (A[k] == B[j], A[k] == C).
 * Any canonical coefficients are accepted, zero included.
 *  - proof_out: the ark-serialize bytes of SumcheckInstanceProof, 8 + 104 * num_rounds bytes (*proof_len receives the
 *    size, also when proof_cap is too small);
 *  - r_out: the num_rounds challenges;
 *  - claims_A_out, claims_B_out (n values each) and claim_C_out: element 0 of every polynomial after the binds, i.e. its
 *    evaluation at (r || 0..0), and at r when num_rounds == num_vars.
 * Errors, each returned before any launch and before the transcript is touched: LASSO_ERR_STRATEGY for n outside 1..32
 * or a polynomial of another context; LASSO_ERR_LENGTH for polynomials of different num_vars, num_rounds outside
 * 1..num_vars, proof_cap too small, or a null transcript, input or output; LASSO_ERR_VALUE for a non-canonical
 * coefficient or claim.  The working memory ((2 n + 1) x 2^(num_vars-1) elements at most) is allocated before the first
 * transcript write.  Collective on a sharded context: every rank sums its shards, the ranks add their round sums, the
 * last rounds run replicated on every rank, and every rank returns the bytes, r and values of a single-GPU context. */
int lasso_sumcheck_prove_cubic_batched(lasso_ctx*, const lasso_poly* const* A, const lasso_poly* const* B, size_t n,
                                       const lasso_poly* C, const uint64_t* coeffs, const uint64_t claim[4],
                                       size_t num_rounds, lasso_transcript*, uint8_t* proof_out, size_t proof_cap,
                                       size_t* proof_len, uint64_t* r_out, uint64_t* claims_A_out,
                                       uint64_t* claims_B_out, uint64_t claim_C_out[4]);
/* Q(x) = g(polys[0](x), .., polys[n_polys-1](x)) at every point of the hypercube, e.g. the fingerprints
 * h(a, v, t) = t gamma^2 + v gamma + a - tau of offline memory checking (lasso/memory_checking.rs:251-252).  g's
 * declared degree is not used.  The result is a full-width polynomial like lasso_poly_create_eq (committed through the
 * Fr windows): it can be committed, evaluated, opened, summed over or made a grand-product circuit.  Errors, before any
 * launch: LASSO_ERR_STRATEGY for n_polys != n_inputs or a polynomial of another context; LASSO_ERR_LENGTH for
 * polynomials of different num_vars or a null output.  Collective on a sharded context: element-wise, each rank maps its
 * own shards, with no exchange. */
int lasso_poly_create_comb(lasso_ctx*, const lasso_comb*, const lasso_poly* const* polys, size_t n_polys,
                           lasso_poly** out);

/* ---------------------------------------------------------------- zero-knowledge sumchecks
 *
 * The hiding form of lasso_sumcheck_prove, so that a caller's Spartan-style protocol over hiding commitments and
 * openings (lasso_poly_commit_hiding, lasso_poly_eval_prove_hiding) puts no round polynomial in the clear.
 *
 * MultiCommitGens { n, G, h } (poly/commitments.rs:14-70) on the device: n points G (1 <= n <= 1024, LASSO_ERR_LENGTH
 * otherwise) and h, in the 64-byte affine layout lasso_sample_generators writes; the points are not validated.  Both ways
 * the reference builds them are explicit points of one stream s: MultiCommitGens::new(n, label) is G = s[0..n),
 * h = s[n]; DotProductProofGens::new(n, label) (dot_product.rs:144-150) is gens_n = (s[0..n), s[n+1]) and
 * gens_1 = ([s[n]], s[n+1]).  The object always builds the 8-bit digit-multiples table of its n + 1 points (393 KB per
 * point, 0.4 GB at n = 1024), the one commitment path; LASSO_B200_NO_MULTIPLES does not apply to it.  LASSO_ERR_GENS for
 * null points or output. */
typedef struct lasso_mc_gens lasso_mc_gens;
int lasso_mc_gens_create(lasso_ctx*, const uint64_t* G_affine, size_t n, const uint64_t h_affine[8], lasso_mc_gens** out);
size_t lasso_mc_gens_n(const lasso_mc_gens*);
void lasso_mc_gens_destroy(lasso_mc_gens*);
/* Commitments::batch_commit (commitments.rs:84-93), and commit when gens.n == 1: out = <scalars, G> + blind h,
 * compressed.  LASSO_ERR_GENS for generators of another context or n != gens.n; LASSO_ERR_LENGTH for a null input or
 * output; LASSO_ERR_VALUE for a scalar or blind that is not a canonical residue. */
int lasso_mc_commit(lasso_ctx*, const lasso_mc_gens*, const uint64_t* scalars, size_t n, const uint64_t blind[4],
                    uint8_t out[32]);
/* DotProductProof::prove (subprotocols/dot_product.rs:31-93) on the caller's transcript and tape, advanced in place:
 * protocol name "dot product proof"; tape d_vec (n), r_delta, r_beta; transcript Cx, Cy, a, delta, beta, then
 * challenge c.  proof_out: {delta, beta, z, z_delta, z_beta}, ark-serialize compressed, 136 + 32 n bytes (*proof_len
 * receives the size, also when proof_cap is too small); Cx_out = <x, G_n> + blind_x h_n and Cy_out = y G_1 + blind_y
 * h_1, the commitments the reference returns alongside.  As in the reference, y is not checked against <x, a>: a wrong y
 * gives a proof the verifier rejects.  Two two-row MSMs over the gens' tables, one host wait.
 * Errors, each before any launch and before the transcript or the tape moves: LASSO_ERR_GENS for null generators or
 * generators of another context, gens_1.n != 1 or gens_n.n != n; LASSO_ERR_LENGTH for a null transcript, tape, input or
 * output, or proof_cap too small; LASSO_ERR_VALUE for an x, a, y or blind that is not a canonical residue. */
int lasso_dot_product_prove(lasso_ctx*, const lasso_mc_gens* gens_1, const lasso_mc_gens* gens_n, lasso_transcript*,
                            lasso_random_tape*, const uint64_t* x, const uint64_t blind_x[4], const uint64_t* a, size_t n,
                            const uint64_t y[4], const uint64_t blind_y[4], uint8_t* proof_out, size_t proof_cap,
                            size_t* proof_len, uint8_t Cx_out[32], uint8_t Cy_out[32]);
/* The sumcheck of lasso_sumcheck_prove (g of degree d over the caller's polynomials, num_rounds R) as a
 * ZKSumcheckInstanceProof { comm_polys, comm_evals, proofs }, whose verifier is subprotocols/sumcheck.rs:331-447.
 * The tape is drawn up front: random_vector("blinds_poly", R), random_vector("blinds_evals", R), then each round's
 * DotProductProof draws.  Round j, with claim_0 = the claim and beta_0 = blind_claim, claim_j = eval_{j-1} and
 * beta_j = blinds_evals[j-1] after it: the round polynomial's coefficients c are committed as comm_poly =
 * <c, G_n> + blinds_poly[j] h_n and appended, r_j is drawn; comm_eval = poly(r_j) G_1 + blinds_evals[j] h_1; the
 * transcript takes comm_claim_per_round (comm_claim in round 0, comm_evals[j-1] after it) and comm_eval and gives
 * w = challenge_vector("combine_two_claims_to_one", 2); then DotProductProof::prove of x = c, a = w0 (2, 1, .., 1) +
 * w1 (1, r_j, r_j^2, ..), y = w0 claim_j + w1 eval, blind_y = w0 beta_j + w1 blinds_evals[j].  The reference has no
 * prover for this struct: this tape order is that of Spartan's prove_*_zk, recalled rather than checked against a
 * source.
 *  - proof_out: ark-serialize compressed, 24 + R (200 + 32 (d + 1)) bytes (*proof_len receives it, also when proof_cap
 *    is too small); r_out: R challenges; final_evals_out: n_polys values, element 0 of every polynomial after the binds;
 *  - claim_out (may be null): the first round polynomial at 0 plus at 1, as lasso_sumcheck_prove's;
 *  - comm_claim_out (may be null): claim G_1 + blind_claim h_1, the commitment the verifier takes;
 *  - blind_eval_out (may be null): blinds_evals[R-1], the blind of the last comm_eval, to link it to the caller's
 *    openings.
 * The polynomials are not modified.  Launches: those of lasso_sumcheck_prove, 2 ceil(R/2) for the deltas (two rounds per
 * MSM, before the first round) and 6 per round (comm_poly; comm_eval, with comm_claim in round 0; Cy with beta): three
 * host waits per round more than the plain call.
 * Errors, each before any launch and before the transcript or the tape moves: those of lasso_sumcheck_prove
 * (LASSO_ERR_STRATEGY on a sharded context); LASSO_ERR_GENS for null generators or generators of another context,
 * gens_1.n != 1 or gens_n.n != d + 1 (sumcheck.rs:358); LASSO_ERR_LENGTH for a null tape, blind_claim, r_out or
 * final_evals_out; LASSO_ERR_VALUE for a blind_claim that is not a canonical residue.  The working memory is allocated
 * before the tape or the transcript moves. */
int lasso_zk_sumcheck_prove(lasso_ctx*, const lasso_comb*, const lasso_poly* const* polys, size_t n_polys,
                            size_t num_rounds, const uint64_t blind_claim[4], const lasso_mc_gens* gens_1,
                            const lasso_mc_gens* gens_n, lasso_transcript*, lasso_random_tape*, uint8_t* proof_out,
                            size_t proof_cap, size_t* proof_len, uint64_t* r_out, uint64_t* final_evals_out,
                            uint64_t claim_out[4], uint8_t comm_claim_out[32], uint64_t blind_eval_out[4]);

/* ---------------------------------------------------------------- Σ-protocols of committed scalars
 *
 * The three proofs of subprotocols/zk.rs, which a Spartan-style protocol runs after its ZK sumcheck: knowledge of the
 * value behind a commitment, one committed value the product of two others, two commitments to the same value.  Each
 * runs on the caller's transcript and tape, advanced in place, as the reference's prove does; gens is a lasso_mc_gens
 * with n == 1 (commitments.rs:79), in practice the gens_1 of the ZK sumcheck, and a commitment to v with blind s is
 * v G + s h.  Proofs are ark-serialize compressed, of fixed size; the commitments are the points the reference returns
 * alongside, 32 bytes compressed.  As in the reference, z is not checked against x y nor v1 against v2: a false
 * statement gives a proof the verifier rejects.  Each call is one short MSM over the gens' table (2 launches) and one
 * host wait.  On a sharded context every rank computes alone and returns the single-GPU bytes.
 * Errors, each before any launch and before the transcript or the tape moves: LASSO_ERR_GENS for null generators,
 * generators of another context or gens.n != 1; LASSO_ERR_LENGTH for a null transcript, tape, scalar or output;
 * LASSO_ERR_VALUE for a value or blind that is not a canonical residue. */
/* KnowledgeProof::prove (zk.rs:23-51): tape t1, t2; transcript "knowledge proof", C, alpha, then challenge c.
 * proof_out: {alpha, z1, z2}, 96 bytes; C_out = x G + r h. */
int lasso_knowledge_prove(lasso_ctx*, const lasso_mc_gens* gens, lasso_transcript*, lasso_random_tape*,
                          const uint64_t x[4], const uint64_t r[4], uint8_t proof_out[96], uint8_t C_out[32]);
/* EqualityProof::prove (zk.rs:89-121): tape r; transcript "equality proof", C1, C2, alpha, then challenge c.
 * proof_out: {alpha, z}, 64 bytes; C1_out = v1 G + s1 h, C2_out = v2 G + s2 h. */
int lasso_equality_prove(lasso_ctx*, const lasso_mc_gens* gens, lasso_transcript*, lasso_random_tape*,
                         const uint64_t v1[4], const uint64_t s1[4], const uint64_t v2[4], const uint64_t s2[4],
                         uint8_t proof_out[64], uint8_t C1_out[32], uint8_t C2_out[32]);
/* ProductProof::prove (zk.rs:169-237): tape b1, .., b5; transcript "product proof", X, Y, Z, alpha, beta, delta, then
 * challenge c.  proof_out: {alpha, beta, delta, z[5]}, 256 bytes (z as a fixed-size array: no length prefix);
 * X_out = x G + rX h, Y_out = y G + rY h, Z_out = z G + rZ h. */
int lasso_product_prove(lasso_ctx*, const lasso_mc_gens* gens, lasso_transcript*, lasso_random_tape*,
                        const uint64_t x[4], const uint64_t rX[4], const uint64_t y[4], const uint64_t rY[4],
                        const uint64_t z[4], const uint64_t rZ[4], uint8_t proof_out[256], uint8_t X_out[32],
                        uint8_t Y_out[32], uint8_t Z_out[32]);

/* ---------------------------------------------------------------- grand products over a caller's polynomials
 *
 * GrandProductCircuit::new (subprotocols/grand_product.rs:38-58) over a polynomial of the context with
 * 1 <= num_vars <= 28 (LASSO_ERR_LENGTH otherwise; a single evaluation has no layers).  Layer 0 is the polynomial
 * itself: it is neither copied nor modified, and it MUST outlive the circuit.  The layers above it (2^num_vars - 2
 * elements) are built on the GPU when the circuit is created; the product of all evaluations (`evaluate`,
 * grand_product.rs:60-65) is then a host value.  LASSO_ERR_STRATEGY for a polynomial of another context or a sharded
 * context. */
typedef struct lasso_gp_circuit lasso_gp_circuit;
int lasso_gp_circuit_create(lasso_ctx*, const lasso_poly*, lasso_gp_circuit** out);
int lasso_gp_circuit_evaluate(const lasso_gp_circuit*, uint64_t out[4]);
size_t lasso_gp_circuit_num_vars(const lasso_gp_circuit*);
void lasso_gp_circuit_destroy(lasso_gp_circuit*);
/* BatchedGrandProductArgument::prove (subprotocols/grand_product.rs:100-201) over n circuits of one num_vars v on the
 * caller's transcript, which is advanced in place.  The caller appends the products (lasso_gp_circuit_evaluate) to the
 * transcript first if its protocol does (lasso/memory_checking.rs:683-713).
 *  - proof_out: the ark-serialize bytes of BatchedGrandProductArgument, 8 + v (24 + 64 n) + 52 v (v - 1) bytes
 *    (*proof_len receives the size, also when proof_cap is too small);
 *  - r_out: the v coordinates of rand; claims_out: n values, the final claims_to_verify, which equal P_k(rand) for the
 *    circuits' polynomials P_k.
 * The proof binds the circuits' own layers in place, as the reference does, so a circuit can be proven once; its
 * polynomial (layer 0) is not modified and can be opened at rand afterwards.
 * Errors, each returned before any launch and before the transcript is touched: LASSO_ERR_STRATEGY for n == 0 or
 * n > 32, a circuit of another context, a sharded context, a circuit already proven or the same circuit twice;
 * LASSO_ERR_LENGTH for circuits of different num_vars, proof_cap too small, or a null transcript or output.  The working
 * memory is allocated before the first transcript write. */
int lasso_gp_prove(lasso_ctx*, const lasso_gp_circuit* const* circuits, size_t n, lasso_transcript*, uint8_t* proof_out,
                   size_t proof_cap, size_t* proof_len, uint64_t* r_out, uint64_t* claims_out);

/* Host-resident benchmark helper: number of kernels launched by this context so far, and the wall time
 * (ms) of the last densify / commit / prove calls. */
unsigned long long lasso_launch_count(const lasso_ctx*);
void lasso_last_timings(const lasso_ctx*, double out_ms[3]);
/* With LASSO_B200_SPANS=1 in the environment the prover synchronises around named spans (the analogue of the
 * reference's tracing spans, e.g. "Sumcheck.prove", "Subtables.commit"); this drains them as "name=ms;..." */
size_t lasso_spans(const lasso_ctx*, char* buf, size_t cap);

/* Device-resident bind benchmark hook (bench.py roofline leg): allocates npolys x len random elements on the
 * device once, then runs `iters` top-binds over them on the context stream and returns the average kernel
 * duration in ms measured with CUDA events on that stream. */
int lasso_bench_bind(lasso_ctx*, size_t len, int npolys, int iters, double* avg_ms);

#ifdef __cplusplus
}
#endif
#endif
