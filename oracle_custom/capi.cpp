// ORACLE FOR CALLER-DEFINED STRATEGIES — TEST INFRASTRUCTURE ONLY.
//
// A caller-defined SubtableStrategy (lasso_b200's lasso_strategy_create): explicit tables and memory maps,
// combine_lookups as a straight-line program and a declared g_poly_degree.  The oracle in oracle/ restates the
// reference for its five built-in strategies; this file builds on it (same primitives, same transcript, same
// serialisation) and restates only the parts of surge.rs / memory_checking.rs / subtables/mod.rs that take the
// strategy as a parameter, with the custom strategy in its place:
//   SparsePolynomialEvaluationProof::prove / verify  surge.rs:118-271
//   MemoryCheckingProof::prove / verify              memory_checking.rs:26-147
//   HashLayerProof::verify                           memory_checking.rs:462-523
//   Subtables::new, compute_sumcheck_claim           subtables/mod.rs:116-129, 186-216
// evaluate_subtable_mle of a custom table is its dense MLE (DensePolynomial::evaluate, point[0] the MSB).
#include "../oracle_dense/sparse_bytes.hpp"

using namespace oracle;

namespace {

Fr ldfr(const uint64_t* p) { return Fr::from_raw(p); }
void stfr(uint64_t* p, const Fr& f) { memcpy(p, f.l, 32); }
Affine ldaff(const uint64_t* p) { return Affine{Fq::from_raw(p), Fq::from_raw(p + 4)}; }
std::vector<Fr> ldvec(const uint64_t* p, size_t n) {
  std::vector<Fr> v(n);
  for (size_t i = 0; i < n; i++) v[i] = ldfr(p + 4 * i);
  return v;
}

// Program: 3 ints {op, a, b} per instruction; slots 0..alpha-1 hold the memory values, instruction j writes slot
// alpha + j, the last slot is g.  op: 0 a + b, 1 a - b, 2 a * b, 3 a * K[b], 4 a + K[b].
struct CustomStrategy {
  size_t C, log_m, degree;
  std::vector<std::vector<Fr>> tables;
  std::vector<size_t> sub, dim;
  std::vector<int32_t> prog;
  std::vector<Fr> K;
  size_t num_memories() const { return sub.size(); }
  Fr combine_lookups(const Fr* vals) const {
    const size_t alpha = sub.size(), n = prog.size() / 3;
    std::vector<Fr> s(vals, vals + alpha);
    s.resize(alpha + n);
    for (size_t j = 0; j < n; j++) {
      const int32_t op = prog[3 * j], a = prog[3 * j + 1], b = prog[3 * j + 2];
      switch (op) {
        case 0: s[alpha + j] = s[a] + s[b]; break;
        case 1: s[alpha + j] = s[a] - s[b]; break;
        case 2: s[alpha + j] = s[a] * s[b]; break;
        case 3: s[alpha + j] = s[a] * K[b]; break;
        default: s[alpha + j] = s[a] + K[b]; break;
      }
    }
    return s.back();
  }
  Fr evaluate_subtable_mle(size_t k, const std::vector<Fr>& point) const {
    return DensePolynomial(tables[k]).evaluate(point);
  }
};

// Subtables::new (subtables/mod.rs:116-129) with the custom tables and maps.  Subtables' own constructor takes a
// built-in strategy: it is given the smallest one and its fields are then replaced.  HashLayerProof::prove and
// Subtables::commit read only lookup_polys and combined_poly.
Subtables make_subtables(const CustomStrategy& S, const DensifiedRepresentation& dense) {
  Subtables st(Strategy{STRAT_AND, 1, 2, 0}, {std::vector<size_t>(dense.s, 0)}, dense.s);
  st.subtable_entries = S.tables;
  st.lookup_polys.clear();
  for (size_t i = 0; i < S.num_memories(); i++) {
    const auto& table = S.tables[S.sub[i]];
    const auto& idx = dense.dim_usize[S.dim[i]];
    std::vector<Fr> lookups(dense.s);
    for (size_t j = 0; j < dense.s; j++) lookups[j] = table[idx[j]];
    st.lookup_polys.emplace_back(std::move(lookups));
  }
  st.combined_poly = DensePolynomial::merge(st.lookup_polys);
  return st;
}

// subtables/mod.rs:186-216
Fr sumcheck_claim(const CustomStrategy& S, const Subtables& st, const EqPolynomial& eq) {
  std::vector<Fr> eq_evals = eq.evals();
  const size_t nm = S.num_memories();
  Fr total = Fr::zero();
  std::vector<Fr> ops(nm);
  for (size_t k = 0; k < st.lookup_polys[0].len; k++) {
    for (size_t j = 0; j < nm; j++) ops[j] = st.lookup_polys[j][k];
    total += eq_evals[k] * S.combine_lookups(ops.data());
  }
  return total;
}

// surge.rs:118-211 with memory_checking.rs:55-83
SparsePolynomialEvaluationProof prove(const CustomStrategy& S, DensifiedRepresentation& dense, const std::vector<Fr>& r,
                                      const SparsePolyCommitmentGens& gens, Transcript& transcript, RandomTape& tape) {
  transcript.append_protocol_name("Lasso SparsePolynomialEvaluationProof");
  if (r.size() != ark_log2(dense.s)) throw std::runtime_error("r.len() != log2(s) (surge.rs:131)");
  SparsePolynomialEvaluationProof out;
  Subtables subtables = make_subtables(S, dense);
  out.comm_derefs = subtables.commit(gens.gens_derefs);
  append_combined_table_commitment(out.comm_derefs, "comm_poly_row_col_ops_val", transcript);
  EqPolynomial eq(r);
  out.claimed_evaluation = sumcheck_claim(S, subtables, eq);
  transcript.append_scalar("claim_eval_scalar_product", out.claimed_evaluation);
  std::vector<DensePolynomial> combined;
  for (auto& p : subtables.lookup_polys) combined.push_back(p.clone());
  combined.emplace_back(eq.evals());
  const size_t alpha = S.num_memories();
  std::vector<Fr> r_z, final_evals;
  out.primary_proof = SumcheckInstanceProof::prove_arbitrary(
      log_2(dense.s), combined, [&](const Fr* v) { return S.combine_lookups(v) * v[alpha]; }, S.degree + 1, transcript,
      r_z, final_evals);
  for (auto& p : subtables.lookup_polys) out.eval_derefs.push_back(p.evaluate(r_z));
  out.proof_derefs = CombinedTableEvalProof::prove(subtables.combined_poly, out.eval_derefs, r_z, gens.gens_derefs,
                                                   transcript, tape);
  std::vector<Fr> r_hash = transcript.challenge_vector("challenge_r_hash", 2);
  // MemoryCheckingProof::prove with Subtables::to_grand_products (subtables/mod.rs:133-175)
  transcript.append_protocol_name("Lasso MemoryCheckingProof");
  std::vector<GrandProducts> gps;
  for (size_t i = 0; i < alpha; i++) {
    const size_t j = S.dim[i];
    gps.push_back(make_grand_products(S.tables[S.sub[i]], dense.dim[j], dense.dim_usize[j], dense.read[j],
                                      dense.final_[j], r_hash[0], r_hash[1]));
  }
  std::vector<Fr> rand_mem, rand_ops;
  out.memory_check.proof_prod_layer = ProductLayerProof::prove(gps, transcript, rand_mem, rand_ops);
  out.memory_check.proof_hash_layer =
      HashLayerProof::prove(rand_mem, rand_ops, dense, subtables, gens, transcript, tape);
  return out;
}

// HashLayerProof::verify (memory_checking.rs:462-523)
bool verify_hash_layer(const HashLayerProof& h, const CustomStrategy& S, const std::vector<Fr>& rand_mem,
                       const std::vector<Fr>& rand_ops, const std::vector<std::array<Fr, 4>>& claims,
                       const SparsePolynomialCommitment& comm, const SparsePolyCommitmentGens& gens,
                       const PolyCommitment& comm_derefs, const Fr& gamma, const Fr& tau, Transcript& transcript) {
  transcript.append_protocol_name("Lasso HashLayerProof");
  if (!h.proof_derefs.verify(rand_ops, h.eval_derefs, gens.gens_derefs, comm_derefs, transcript)) return false;
  std::vector<Fr> evals_ops = h.eval_dim;
  evals_ops.insert(evals_ops.end(), h.eval_read.begin(), h.eval_read.end());
  evals_ops.resize(next_power_of_two(evals_ops.size()), Fr::zero());
  transcript.append_scalars("claim_evals_ops", evals_ops);
  std::vector<Fr> challenges_ops = transcript.challenge_vector("challenge_combine_n_to_one", log_2(evals_ops.size()));
  DensePolynomial poly_evals_ops(evals_ops);
  for (size_t i = challenges_ops.size(); i-- > 0;) poly_evals_ops.bound_poly_var_bot(challenges_ops[i]);
  Fr joint_claim_eval_ops = poly_evals_ops[0];
  std::vector<Fr> r_joint_ops = challenges_ops;
  r_joint_ops.insert(r_joint_ops.end(), rand_ops.begin(), rand_ops.end());
  transcript.append_scalar("joint_claim_eval_ops", joint_claim_eval_ops);
  if (!h.proof_ops.verify_plain(gens.gens_combined_l_variate, transcript, r_joint_ops, joint_claim_eval_ops,
                                comm.l_variate_polys_commitment))
    return false;
  transcript.append_scalars("claim_evals_mem", h.eval_final);
  std::vector<Fr> challenges_mem = transcript.challenge_vector("challenge_combine_two_to_one", log_2(h.eval_final.size()));
  DensePolynomial poly_evals_mem = DensePolynomial::new_padded(h.eval_final);
  for (size_t i = challenges_mem.size(); i-- > 0;) poly_evals_mem.bound_poly_var_bot(challenges_mem[i]);
  Fr joint_claim_eval_mem = poly_evals_mem[0];
  std::vector<Fr> r_joint_mem = challenges_mem;
  r_joint_mem.insert(r_joint_mem.end(), rand_mem.begin(), rand_mem.end());
  transcript.append_scalar("joint_claim_eval_mem", joint_claim_eval_mem);
  if (!h.proof_mem.verify_plain(gens.gens_combined_log_m_variate, transcript, r_joint_mem, joint_claim_eval_mem,
                                comm.log_m_variate_polys_commitment))
    return false;
  // check_reed_solomon_fingerprints (memory_checking.rs:477-523)
  Fr init_addr = identity_poly_evaluate(rand_mem);
  Fr g2 = gamma.square();
  auto hash_func = [&](const Fr& a, const Fr& v, const Fr& t) { return t * g2 + v * gamma + a - tau; };
  for (size_t i = 0; i < claims.size(); i++) {
    size_t j = S.dim[i], k = S.sub[i];
    Fr init_memory = S.evaluate_subtable_mle(k, rand_mem);
    if (hash_func(init_addr, init_memory, Fr::zero()) != claims[i][0]) return false;
    if (hash_func(h.eval_dim[j], h.eval_derefs[i], h.eval_read[j]) != claims[i][1]) return false;
    if (hash_func(h.eval_dim[j], h.eval_derefs[i], h.eval_read[j] + Fr::one()) != claims[i][2]) return false;
    if (hash_func(init_addr, init_memory, h.eval_final[j]) != claims[i][3]) return false;
  }
  return true;
}

// surge.rs:213-271 with MemoryCheckingProof::verify (memory_checking.rs:85-147)
bool verify(const SparsePolynomialEvaluationProof& p, const CustomStrategy& S, const SparsePolynomialCommitment& comm,
            const std::vector<Fr>& eq_randomness, const SparsePolyCommitmentGens& gens, Transcript& transcript) {
  transcript.append_protocol_name("Lasso SparsePolynomialEvaluationProof");
  append_combined_table_commitment(p.comm_derefs, "comm_poly_row_col_ops_val", transcript);
  transcript.append_scalar("claim_eval_scalar_product", p.claimed_evaluation);
  Fr claim_last;
  std::vector<Fr> r_z;
  if (!p.primary_proof.verify(p.claimed_evaluation, log_2(comm.s), S.degree + 1, transcript, claim_last, r_z))
    return false;
  Fr eq_eval = EqPolynomial(eq_randomness).evaluate(r_z);
  if (p.eval_derefs.size() != S.num_memories()) return false;
  if (eq_eval * S.combine_lookups(p.eval_derefs.data()) != claim_last) return false;
  if (!p.proof_derefs.verify(r_z, p.eval_derefs, gens.gens_derefs, p.comm_derefs, transcript)) return false;
  std::vector<Fr> r_hash = transcript.challenge_vector("challenge_r_hash", 2);
  transcript.append_protocol_name("Lasso MemoryCheckingProof");
  std::vector<Fr> claims_mem, rand_mem, claims_ops, rand_ops;
  if (!p.memory_check.proof_prod_layer.verify(next_power_of_two(comm.s), comm.m, transcript, claims_mem, rand_mem,
                                               claims_ops, rand_ops))
    return false;
  std::vector<std::array<Fr, 4>> claims;
  for (size_t i = 0; i < S.num_memories(); i++)
    claims.push_back({claims_mem[2 * i], claims_ops[2 * i], claims_ops[2 * i + 1], claims_mem[2 * i + 1]});
  return verify_hash_layer(p.memory_check.proof_hash_layer, S, rand_mem, rand_ops, claims, comm, gens, p.comm_derefs,
                           r_hash[0], r_hash[1], transcript);
}

// tables = nsub x M u32 (row-major); maps, program as int32; K = n_k Fr.  Taken as given (the GPU library checks
// its own copy of the descriptor).
CustomStrategy make(size_t C, size_t log_m, size_t nsub, const uint32_t* tables, size_t alpha, const int32_t* sub,
                    const int32_t* dim, const int32_t* prog, size_t n_ops, const uint64_t* K, size_t n_k,
                    size_t degree) {
  CustomStrategy S;
  S.C = C;
  S.log_m = log_m;
  S.degree = degree;
  const size_t M = pow2(log_m);
  S.tables.assign(nsub, std::vector<Fr>(M));
  for (size_t k = 0; k < nsub; k++)
    for (size_t i = 0; i < M; i++) S.tables[k][i] = Fr::from_u64(tables[k * M + i]);
  S.sub.assign(sub, sub + alpha);
  S.dim.assign(dim, dim + alpha);
  S.prog.assign(prog, prog + 3 * n_ops);
  S.K = ldvec(K, n_k);
  return S;
}
// the same with tables = nsub x M Fr (4 Montgomery limbs each, row-major): entries of any width
CustomStrategy make_fr(size_t C, size_t log_m, size_t nsub, const uint64_t* tables, size_t alpha, const int32_t* sub,
                       const int32_t* dim, const int32_t* prog, size_t n_ops, const uint64_t* K, size_t n_k,
                       size_t degree) {
  const uint32_t zero = 0;
  CustomStrategy S = make(C, log_m, 0, &zero, alpha, sub, dim, prog, n_ops, K, n_k, degree);
  const size_t M = pow2(log_m);
  for (size_t k = 0; k < nsub; k++) S.tables.push_back(ldvec(tables + 4 * k * M, M));
  return S;
}

// one round of the primary sumcheck's evaluation loop (sumcheck.rs:179-237): polys = (alpha+1) x len, the last eq
void sumcheck_round(const CustomStrategy& S, const uint64_t* polys, size_t len, uint64_t* evals_out) {
  const size_t alpha = S.num_memories(), np = alpha + 1, deg = S.degree + 1, half = len / 2;
  auto g = [&](const std::vector<Fr>& v) { return S.combine_lookups(v.data()) * v[alpha]; };
  std::vector<Fr> ev(deg + 1, Fr::zero()), cur(np), nxt(np);
  for (size_t i = 0; i < half; i++) {
    for (size_t j = 0; j < np; j++) cur[j] = ldfr(polys + 4 * (j * len + i));
    ev[0] += g(cur);
    for (size_t j = 0; j < np; j++) cur[j] = ldfr(polys + 4 * (j * len + half + i));
    ev[1] += g(cur);
    for (size_t t = 2; t <= deg; t++) {
      for (size_t j = 0; j < np; j++)
        nxt[j] = cur[j] + ldfr(polys + 4 * (j * len + half + i)) - ldfr(polys + 4 * (j * len + i));
      ev[t] += g(nxt);
      cur.swap(nxt);
    }
  }
  memcpy(evals_out, ev.data(), (deg + 1) * 32);
}

// Densify -> commit -> prove (-> verify): see orc_custom_prove
int prove_all(const CustomStrategy& S, const uint64_t* indices, size_t n, const uint64_t* r, const uint64_t* gens,
              size_t n_gens, const uint64_t* tape_seed, int flags, uint8_t* proof_out, size_t proof_cap, size_t* proof_len,
              uint8_t* commit_out, size_t commit_cap, size_t* commit_len, uint64_t* challenges_out, size_t challenges_cap,
              size_t* n_challenges) {
  try {
    const size_t C = S.C, log_m = S.log_m, alpha = S.num_memories();
    std::vector<std::vector<size_t>> idx(n, std::vector<size_t>(C));
    for (size_t j = 0; j < n; j++)
      for (size_t i = 0; i < C; i++) idx[j][i] = indices[j * C + i];
    std::vector<Affine> stream(n_gens);
    for (size_t i = 0; i < n_gens; i++) stream[i] = ldaff(gens + 8 * i);
    DensifiedRepresentation dense = DensifiedRepresentation::from_lookup_indices(idx, C, log_m);
    if (n_gens < SparsePolyCommitmentGens::needs_points(C, dense.s, alpha, log_m)) return -2;
    SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(C, dense.s, alpha, log_m, stream);
    SparsePolynomialCommitment commitment = densified_commit(dense, pg);
    std::vector<Fr> rv = ldvec(r, ark_log2(dense.s));
    RandomTape tape("proof", ldfr(tape_seed));
    Transcript tp("example");
    std::vector<Fr> trace;
    tp.trace = &trace;
    SparsePolynomialEvaluationProof proof = prove(S, dense, rv, pg, tp, tape);
    std::vector<uint8_t> pb = serialize_proof(proof), cb = serialize_commitment(commitment);
    *proof_len = pb.size();
    if (proof_out && pb.size() <= proof_cap) memcpy(proof_out, pb.data(), pb.size());
    *commit_len = cb.size();
    if (commit_out && cb.size() <= commit_cap) memcpy(commit_out, cb.data(), cb.size());
    *n_challenges = trace.size();
    if (challenges_out)
      for (size_t i = 0; i < trace.size() && i < challenges_cap; i++) stfr(challenges_out + 4 * i, trace[i]);
    if (flags & 1) {
      if (flags & 2) proof.claimed_evaluation += Fr::one();
      if (flags & 4) proof.memory_check.proof_hash_layer.eval_read[0] += Fr::one();
      Transcript tv("example");
      return verify(proof, S, commitment, rv, pg, tv) ? 0 : 1;
    }
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "orc_custom_prove: %s\n", e.what());
    return -1;
  }
}

// The same proof on a caller's transcript and tape (oracle_dense's Transcript / RandomTape objects): densify, commit
// (comm_out: the serialised commitment), prove at r.  Returns the proof's length, 0 on error; claim_out = the claimed
// evaluation.
size_t prove_transcript(const CustomStrategy& S, const uint64_t* indices, size_t n, const uint64_t* r, const uint64_t* gens,
                        size_t n_gens, void* transcript, void* tape, uint8_t* out, size_t cap, uint8_t* comm_out,
                        size_t comm_cap, uint64_t* claim_out) {
  try {
    const size_t C = S.C, log_m = S.log_m, alpha = S.num_memories();
    std::vector<std::vector<size_t>> idx(n, std::vector<size_t>(C));
    for (size_t j = 0; j < n; j++)
      for (size_t i = 0; i < C; i++) idx[j][i] = indices[j * C + i];
    std::vector<Affine> stream(n_gens);
    for (size_t i = 0; i < n_gens; i++) stream[i] = ldaff(gens + 8 * i);
    DensifiedRepresentation dense = DensifiedRepresentation::from_lookup_indices(idx, C, log_m);
    if (n_gens < SparsePolyCommitmentGens::needs_points(C, dense.s, alpha, log_m)) return 0;
    SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(C, dense.s, alpha, log_m, stream);
    const std::vector<uint8_t> cb = serialize_commitment(densified_commit(dense, pg));
    const SparsePolynomialEvaluationProof proof =
        prove(S, dense, ldvec(r, ark_log2(dense.s)), pg, *(Transcript*)transcript, *(RandomTape*)tape);
    const std::vector<uint8_t> pb = serialize_proof(proof);
    if (pb.size() > cap || cb.size() > comm_cap) return 0;
    memcpy(out, pb.data(), pb.size());
    memcpy(comm_out, cb.data(), cb.size());
    stfr(claim_out, proof.claimed_evaluation);
    return pb.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orc_custom_prove_transcript: %s\n", e.what());
    return 0;
  }
}
// verify of serialised proof and commitment bytes on a caller's transcript: 0 accepted, 1 rejected, 2 the bytes do not
// parse or the generator stream is too short
int verify_transcript(const CustomStrategy& S, const uint64_t* gens, size_t n_gens, const uint8_t* comm, size_t comm_len,
                      const uint8_t* proof, size_t proof_len, const uint64_t* r, void* transcript) {
  SparsePolynomialCommitment c;
  SparsePolynomialEvaluationProof p;
  if (!read_sparse_commitment(comm, comm_len, c) || !read_sparse_proof(proof, proof_len, S.num_memories(), S.C, p)) return 2;
  if (n_gens < SparsePolyCommitmentGens::needs_points(S.C, c.s, S.num_memories(), S.log_m)) return 2;
  std::vector<Affine> stream(n_gens);
  for (size_t i = 0; i < n_gens; i++) stream[i] = ldaff(gens + 8 * i);
  SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(S.C, c.s, S.num_memories(), S.log_m, stream);
  return verify(p, S, c, ldvec(r, ark_log2(c.s)), pg, *(Transcript*)transcript) ? 0 : 1;
}

}  // namespace

#define ORC_CUSTOM_ARGS                                                                                             \
  size_t C, size_t log_m, size_t nsub, const uint32_t *tables, size_t alpha, const int32_t *sub, const int32_t *dim, \
      const int32_t *prog, size_t n_ops, const uint64_t *K, size_t n_k, size_t degree
#define ORC_CUSTOM make(C, log_m, nsub, tables, alpha, sub, dim, prog, n_ops, K, n_k, degree)
#define ORC_CUSTOM_ARGS_FR                                                                                          \
  size_t C, size_t log_m, size_t nsub, const uint64_t *tables, size_t alpha, const int32_t *sub, const int32_t *dim, \
      const int32_t *prog, size_t n_ops, const uint64_t *K, size_t n_k, size_t degree
#define ORC_CUSTOM_FR make_fr(C, log_m, nsub, tables, alpha, sub, dim, prog, n_ops, K, n_k, degree)

extern "C" {

void orc_custom_combine_lookups(ORC_CUSTOM_ARGS, const uint64_t* vals, uint64_t* out) {
  stfr(out, ORC_CUSTOM.combine_lookups(ldvec(vals, alpha).data()));
}
void orc_custom_evaluate_subtable_mle(ORC_CUSTOM_ARGS, size_t idx, const uint64_t* point, size_t npoint,
                                      uint64_t* out) {
  stfr(out, ORC_CUSTOM.evaluate_subtable_mle(idx, ldvec(point, npoint)));
}
// one round of the primary sumcheck's evaluation loop (sumcheck.rs:179-237): polys = (alpha+1) x len, the last eq
void orc_custom_sumcheck_round(ORC_CUSTOM_ARGS, const uint64_t* polys, size_t len, uint64_t* evals_out) {
  sumcheck_round(ORC_CUSTOM, polys, len, evals_out);
}
// Densify -> commit -> prove (-> verify), as orc_prove in oracle/capi.cpp.  indices: n x C row-major; gens: affine
// generator stream of n_gens points.  flags: bit0 = run verify, bit1 = tamper with the claimed evaluation before
// verifying, bit2 = tamper with a memory-checking evaluation instead.  Returns 0 ok; 1 verify rejected; < 0 error.
int orc_custom_prove(ORC_CUSTOM_ARGS, const uint64_t* indices, size_t n, const uint64_t* r, const uint64_t* gens,
                     size_t n_gens, const uint64_t* tape_seed, int flags, uint8_t* proof_out, size_t proof_cap,
                     size_t* proof_len, uint8_t* commit_out, size_t commit_cap, size_t* commit_len,
                     uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges) {
  return prove_all(ORC_CUSTOM, indices, n, r, gens, n_gens, tape_seed, flags, proof_out, proof_cap, proof_len, commit_out,
                   commit_cap, commit_len, challenges_out, challenges_cap, n_challenges);
}

// _fr twins: the tables as nsub x M Fr (Montgomery limbs) instead of u32
void orc_custom_combine_lookups_fr(ORC_CUSTOM_ARGS_FR, const uint64_t* vals, uint64_t* out) {
  stfr(out, ORC_CUSTOM_FR.combine_lookups(ldvec(vals, alpha).data()));
}
void orc_custom_evaluate_subtable_mle_fr(ORC_CUSTOM_ARGS_FR, size_t idx, const uint64_t* point, size_t npoint,
                                         uint64_t* out) {
  stfr(out, ORC_CUSTOM_FR.evaluate_subtable_mle(idx, ldvec(point, npoint)));
}
void orc_custom_sumcheck_round_fr(ORC_CUSTOM_ARGS_FR, const uint64_t* polys, size_t len, uint64_t* evals_out) {
  sumcheck_round(ORC_CUSTOM_FR, polys, len, evals_out);
}
int orc_custom_prove_fr(ORC_CUSTOM_ARGS_FR, const uint64_t* indices, size_t n, const uint64_t* r, const uint64_t* gens,
                        size_t n_gens, const uint64_t* tape_seed, int flags, uint8_t* proof_out, size_t proof_cap,
                        size_t* proof_len, uint8_t* commit_out, size_t commit_cap, size_t* commit_len,
                        uint64_t* challenges_out, size_t challenges_cap, size_t* n_challenges) {
  return prove_all(ORC_CUSTOM_FR, indices, n, r, gens, n_gens, tape_seed, flags, proof_out, proof_cap, proof_len,
                   commit_out, commit_cap, commit_len, challenges_out, challenges_cap, n_challenges);
}

// prove_transcript / verify_transcript above, tables as u32 and as Fr
size_t orc_custom_prove_transcript(ORC_CUSTOM_ARGS, const uint64_t* indices, size_t n, const uint64_t* r,
                                   const uint64_t* gens, size_t n_gens, void* transcript, void* tape, uint8_t* out,
                                   size_t cap, uint8_t* comm_out, size_t comm_cap, uint64_t* claim_out) {
  return prove_transcript(ORC_CUSTOM, indices, n, r, gens, n_gens, transcript, tape, out, cap, comm_out, comm_cap, claim_out);
}
int orc_custom_verify_transcript(ORC_CUSTOM_ARGS, const uint64_t* gens, size_t n_gens, const uint8_t* comm, size_t comm_len,
                                 const uint8_t* proof, size_t proof_len, const uint64_t* r, void* transcript) {
  return verify_transcript(ORC_CUSTOM, gens, n_gens, comm, comm_len, proof, proof_len, r, transcript);
}
size_t orc_custom_prove_transcript_fr(ORC_CUSTOM_ARGS_FR, const uint64_t* indices, size_t n, const uint64_t* r,
                                      const uint64_t* gens, size_t n_gens, void* transcript, void* tape, uint8_t* out,
                                      size_t cap, uint8_t* comm_out, size_t comm_cap, uint64_t* claim_out) {
  return prove_transcript(ORC_CUSTOM_FR, indices, n, r, gens, n_gens, transcript, tape, out, cap, comm_out, comm_cap,
                          claim_out);
}
int orc_custom_verify_transcript_fr(ORC_CUSTOM_ARGS_FR, const uint64_t* gens, size_t n_gens, const uint8_t* comm,
                                    size_t comm_len, const uint8_t* proof, size_t proof_len, const uint64_t* r,
                                    void* transcript) {
  return verify_transcript(ORC_CUSTOM_FR, gens, n_gens, comm, comm_len, proof, proof_len, r, transcript);
}

}  // extern "C"
