// ORACLE — TEST INFRASTRUCTURE ONLY.  ark-serialize (compressed) reading of what lasso_b200 returns as bytes, for the
// oracles of oracle_dense/ and oracle_custom/: PolyEvalProof pieces, BatchedGrandProductArgument, and the
// SparsePolynomialCommitment / SparsePolynomialEvaluationProof that oracle/lasso.hpp serialises (serialize_commitment,
// serialize_proof), read back field by field in the same order.
#pragma once
#include "../oracle/lasso.hpp"

namespace oracle {
namespace {

inline bool ldpoint(const uint8_t* in, Point& out) {
  Affine a;
  if (!decompress(in, a)) return false;
  out = Point::from_affine(a);
  return true;
}
struct Reader {
  const uint8_t* p;
  size_t n, at = 0;
  bool ok = true;
  const uint8_t* take(size_t k) {
    if (!ok || n - at < k) {
      ok = false;
      return nullptr;
    }
    at += k;
    return p + at - k;
  }
  uint64_t u64() {
    const uint8_t* b = take(8);
    uint64_t v = 0;
    if (b) memcpy(&v, b, 8);
    return v;
  }
  Point point() {
    const uint8_t* b = take(32);
    Point q = Point::zero();
    if (b && !ldpoint(b, q)) ok = false;
    return q;
  }
  std::vector<Point> points() {
    const uint64_t k = u64();
    std::vector<Point> v;
    if (k > (n - at) / 32) ok = false;
    for (uint64_t i = 0; ok && i < k; i++) v.push_back(point());
    return v;
  }
  Fr fr() {  // ark rejects a non-canonical encoding
    const uint8_t* b = take(32);
    if (!b) return Fr::zero();
    Fr f = Fr::from_bytes32_mod_order(b);
    uint8_t back[32];
    f.to_bytes(back);
    if (memcmp(back, b, 32)) ok = false;
    return f;
  }
};

inline DotProductProofLog read_dpl(Reader& rd) {
  DotProductProofLog d;
  d.bullet_reduction_proof.L_vec = rd.points();
  d.bullet_reduction_proof.R_vec = rd.points();
  d.delta = rd.point();
  d.beta = rd.point();
  d.z1 = rd.fr();
  d.z2 = rd.fr();
  return d;
}
inline std::vector<Fr> read_frs(Reader& rd, size_t n) {
  std::vector<Fr> v;
  for (size_t i = 0; rd.ok && i < n; i++) v.push_back(rd.fr());
  return v;
}
inline std::vector<Fr> read_vec_fr(Reader& rd) {
  const uint64_t m = rd.u64();
  if (m > (rd.n - rd.at) / 32) rd.ok = false;
  return rd.ok ? read_frs(rd, m) : std::vector<Fr>();
}
inline SumcheckInstanceProof read_sumcheck(Reader& rd) {
  SumcheckInstanceProof p;
  const uint64_t rounds = rd.u64();
  if (rounds > rd.n) rd.ok = false;
  for (uint64_t j = 0; rd.ok && j < rounds; j++) {
    CompressedUniPoly c;
    c.coeffs_except_linear_term = read_vec_fr(rd);
    if (c.coeffs_except_linear_term.empty()) rd.ok = false;
    p.compressed_polys.push_back(c);
  }
  return p;
}
inline BatchedGrandProductArgument read_gpa(Reader& rd) {
  BatchedGrandProductArgument p;
  const uint64_t layers = rd.u64();
  if (layers > rd.n) rd.ok = false;
  for (uint64_t l = 0; rd.ok && l < layers; l++) {
    LayerProofBatched lp;
    lp.proof = read_sumcheck(rd);
    lp.claims_prod_left = read_vec_fr(rd);
    lp.claims_prod_right = read_vec_fr(rd);
    p.proof.push_back(std::move(lp));
  }
  return p;
}
// lasso_commit's bytes; false when they do not parse or have bytes left over
inline bool read_sparse_commitment(const uint8_t* b, size_t n, SparsePolynomialCommitment& c) {
  Reader rd{b, n};
  c.l_variate_polys_commitment.C = rd.points();
  c.log_m_variate_polys_commitment.C = rd.points();
  c.s = rd.u64();
  c.log_m = rd.u64();
  c.m = rd.u64();
  return rd.ok && rd.at == n;
}
// a proof with alpha memories over C dimensions; false when the bytes do not parse or have bytes left over
inline bool read_sparse_proof(const uint8_t* b, size_t n, size_t alpha, size_t C, SparsePolynomialEvaluationProof& p) {
  Reader rd{b, n};
  p.comm_derefs.C = rd.points();
  p.primary_proof = read_sumcheck(rd);
  p.claimed_evaluation = rd.fr();
  p.eval_derefs = read_frs(rd, alpha);
  p.proof_derefs.proof_table_eval.proof = read_dpl(rd);
  auto& pl = p.memory_check.proof_prod_layer;
  for (size_t i = 0; rd.ok && i < alpha; i++) {
    std::array<Fr, 4> e;
    for (int k = 0; k < 4; k++) e[k] = rd.fr();
    pl.grand_product_evals.push_back(e);
  }
  pl.proof_mem = read_gpa(rd);
  pl.proof_ops = read_gpa(rd);
  auto& hl = p.memory_check.proof_hash_layer;
  hl.eval_dim = read_frs(rd, C);
  hl.eval_read = read_frs(rd, C);
  hl.eval_final = read_frs(rd, C);
  hl.eval_derefs = read_frs(rd, alpha);
  hl.proof_ops.proof = read_dpl(rd);
  hl.proof_mem.proof = read_dpl(rd);
  hl.proof_derefs.proof_table_eval.proof = read_dpl(rd);
  return rd.ok && rd.at == n;
}
// SparsePolynomialCommitment::append_to_transcript (surge.rs:70-82); oracle/lasso.hpp has the PolyCommitment half
inline void append_sparse_commitment(const SparsePolynomialCommitment& c, Transcript& t) {
  c.l_variate_polys_commitment.append_to_transcript("l_variate_polys_commitment", t);
  c.log_m_variate_polys_commitment.append_to_transcript("log_m_variate_polys_commitment", t);
  t.append_u64("s", c.s);
  t.append_u64("log_m", c.log_m);
  t.append_u64("m", c.m);
}

}  // namespace
}  // namespace oracle
