// ORACLE FOR DENSE POLYNOMIALS ON A CALLER'S TRANSCRIPT — TEST INFRASTRUCTURE ONLY.
//
// lasso_b200's lasso_transcript_* / lasso_random_tape_* / lasso_poly_* expose the reference's dense-polynomial items to
// a caller that holds its own Fiat-Shamir transcript.  The oracle in oracle/ restates those items (PolyCommitmentGens,
// DensePolynomial::commit / evaluate, PolyEvalProof::prove / verify_plain, ProofTranscript, RandomTape) but drives them
// only inside its own round trips; this file puts C entry points on the same code that take and return what the
// library takes and returns: serialised bytes, an explicit generator stream, and transcript / tape objects that live
// across calls.  Nothing here is restated anew except the ark-serialize reading of a PolyEvalProof, the hiding forms
// of DensePolynomial::commit / PolyEvalProof::prove (blinds on h), DotProductProof and ZKSumcheckInstanceProof with
// a prover for the latter (DESIGN §3.16), and the Σ-protocols of subprotocols/zk.rs (DESIGN §3.17), which oracle/ leaves
// out.
#include "sparse_bytes.hpp"

using namespace oracle;

namespace {

Fr ldfr(const uint64_t* p) { return Fr::from_raw(p); }
void stfr(uint64_t* p, const Fr& f) { memcpy(p, f.l, 32); }
std::vector<Fr> ldvec(const uint64_t* p, size_t n) {
  std::vector<Fr> v(n);
  for (size_t i = 0; i < n; i++) v[i] = ldfr(p + 4 * i);
  return v;
}
std::vector<Affine> ldstream(const uint64_t* p, size_t n) {
  std::vector<Affine> s(n);
  for (size_t i = 0; i < n; i++) s[i] = Affine{Fq::from_raw(p + 8 * i), Fq::from_raw(p + 8 * i + 4)};
  return s;
}
void put_u64(std::vector<uint8_t>& b, uint64_t v) {
  for (int i = 0; i < 8; i++) b.push_back((uint8_t)(v >> (8 * i)));
}
void put_point(std::vector<uint8_t>& b, const Point& p) {
  uint8_t c[32];
  p.compress(c);
  b.insert(b.end(), c, c + 32);
}
void put_fr(std::vector<uint8_t>& b, const Fr& f) {
  uint8_t c[32];
  f.to_bytes(c);
  b.insert(b.end(), c, c + 32);
}
// ark-serialize (compressed) of PolyCommitment { C: Vec<G> }
std::vector<uint8_t> ser_commitment(const PolyCommitment& c) {
  std::vector<uint8_t> b;
  put_u64(b, c.C.size());
  for (const Point& p : c.C) put_point(b, p);
  return b;
}
// PolyEvalProof { proof: DotProductProofLog { bullet_reduction_proof { L_vec, R_vec }, delta, beta, z1, z2 } }
std::vector<uint8_t> ser_proof(const PolyEvalProof& p) {
  std::vector<uint8_t> b;
  const DotProductProofLog& d = p.proof;
  put_u64(b, d.bullet_reduction_proof.L_vec.size());
  for (const Point& q : d.bullet_reduction_proof.L_vec) put_point(b, q);
  put_u64(b, d.bullet_reduction_proof.R_vec.size());
  for (const Point& q : d.bullet_reduction_proof.R_vec) put_point(b, q);
  put_point(b, d.delta);
  put_point(b, d.beta);
  put_fr(b, d.z1);
  put_fr(b, d.z2);
  return b;
}
// PolyEvalProof { proof } of serialised bytes; false when they do not parse
bool read_poly_eval_proof(const uint8_t* proof, size_t proof_len, PolyEvalProof& p) {
  Reader rp{proof, proof_len};
  p.proof.bullet_reduction_proof.L_vec = rp.points();
  p.proof.bullet_reduction_proof.R_vec = rp.points();
  p.proof.delta = rp.point();
  p.proof.beta = rp.point();
  p.proof.z1 = rp.fr();
  p.proof.z2 = rp.fr();
  return rp.ok && rp.at == proof_len;
}
// The hiding forms of DensePolynomial::commit and PolyEvalProof::prove, restated beside the unblinded ones of oracle/:
// commit (dense_mlpoly.rs:152-181): row i is batch_commit(row_i, blinds[i]) = <row_i, G> + blinds[i] h
PolyCommitment commit_hiding(const DensePolynomial& poly, const PolyCommitmentGens& gens, const std::vector<Fr>& blinds) {
  size_t lv, rv;
  EqPolynomial::compute_factored_lens(poly.num_vars, lv, rv);
  const size_t L_size = pow2(lv), R_size = pow2(rv);
  if (blinds.size() != L_size) throw std::runtime_error("commit_hiding: one blind per row");
  PolyCommitment pc;
  pc.C.resize(L_size);
#pragma omp parallel for schedule(dynamic, 1)
  for (size_t i = 0; i < L_size; i++) pc.C[i] = batch_commit(&poly.Z[R_size * i], R_size, blinds[i], gens.gens.gens_n);
  return pc;
}
// prove (dense_mlpoly.rs:301-359) with Some(blinds) (empty: None, all zero) and blind_Zr: LZ_blind = <L, blinds> is
// the dot-product proof's blind_x, blind_Zr its blind_y; C_Zr = Zr Q + blind_Zr h is returned alongside
PolyEvalProof prove_hiding(const DensePolynomial& poly, const std::vector<Fr>& blinds, const std::vector<Fr>& r,
                           const Fr& Zr, const Fr& blind_Zr, const PolyCommitmentGens& gens, Transcript& transcript,
                           RandomTape& tape, Point& C_Zr) {
  transcript.append_protocol_name("polynomial evaluation proof");
  std::vector<Fr> L, R;
  EqPolynomial(r).compute_factored_evals(L, R);
  if (!blinds.empty() && blinds.size() != L.size()) throw std::runtime_error("prove_hiding: one blind per row");
  Fr LZ_blind = Fr::zero();
  for (size_t i = 0; i < blinds.size(); i++) LZ_blind += L[i] * blinds[i];
  Point Cx;
  PolyEvalProof out;
  out.proof = DotProductProofLog::prove(gens.gens, transcript, tape, poly.bound(L), LZ_blind, R, Zr, blind_Zr, Cx, C_Zr);
  return out;
}

// A combining function as lasso_comb_create takes it: 3 ints {op, a, b} per instruction, slots 0..n-1 the inputs,
// instruction j writes slot n + j, the last slot is g; op: 0 a + b, 1 a - b, 2 a * b, 3 a * K[b], 4 a + K[b].
// Interpreted directly, SSA slot by SSA slot (no slot allocation).  Taken as given: the GPU library checks it.
struct Program {
  size_t n;
  std::vector<int32_t> prog;
  std::vector<Fr> K;
  Fr operator()(const Fr* vals) const {
    Fr s[16 + 128];
    const size_t m = prog.size() / 3;
    for (size_t j = 0; j < n; j++) s[j] = vals[j];
    for (size_t j = 0; j < m; j++) {
      const int32_t op = prog[3 * j], a = prog[3 * j + 1], b = prog[3 * j + 2];
      switch (op) {
        case 0: s[n + j] = s[a] + s[b]; break;
        case 1: s[n + j] = s[a] - s[b]; break;
        case 2: s[n + j] = s[a] * s[b]; break;
        case 3: s[n + j] = s[a] * K[b]; break;
        default: s[n + j] = s[a] + K[b]; break;
      }
    }
    return s[n + m - 1];
  }
};
// ark-serialize (compressed) of SumcheckInstanceProof { compressed_polys: Vec<CompressedUniPoly> }
std::vector<uint8_t> ser_sumcheck(const SumcheckInstanceProof& p) {
  std::vector<uint8_t> b;
  put_u64(b, p.compressed_polys.size());
  for (const CompressedUniPoly& c : p.compressed_polys) {
    put_u64(b, c.coeffs_except_linear_term.size());
    for (const Fr& f : c.coeffs_except_linear_term) put_fr(b, f);
  }
  return b;
}

// ---- zero-knowledge sumchecks: DotProductProof (subprotocols/dot_product.rs:11-136) and ZKSumcheckInstanceProof
// (subprotocols/sumcheck.rs:331-447), restated over the MultiCommitGens / batch_commit / commit_scalar of oracle/
MultiCommitGens ldgens(const uint64_t* G, size_t n, const uint64_t* h) {
  const std::vector<Affine> s = ldstream(G, n);
  MultiCommitGens g;
  g.n = n;
  for (const Affine& a : s) g.G.push_back(Point::from_affine(a));
  g.h = Point::from_affine(ldstream(h, 1)[0]);
  return g;
}
Fr dotp(const std::vector<Fr>& a, const std::vector<Fr>& b) {  // compute_dotproduct (dot_product.rs:26-29)
  Fr s = Fr::zero();
  for (size_t i = 0; i < a.size(); i++) s += a[i] * b[i];
  return s;
}
struct DotProductProof {
  Point delta, beta;
  std::vector<Fr> z;
  Fr z_delta, z_beta;
};
// dot_product.rs:31-93
DotProductProof dot_prove(const MultiCommitGens& gens_1, const MultiCommitGens& gens_n, Transcript& transcript,
                          RandomTape& tape, const std::vector<Fr>& x, const Fr& blind_x, const std::vector<Fr>& a,
                          const Fr& y, const Fr& blind_y, Point& Cx, Point& Cy) {
  transcript.append_protocol_name("dot product proof");
  const size_t n = x.size();
  if (a.size() != n || gens_n.n != n || gens_1.n != 1) throw std::runtime_error("dot_prove: lengths");
  const std::vector<Fr> d_vec = tape.random_vector("d_vec", n);
  const Fr r_delta = tape.random_scalar("r_delta");
  const Fr r_beta = tape.random_scalar("r_beta");
  Cx = batch_commit(x.data(), n, blind_x, gens_n);
  transcript.append_point("Cx", Cx);
  Cy = commit_scalar(y, blind_y, gens_1);
  transcript.append_point("Cy", Cy);
  transcript.append_scalars("a", a);
  DotProductProof p;
  p.delta = batch_commit(d_vec.data(), n, r_delta, gens_n);
  transcript.append_point("delta", p.delta);
  p.beta = commit_scalar(dotp(a, d_vec), r_beta, gens_1);
  transcript.append_point("beta", p.beta);
  const Fr c = transcript.challenge_scalar("c");
  for (size_t i = 0; i < n; i++) p.z.push_back(c * x[i] + d_vec[i]);
  p.z_delta = c * blind_x + r_delta;
  p.z_beta = c * blind_y + r_beta;
  return p;
}
// dot_product.rs:95-136
bool dot_verify(const DotProductProof& p, const MultiCommitGens& gens_1, const MultiCommitGens& gens_n,
                Transcript& transcript, const std::vector<Fr>& a, const Point& Cx, const Point& Cy) {
  if (a.size() != gens_n.n || gens_1.n != 1 || p.z.size() != gens_n.n) return false;
  transcript.append_protocol_name("dot product proof");
  transcript.append_point("Cx", Cx);
  transcript.append_point("Cy", Cy);
  transcript.append_scalars("a", a);
  transcript.append_point("delta", p.delta);
  transcript.append_point("beta", p.beta);
  const Fr c = transcript.challenge_scalar("c");
  bool ok = Cx * c + p.delta == batch_commit(p.z.data(), p.z.size(), p.z_delta, gens_n);
  ok &= Cy * c + p.beta == commit_scalar(dotp(p.z, a), p.z_beta, gens_1);
  return ok;
}
void ser_dot(std::vector<uint8_t>& b, const DotProductProof& p) {
  put_point(b, p.delta);
  put_point(b, p.beta);
  put_u64(b, p.z.size());
  for (const Fr& f : p.z) put_fr(b, f);
  put_fr(b, p.z_delta);
  put_fr(b, p.z_beta);
}
DotProductProof read_dot(Reader& rd) {
  DotProductProof p;
  p.delta = rd.point();
  p.beta = rd.point();
  const uint64_t m = rd.u64();
  if (m > (rd.n - rd.at) / 32) rd.ok = false;
  for (uint64_t i = 0; rd.ok && i < m; i++) p.z.push_back(rd.fr());
  p.z_delta = rd.fr();
  p.z_beta = rd.fr();
  return p;
}
struct ZKSumcheckInstanceProof {
  std::vector<Point> comm_polys, comm_evals;
  std::vector<DotProductProof> proofs;
};
std::vector<uint8_t> ser_zk(const ZKSumcheckInstanceProof& p) {
  std::vector<uint8_t> b;
  put_u64(b, p.comm_polys.size());
  for (const Point& q : p.comm_polys) put_point(b, q);
  put_u64(b, p.comm_evals.size());
  for (const Point& q : p.comm_evals) put_point(b, q);
  put_u64(b, p.proofs.size());
  for (const DotProductProof& d : p.proofs) ser_dot(b, d);
  return b;
}
// sumcheck.rs:347-446: false where the reference returns Err or fails an assertion; e = the last comm_eval
bool zk_verify(const ZKSumcheckInstanceProof& p, const Point& comm_claim, size_t num_rounds, size_t degree_bound,
               const MultiCommitGens& gens_1, const MultiCommitGens& gens_n, Transcript& transcript, Point& e,
               std::vector<Fr>& r) {
  if (gens_n.n != degree_bound + 1) return false;
  if (p.comm_polys.size() != num_rounds || p.comm_evals.size() != num_rounds || p.proofs.size() < num_rounds) return false;
  r.clear();
  for (size_t i = 0; i < p.comm_polys.size(); i++) {
    const Point& comm_poly = p.comm_polys[i];
    transcript.append_point("comm_poly", comm_poly);
    const Fr r_i = transcript.challenge_scalar("challenge_nextround");
    const Point& comm_claim_per_round = i == 0 ? comm_claim : p.comm_evals[i - 1];
    const Point& comm_eval = p.comm_evals[i];
    transcript.append_point("comm_claim_per_round", comm_claim_per_round);
    transcript.append_point("comm_eval", comm_eval);
    const std::vector<Fr> w = transcript.challenge_vector("combine_two_claims_to_one", 2);
    const Point comm_target = comm_claim_per_round * w[0] + comm_eval * w[1];
    std::vector<Fr> a_sc(degree_bound + 1, Fr::one()), a_eval(degree_bound + 1, Fr::one()), a(degree_bound + 1);
    a_sc[0] += Fr::one();
    for (size_t j = 1; j < a_eval.size(); j++) a_eval[j] = a_eval[j - 1] * r_i;
    for (size_t j = 0; j < a.size(); j++) a[j] = w[0] * a_sc[j] + w[1] * a_eval[j];
    if (!dot_verify(p.proofs[i], gens_1, gens_n, transcript, a, p.comm_polys[i], comm_target)) return false;
    r.push_back(r_i);
  }
  if (p.comm_evals.empty()) return false;  // the reference indexes comm_evals[len - 1]
  e = p.comm_evals.back();
  return true;
}
// The prover: the round polynomials of prove_arbitrary (oracle/lasso.hpp, restated: the transcript takes commitments
// instead of the polynomials), the tape drawn up front as Spartan's prove_*_zk does (blinds_poly, blinds_evals, then
// each round's DotProductProof draws), each round's transcript steps in the order of zk_verify above
ZKSumcheckInstanceProof zk_prove(std::vector<DensePolynomial>& polys, const Program& g, size_t degree, size_t num_rounds,
                                 const Fr& blind_claim, const MultiCommitGens& gens_1, const MultiCommitGens& gens_n,
                                 Transcript& transcript, RandomTape& tape, std::vector<Fr>& r,
                                 std::vector<Fr>& final_evals, Fr& claim, Point& comm_claim, Fr& blind_eval) {
  const size_t alpha = polys.size(), n = degree + 1;
  const std::vector<Fr> blinds_poly = tape.random_vector("blinds_poly", num_rounds);
  const std::vector<Fr> blinds_evals = tape.random_vector("blinds_evals", num_rounds);
  ZKSumcheckInstanceProof proof;
  Fr claim_j, beta_j = blind_claim;
  r.clear();
  for (size_t round = 0; round < num_rounds; round++) {
    std::vector<Fr> evals(n, Fr::zero());
    const size_t half = polys[0].len / 2;
#pragma omp parallel
    {
      std::vector<Fr> local(n, Fr::zero()), cur(alpha), nxt(alpha);
#pragma omp for nowait
      for (size_t i = 0; i < half; i++) {
        for (size_t j = 0; j < alpha; j++) cur[j] = polys[j][i];
        local[0] += g(cur.data());
        for (size_t j = 0; j < alpha; j++) cur[j] = polys[j][half + i];
        local[1] += g(cur.data());
        for (size_t t = 2; t < n; t++) {
          for (size_t j = 0; j < alpha; j++) nxt[j] = cur[j] + polys[j][half + i] - polys[j][i];
          local[t] += g(nxt.data());
          cur.swap(nxt);
        }
      }
#pragma omp critical
      for (size_t t = 0; t < n; t++) evals[t] += local[t];
    }
    if (round == 0) {
      claim_j = claim = evals[0] + evals[1];
      comm_claim = commit_scalar(claim, blind_claim, gens_1);
    }
    const UniPoly poly = UniPoly::from_evals(evals);
    const Point comm_poly = batch_commit(poly.coeffs.data(), n, blinds_poly[round], gens_n);
    transcript.append_point("comm_poly", comm_poly);
    const Fr r_j = transcript.challenge_scalar("challenge_nextround");
    r.push_back(r_j);
    const Fr eval = poly.evaluate(r_j);
    const Point comm_eval = commit_scalar(eval, blinds_evals[round], gens_1);
    transcript.append_point("comm_claim_per_round", round == 0 ? comm_claim : proof.comm_evals.back());
    transcript.append_point("comm_eval", comm_eval);
    const std::vector<Fr> w = transcript.challenge_vector("combine_two_claims_to_one", 2);
    std::vector<Fr> a(n);
    Fr pw = Fr::one();
    for (size_t j = 0; j < n; j++) {
      a[j] = w[0] * (j == 0 ? Fr::one() + Fr::one() : Fr::one()) + w[1] * pw;
      pw *= r_j;
    }
    const Fr blind_y = w[0] * beta_j + w[1] * blinds_evals[round];
    Point Cx, Cy;
    proof.proofs.push_back(dot_prove(gens_1, gens_n, transcript, tape, poly.coeffs, blinds_poly[round], a,
                                     w[0] * claim_j + w[1] * eval, blind_y, Cx, Cy));
    proof.comm_polys.push_back(comm_poly);
    proof.comm_evals.push_back(comm_eval);
    for (auto& p : polys) p.bound_poly_var_top(r_j);
    claim_j = eval;
    beta_j = blinds_evals[round];
  }
  final_evals.clear();
  for (auto& p : polys) final_evals.push_back(p[0]);
  blind_eval = blinds_evals[num_rounds - 1];
  return proof;
}

// ---- Σ-protocols of committed scalars (subprotocols/zk.rs), restated over commit_scalar of oracle/.  gens has n == 1.
// Proofs serialise as ark-serialize compressed: points, then scalars; ProductProof's z is [F; 5], a fixed-size array
// written with no length prefix (recalled, not checked: no ark-serialize source is at hand).
struct KnowledgeProof {
  Point alpha;
  Fr z1, z2;
};
// zk.rs:23-51
KnowledgeProof knowledge_prove(const MultiCommitGens& g, Transcript& transcript, RandomTape& tape, const Fr& x,
                               const Fr& r, Point& C) {
  transcript.append_protocol_name("knowledge proof");
  const Fr t1 = tape.random_scalar("t1");
  const Fr t2 = tape.random_scalar("t2");
  C = commit_scalar(x, r, g);
  transcript.append_point("C", C);
  KnowledgeProof p;
  p.alpha = commit_scalar(t1, t2, g);
  transcript.append_point("alpha", p.alpha);
  const Fr c = transcript.challenge_scalar("c");
  p.z1 = x * c + t1;
  p.z2 = r * c + t2;
  return p;
}
// zk.rs:53-75
bool knowledge_verify(const KnowledgeProof& p, const MultiCommitGens& g, Transcript& transcript, const Point& C) {
  transcript.append_protocol_name("knowledge proof");
  transcript.append_point("C", C);
  transcript.append_point("alpha", p.alpha);
  const Fr c = transcript.challenge_scalar("c");
  return commit_scalar(p.z1, p.z2, g) == C * c + p.alpha;
}
struct EqualityProof {
  Point alpha;
  Fr z;
};
// zk.rs:89-121
EqualityProof equality_prove(const MultiCommitGens& g, Transcript& transcript, RandomTape& tape, const Fr& v1,
                             const Fr& s1, const Fr& v2, const Fr& s2, Point& C1, Point& C2) {
  transcript.append_protocol_name("equality proof");
  const Fr r = tape.random_scalar("r");
  C1 = commit_scalar(v1, s1, g);
  transcript.append_point("C1", C1);
  C2 = commit_scalar(v2, s2, g);
  transcript.append_point("C2", C2);
  EqualityProof p;
  p.alpha = g.h * r;
  transcript.append_point("alpha", p.alpha);
  const Fr c = transcript.challenge_scalar("c");
  p.z = c * (s1 - s2) + r;
  return p;
}
// zk.rs:123-153
bool equality_verify(const EqualityProof& p, const MultiCommitGens& g, Transcript& transcript, const Point& C1,
                     const Point& C2) {
  transcript.append_protocol_name("equality proof");
  transcript.append_point("C1", C1);
  transcript.append_point("C2", C2);
  transcript.append_point("alpha", p.alpha);
  const Fr c = transcript.challenge_scalar("c");
  return g.h * p.z == (C1 + -C2) * c + p.alpha;
}
struct ProductProof {
  Point alpha, beta, delta;
  Fr z[5];
};
// zk.rs:169-237; delta = b3 X + b5 h over the variable base X, as the reference computes it
ProductProof product_prove(const MultiCommitGens& g, Transcript& transcript, RandomTape& tape, const Fr& x, const Fr& rX,
                           const Fr& y, const Fr& rY, const Fr& z, const Fr& rZ, Point& X, Point& Y, Point& Z) {
  transcript.append_protocol_name("product proof");
  const Fr b1 = tape.random_scalar("b1");
  const Fr b2 = tape.random_scalar("b2");
  const Fr b3 = tape.random_scalar("b3");
  const Fr b4 = tape.random_scalar("b4");
  const Fr b5 = tape.random_scalar("b5");
  X = commit_scalar(x, rX, g);
  transcript.append_point("X", X);
  Y = commit_scalar(y, rY, g);
  transcript.append_point("Y", Y);
  Z = commit_scalar(z, rZ, g);
  transcript.append_point("Z", Z);
  ProductProof p;
  p.alpha = commit_scalar(b1, b2, g);
  transcript.append_point("alpha", p.alpha);
  p.beta = commit_scalar(b3, b4, g);
  transcript.append_point("beta", p.beta);
  p.delta = X * b3 + g.h * b5;
  transcript.append_point("delta", p.delta);
  const Fr c = transcript.challenge_scalar("c");
  p.z[0] = b1 + c * x;
  p.z[1] = b2 + c * rX;
  p.z[2] = b3 + c * y;
  p.z[3] = b4 + c * rY;
  p.z[4] = b5 + c * (rZ - rX * y);
  return p;
}
// zk.rs:239-300 (check_equality: P + c X == z1 G + z2 h, the last one over the bases (X, h))
bool product_verify(const ProductProof& p, const MultiCommitGens& g, Transcript& transcript, const Point& X,
                    const Point& Y, const Point& Z) {
  transcript.append_protocol_name("product proof");
  transcript.append_point("X", X);
  transcript.append_point("Y", Y);
  transcript.append_point("Z", Z);
  transcript.append_point("alpha", p.alpha);
  transcript.append_point("beta", p.beta);
  transcript.append_point("delta", p.delta);
  const Fr c = transcript.challenge_scalar("c");
  bool ok = p.alpha + X * c == commit_scalar(p.z[0], p.z[1], g);
  ok &= p.beta + Y * c == commit_scalar(p.z[2], p.z[3], g);
  ok &= p.delta + Z * c == X * p.z[2] + g.h * p.z[4];
  return ok;
}

}  // namespace

extern "C" {

// ---- ProofTranscript (utils/transcript.rs) and RandomTape (utils/random.rs), one call per method
void* orcd_transcript_new(const char* label) { return new Transcript(label); }
void orcd_transcript_free(void* t) { delete (Transcript*)t; }
void orcd_transcript_append_message(void* t, const char* label, const uint8_t* msg, size_t n) {
  ((Transcript*)t)->append_message(label, msg, n);
}
void orcd_transcript_append_u64(void* t, const char* label, uint64_t x) { ((Transcript*)t)->append_u64(label, x); }
void orcd_transcript_append_protocol_name(void* t, const char* name) { ((Transcript*)t)->append_protocol_name(name); }
void orcd_transcript_append_scalar(void* t, const char* label, const uint64_t* s) {
  ((Transcript*)t)->append_scalar(label, ldfr(s));
}
void orcd_transcript_append_scalars(void* t, const char* label, const uint64_t* s, size_t n) {
  ((Transcript*)t)->append_scalars(label, ldvec(s, n));
}
// points as 32-byte compressed encodings: decompressed, then appended through the oracle's own compression
int orcd_transcript_append_point(void* t, const char* label, const uint8_t* p32) {
  Point q;
  if (!ldpoint(p32, q)) return 1;
  ((Transcript*)t)->append_point(label, q);
  return 0;
}
int orcd_transcript_append_points(void* t, const char* label, const uint8_t* pts, size_t n) {  // transcript.rs:50-56
  std::vector<Point> v(n);
  for (size_t i = 0; i < n; i++)
    if (!ldpoint(pts + 32 * i, v[i])) return 1;
  Transcript& tr = *(Transcript*)t;
  tr.append_message(label, "begin_append_vector");
  for (const Point& q : v) tr.append_point(label, q);
  tr.append_message(label, "end_append_vector");
  return 0;
}
// PolyCommitment::append_to_transcript (dense_mlpoly.rs:281-289) of serialised commitment bytes
int orcd_transcript_append_poly_commitment(void* t, const char* label, const uint8_t* bytes, size_t len) {
  Reader rd{bytes, len};
  PolyCommitment c;
  c.C = rd.points();
  if (!rd.ok || rd.at != len) return 1;
  c.append_to_transcript(label, *(Transcript*)t);
  return 0;
}
void orcd_transcript_challenge_scalar(void* t, const char* label, uint64_t* out) {
  stfr(out, ((Transcript*)t)->challenge_scalar(label));
}
void orcd_transcript_challenge_vector(void* t, const char* label, size_t n, uint64_t* out) {
  std::vector<Fr> v = ((Transcript*)t)->challenge_vector(label, n);
  for (size_t i = 0; i < n; i++) stfr(out + 4 * i, v[i]);
}
void* orcd_tape_new(const char* label, const uint64_t* seed) { return new RandomTape(label, ldfr(seed)); }
void orcd_tape_free(void* t) { delete (RandomTape*)t; }
void orcd_tape_random_vector(void* t, const char* label, size_t n, uint64_t* out) {
  std::vector<Fr> v = ((RandomTape*)t)->random_vector(label, n);
  for (size_t i = 0; i < n; i++) stfr(out + 4 * i, v[i]);
}

// ---- DensePolynomial / PolyCommitmentGens / PolyEvalProof (dense_mlpoly.rs)
// Z: n = 2^nv Montgomery elements; stream: n_points affine generators (G.., Q, h for R = 2^(nv - nv/2))
// commit: out receives the serialised PolyCommitment; returns its length, 0 when the stream is too short or cap too small
size_t orcd_poly_commit(const uint64_t* Z, size_t n, const uint64_t* stream, size_t n_points, uint8_t* out, size_t cap) {
  try {
    DensePolynomial poly(ldvec(Z, n));
    size_t l, r;
    EqPolynomial::compute_factored_lens(poly.num_vars, l, r);
    if (n_points < pow2(r) + 2) return 0;
    PolyCommitmentGens gens = PolyCommitmentGens::make(poly.num_vars, ldstream(stream, n_points));
    std::vector<uint8_t> b = ser_commitment(poly.commit(gens));
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_poly_commit: %s\n", e.what());
    return 0;
  }
}
void orcd_evaluate(const uint64_t* Z, size_t n, const uint64_t* r, uint64_t* out) {
  DensePolynomial poly(ldvec(Z, n));
  stfr(out, poly.evaluate(ldvec(r, poly.num_vars)));
}
// PolyEvalProof::prove on a caller's transcript and tape: returns the proof's length (0 on error); C_Zr_out = the
// compressed C_Zr_prime (Zr * Q + 0 * h)
size_t orcd_poly_prove(const uint64_t* Z, size_t n, const uint64_t* r, const uint64_t* Zr, const uint64_t* stream,
                       size_t n_points, void* transcript, void* tape, uint8_t* out, size_t cap, uint8_t* C_Zr_out) {
  try {
    DensePolynomial poly(ldvec(Z, n));
    size_t l, rr;
    EqPolynomial::compute_factored_lens(poly.num_vars, l, rr);
    if (n_points < pow2(rr) + 2) return 0;
    PolyCommitmentGens gens = PolyCommitmentGens::make(poly.num_vars, ldstream(stream, n_points));
    PolyEvalProof proof = PolyEvalProof::prove(poly, ldvec(r, poly.num_vars), ldfr(Zr), gens, *(Transcript*)transcript,
                                               *(RandomTape*)tape);
    commit_scalar(ldfr(Zr), Fr::zero(), gens.gens.gens_1).compress(C_Zr_out);
    std::vector<uint8_t> b = ser_proof(proof);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_poly_prove: %s\n", e.what());
    return 0;
  }
}
// PolyEvalProof::verify_plain (dense_mlpoly.rs:388-400) of serialised bytes: 0 accepted, 1 rejected, 2 the commitment
// or the proof does not parse
int orcd_poly_verify(const uint64_t* stream, size_t n_points, size_t nv, const uint8_t* comm, size_t comm_len,
                     const uint8_t* proof, size_t proof_len, const uint64_t* r, const uint64_t* Zr, void* transcript) {
  size_t l, rr;
  EqPolynomial::compute_factored_lens(nv, l, rr);
  if (n_points < pow2(rr) + 2) return 2;
  PolyCommitmentGens gens = PolyCommitmentGens::make(nv, ldstream(stream, n_points));
  Reader rc{comm, comm_len};
  PolyCommitment c;
  c.C = rc.points();
  if (!rc.ok || rc.at != comm_len || c.C.size() != pow2(l)) return 2;
  PolyEvalProof p;
  if (!read_poly_eval_proof(proof, proof_len, p)) return 2;
  return p.verify_plain(gens, *(Transcript*)transcript, ldvec(r, nv), ldfr(Zr), c) ? 0 : 1;
}
// The hiding commitment: with a tape (non-null) its L = 2^(nv/2) blinds are drawn as random_vector("poly_blinds", L)
// and written to blinds (L x 4 limbs); without one, blinds holds them.  Returns the commitment's length, 0 on error.
size_t orcd_poly_commit_hiding(const uint64_t* Z, size_t n, const uint64_t* stream, size_t n_points, void* tape,
                               uint64_t* blinds, uint8_t* out, size_t cap) {
  try {
    DensePolynomial poly(ldvec(Z, n));
    size_t l, r;
    EqPolynomial::compute_factored_lens(poly.num_vars, l, r);
    if (n_points < pow2(r) + 2) return 0;
    PolyCommitmentGens gens = PolyCommitmentGens::make(poly.num_vars, ldstream(stream, n_points));
    std::vector<Fr> bl = tape ? ((RandomTape*)tape)->random_vector("poly_blinds", pow2(l)) : ldvec(blinds, pow2(l));
    for (size_t i = 0; i < bl.size(); i++) stfr(blinds + 4 * i, bl[i]);
    std::vector<uint8_t> b = ser_commitment(commit_hiding(poly, gens, bl));
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_poly_commit_hiding: %s\n", e.what());
    return 0;
  }
}
// PolyEvalProof::prove with blinds (n_blinds == 0: None) and blind_Zr (null: None) on a caller's transcript and tape:
// returns the proof's length (0 on error); C_Zr_out = the compressed Zr * Q + blind_Zr * h
size_t orcd_poly_prove_hiding(const uint64_t* Z, size_t n, const uint64_t* blinds, size_t n_blinds, const uint64_t* r,
                              const uint64_t* Zr, const uint64_t* blind_Zr, const uint64_t* stream, size_t n_points,
                              void* transcript, void* tape, uint8_t* out, size_t cap, uint8_t* C_Zr_out) {
  try {
    DensePolynomial poly(ldvec(Z, n));
    size_t l, rr;
    EqPolynomial::compute_factored_lens(poly.num_vars, l, rr);
    if (n_points < pow2(rr) + 2) return 0;
    PolyCommitmentGens gens = PolyCommitmentGens::make(poly.num_vars, ldstream(stream, n_points));
    Point C_Zr;
    PolyEvalProof proof = prove_hiding(poly, ldvec(blinds, n_blinds), ldvec(r, poly.num_vars), ldfr(Zr),
                                       blind_Zr ? ldfr(blind_Zr) : Fr::zero(), gens, *(Transcript*)transcript,
                                       *(RandomTape*)tape, C_Zr);
    C_Zr.compress(C_Zr_out);
    std::vector<uint8_t> b = ser_proof(proof);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_poly_prove_hiding: %s\n", e.what());
    return 0;
  }
}
// PolyEvalProof::verify (dense_mlpoly.rs:361-386) of serialised bytes against a compressed C_Zr: 0 accepted,
// 1 rejected, 2 the commitment, the proof or C_Zr does not parse
int orcd_poly_verify_czr(const uint64_t* stream, size_t n_points, size_t nv, const uint8_t* comm, size_t comm_len,
                         const uint8_t* proof, size_t proof_len, const uint64_t* r, const uint8_t* C_Zr, void* transcript) {
  size_t l, rr;
  EqPolynomial::compute_factored_lens(nv, l, rr);
  if (n_points < pow2(rr) + 2) return 2;
  PolyCommitmentGens gens = PolyCommitmentGens::make(nv, ldstream(stream, n_points));
  Reader rc{comm, comm_len};
  PolyCommitment c;
  c.C = rc.points();
  if (!rc.ok || rc.at != comm_len || c.C.size() != pow2(l)) return 2;
  PolyEvalProof p;
  Point czr;
  if (!read_poly_eval_proof(proof, proof_len, p) || !ldpoint(C_Zr, czr)) return 2;
  return p.verify(gens, *(Transcript*)transcript, ldvec(r, nv), czr, c) ? 0 : 1;
}

// ---- SumcheckInstanceProof (subprotocols/sumcheck.rs)
// prove_arbitrary on copies of polys (k x len Montgomery elements, row-major) with the program interpreted on the host,
// on a caller's transcript.  out: the serialised proof (returns its length, 0 on error); r_out: num_rounds challenges;
// final_out: k values; claim_out: e_0 + e_1 of the first round; round_evals_out (may be null): num_rounds x (degree + 1)
// evaluations of the round polynomials at 0..degree.
size_t orcd_sumcheck_prove(const uint64_t* polys, size_t k, size_t len, size_t num_rounds, const int32_t* prog, size_t n_ops,
                           const uint64_t* K, size_t n_k, size_t degree, void* transcript, uint8_t* out, size_t cap,
                           uint64_t* r_out, uint64_t* final_out, uint64_t* claim_out, uint64_t* round_evals_out) {
  try {
    std::vector<DensePolynomial> ps;
    for (size_t j = 0; j < k; j++) ps.emplace_back(ldvec(polys + 4 * len * j, len));
    const Program g{k, std::vector<int32_t>(prog, prog + 3 * n_ops), ldvec(K, n_k)};
    std::vector<Fr> r, final_evals;
    std::vector<std::vector<Fr>> rounds;
    SumcheckInstanceProof proof = SumcheckInstanceProof::prove_arbitrary(
        num_rounds, ps, [&](const Fr* v) { return g(v); }, degree, *(Transcript*)transcript, r, final_evals, nullptr, &rounds);
    std::vector<uint8_t> b = ser_sumcheck(proof);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    for (size_t j = 0; j < num_rounds; j++) stfr(r_out + 4 * j, r[j]);
    for (size_t j = 0; j < k; j++) stfr(final_out + 4 * j, final_evals[j]);
    stfr(claim_out, rounds[0][0] + rounds[0][1]);
    if (round_evals_out)
      for (size_t j = 0; j < num_rounds; j++)
        for (size_t t = 0; t <= degree; t++) stfr(round_evals_out + 4 * (j * (degree + 1) + t), rounds[j][t]);
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_sumcheck_prove: %s\n", e.what());
    return 0;
  }
}
// SumcheckInstanceProof::verify (sumcheck.rs:286-328) of serialised bytes: 0 accepted (e_out = the final claim,
// r_out = num_rounds challenges), 1 rejected, 2 the bytes do not parse
int orcd_sumcheck_verify(const uint8_t* bytes, size_t n, const uint64_t* claim, size_t num_rounds, size_t degree,
                         void* transcript, uint64_t* e_out, uint64_t* r_out) {
  Reader rd{bytes, n};
  SumcheckInstanceProof p;
  const uint64_t rounds = rd.u64();
  for (uint64_t j = 0; rd.ok && j < rounds; j++) {
    const uint64_t m = rd.u64();
    if (m > (n - rd.at) / 32) rd.ok = false;
    CompressedUniPoly c;
    for (uint64_t i = 0; rd.ok && i < m; i++) c.coeffs_except_linear_term.push_back(rd.fr());
    if (c.coeffs_except_linear_term.empty()) rd.ok = false;
    p.compressed_polys.push_back(c);
  }
  if (!rd.ok || rd.at != n) return 2;
  Fr e;
  std::vector<Fr> r;
  if (!p.verify(ldfr(claim), num_rounds, degree, *(Transcript*)transcript, e, r)) return 1;
  stfr(e_out, e);
  for (size_t j = 0; j < num_rounds; j++) stfr(r_out + 4 * j, r[j]);
  return 0;
}
// SumcheckInstanceProof::prove_cubic_batched (sumcheck.rs:26-135) on copies of n pairs (A, B: n x len elements each,
// row-major) and C, with the caller's claim and coefficients, on a caller's transcript.  out: the serialised proof
// (returns its length, 0 on error); r_out: num_rounds challenges; finals_out: A_0.., B_0.., C after the binds (2n + 1).
size_t orcd_cubic_prove(const uint64_t* A, const uint64_t* B, size_t n, const uint64_t* Cz, size_t len, const uint64_t* coeffs,
                        const uint64_t* claim, size_t num_rounds, void* transcript, uint8_t* out, size_t cap, uint64_t* r_out,
                        uint64_t* finals_out) {
  try {
    std::vector<DensePolynomial> pa, pb;
    for (size_t k = 0; k < n; k++) {
      pa.emplace_back(ldvec(A + 4 * len * k, len));
      pb.emplace_back(ldvec(B + 4 * len * k, len));
    }
    DensePolynomial pc(ldvec(Cz, len));
    std::vector<DensePolynomial*> va, vb;
    for (size_t k = 0; k < n; k++) {
      va.push_back(&pa[k]);
      vb.push_back(&pb[k]);
    }
    std::vector<Fr> r, fa, fb;
    Fr fc;
    SumcheckInstanceProof proof = SumcheckInstanceProof::prove_cubic_batched(
        ldfr(claim), num_rounds, va, vb, pc, ldvec(coeffs, n), *(Transcript*)transcript, r, fa, fb, fc);
    std::vector<uint8_t> b = ser_sumcheck(proof);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    for (size_t j = 0; j < num_rounds; j++) stfr(r_out + 4 * j, r[j]);
    for (size_t k = 0; k < n; k++) {
      stfr(finals_out + 4 * k, fa[k]);
      stfr(finals_out + 4 * (n + k), fb[k]);
    }
    stfr(finals_out + 8 * n, fc);
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_cubic_prove: %s\n", e.what());
    return 0;
  }
}
// out[i] = g(polys[0][i], .., polys[k-1][i]) (k x len Montgomery elements, row-major), the program interpreted on the host
void orcd_comb_map(const uint64_t* polys, size_t k, size_t len, const int32_t* prog, size_t n_ops, const uint64_t* K, size_t n_k,
                   uint64_t* out) {
  const Program g{k, std::vector<int32_t>(prog, prog + 3 * n_ops), ldvec(K, n_k)};
  std::vector<Fr> vals(k);
  for (size_t i = 0; i < len; i++) {
    for (size_t j = 0; j < k; j++) vals[j] = ldfr(polys + 4 * (j * len + i));
    stfr(out + 4 * i, g(vals.data()));
  }
}

// ---- GrandProductCircuit / BatchedGrandProductArgument (subprotocols/grand_product.rs)
// GrandProductCircuit::new over each of n polynomials (n x len Montgomery elements, row-major, len >= 2), then
// BatchedGrandProductArgument::prove on a caller's transcript (the products are not appended to it: the caller's
// protocol does that).  out: the serialised proof (returns its length, 0 on error); products_out: n evaluate() values;
// rand_out: log2(len) values; claims_out: n final claims_to_verify.
size_t orcd_gp_prove(const uint64_t* polys, size_t n, size_t len, void* transcript, uint8_t* out, size_t cap,
                     uint64_t* products_out, uint64_t* rand_out, uint64_t* claims_out) {
  try {
    std::vector<GrandProductCircuit> cs;
    for (size_t k = 0; k < n; k++) cs.emplace_back(DensePolynomial(ldvec(polys + 4 * len * k, len)));
    std::vector<GrandProductCircuit*> ptrs;
    for (size_t k = 0; k < n; k++) {
      stfr(products_out + 4 * k, cs[k].evaluate());
      ptrs.push_back(&cs[k]);
    }
    std::vector<Fr> rand;
    const BatchedGrandProductArgument p = BatchedGrandProductArgument::prove(ptrs, *(Transcript*)transcript, rand);
    ByteWriter w;
    ser(w, p);
    if (w.b.size() > cap) return 0;
    memcpy(out, w.b.data(), w.b.size());
    for (size_t j = 0; j < rand.size(); j++) stfr(rand_out + 4 * j, rand[j]);
    const LayerProofBatched& last = p.proof.back();  // grand_product.rs:189-195, rand[0] = the last r_layer
    for (size_t k = 0; k < n; k++)
      stfr(claims_out + 4 * k, last.claims_prod_left[k] + rand[0] * (last.claims_prod_right[k] - last.claims_prod_left[k]));
    return w.b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_gp_prove: %s\n", e.what());
    return 0;
  }
}
// BatchedGrandProductArgument::verify (grand_product.rs:203-261) of serialised bytes against n products of circuits of
// num_vars variables: 0 accepted (claims_out = the n final claims, rand_out = num_vars values), 1 rejected, 2 the bytes
// do not parse
int orcd_gp_verify(const uint8_t* bytes, size_t nbytes, const uint64_t* products, size_t n, size_t num_vars, void* transcript,
                   uint64_t* claims_out, uint64_t* rand_out) {
  Reader rd{bytes, nbytes};
  BatchedGrandProductArgument p;
  auto frs = [&]() {
    const uint64_t m = rd.u64();
    std::vector<Fr> v;
    if (m > (nbytes - rd.at) / 32) rd.ok = false;
    for (uint64_t i = 0; rd.ok && i < m; i++) v.push_back(rd.fr());
    return v;
  };
  const uint64_t layers = rd.u64();
  if (layers > nbytes) rd.ok = false;
  for (uint64_t l = 0; rd.ok && l < layers; l++) {
    LayerProofBatched lp;
    const uint64_t rounds = rd.u64();
    if (rounds > nbytes) rd.ok = false;
    for (uint64_t j = 0; rd.ok && j < rounds; j++) {
      CompressedUniPoly c;
      c.coeffs_except_linear_term = frs();
      if (c.coeffs_except_linear_term.empty()) rd.ok = false;
      lp.proof.compressed_polys.push_back(c);
    }
    lp.claims_prod_left = frs();
    lp.claims_prod_right = frs();
    p.proof.push_back(std::move(lp));
  }
  if (!rd.ok || rd.at != nbytes) return 2;
  std::vector<Fr> claims, rand;
  if (!p.verify(ldvec(products, n), pow2(num_vars), *(Transcript*)transcript, claims, rand)) return 1;
  for (size_t k = 0; k < n; k++) stfr(claims_out + 4 * k, claims[k]);
  for (size_t j = 0; j < rand.size(); j++) stfr(rand_out + 4 * j, rand[j]);
  return 0;
}

// ---- DensePolynomial::merge and CombinedTableEvalProof (dense_mlpoly.rs:251-261, subtables/mod.rs:225-375)
// merge of k polynomials (polys: their evaluations one after another, lens[j] of polynomial j): out receives the merged
// evaluations (cap elements); returns their count, 0 when cap is too small
size_t orcd_merge(const uint64_t* polys, const size_t* lens, size_t k, uint64_t* out, size_t cap) {
  std::vector<DensePolynomial> ps;
  size_t at = 0;
  for (size_t j = 0; j < k; j++) {
    ps.emplace_back(ldvec(polys + 4 * at, lens[j]));
    at += lens[j];
  }
  const DensePolynomial m = DensePolynomial::merge(ps);
  if (m.len > cap) return 0;
  for (size_t i = 0; i < m.len; i++) stfr(out + 4 * i, m.Z[i]);
  return m.len;
}
// CombinedTableEvalProof::prove over the polynomial Z (n = 2^nv elements) for n_evals claims at r (nv - log2 of the
// padded count coordinates), on a caller's transcript and tape: returns the proof's length (0 on error)
size_t orcd_combined_eval_prove(const uint64_t* Z, size_t n, const uint64_t* evals, size_t n_evals, const uint64_t* r,
                                size_t r_len, const uint64_t* stream, size_t n_points, void* transcript, void* tape,
                                uint8_t* out, size_t cap) {
  try {
    DensePolynomial poly(ldvec(Z, n));
    if (n_evals == 0 || poly.num_vars != r_len + log_2(next_power_of_two(n_evals))) return 0;
    size_t l, rr;
    EqPolynomial::compute_factored_lens(poly.num_vars, l, rr);
    if (n_points < pow2(rr) + 2) return 0;
    PolyCommitmentGens gens = PolyCommitmentGens::make(poly.num_vars, ldstream(stream, n_points));
    const CombinedTableEvalProof p = CombinedTableEvalProof::prove(poly, ldvec(evals, n_evals), ldvec(r, r_len), gens,
                                                                   *(Transcript*)transcript, *(RandomTape*)tape);
    std::vector<uint8_t> b = ser_proof(p.proof_table_eval);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_combined_eval_prove: %s\n", e.what());
    return 0;
  }
}
// CombinedTableEvalProof::verify (subtables/mod.rs:315-375) of serialised bytes against the serialised commitment of a
// polynomial of nv variables: 0 accepted, 1 rejected, 2 the commitment or the proof does not parse or nv does not fit
int orcd_combined_eval_verify(const uint64_t* stream, size_t n_points, size_t nv, const uint8_t* comm, size_t comm_len,
                              const uint8_t* proof, size_t proof_len, const uint64_t* evals, size_t n_evals,
                              const uint64_t* r, size_t r_len, void* transcript) {
  if (n_evals == 0 || nv != r_len + log_2(next_power_of_two(n_evals))) return 2;
  size_t l, rr;
  EqPolynomial::compute_factored_lens(nv, l, rr);
  if (n_points < pow2(rr) + 2) return 2;
  PolyCommitmentGens gens = PolyCommitmentGens::make(nv, ldstream(stream, n_points));
  Reader rc{comm, comm_len};
  PolyCommitment c;
  c.C = rc.points();
  if (!rc.ok || rc.at != comm_len || c.C.size() != pow2(l)) return 2;
  Reader rp{proof, proof_len};
  CombinedTableEvalProof p;
  p.proof_table_eval.proof.bullet_reduction_proof.L_vec = rp.points();
  p.proof_table_eval.proof.bullet_reduction_proof.R_vec = rp.points();
  p.proof_table_eval.proof.delta = rp.point();
  p.proof_table_eval.proof.beta = rp.point();
  p.proof_table_eval.proof.z1 = rp.fr();
  p.proof_table_eval.proof.z2 = rp.fr();
  if (!rp.ok || rp.at != proof_len) return 2;
  return p.verify(ldvec(r, r_len), ldvec(evals, n_evals), gens, c, *(Transcript*)transcript) ? 0 : 1;
}

// ---- SparsePolynomialEvaluationProof on a caller's transcript and tape (surge.rs:70-82, 118-271), built-in strategies
// SparsePolynomialCommitment::append_to_transcript of lasso_commit-shaped bytes: 0 absorbed, 1 they do not parse (nothing
// is absorbed then)
int orcd_sparse_append_commitment(void* t, const uint8_t* bytes, size_t len) {
  SparsePolynomialCommitment c;
  if (!read_sparse_commitment(bytes, len, c)) return 1;
  append_sparse_commitment(c, *(Transcript*)t);
  return 0;
}
// Densify n x C indices, commit (comm_out: serialize_commitment's bytes, comm_cap) and prove at r on a caller's
// transcript and tape: returns the proof's length (0 on error); claim_out = the claimed evaluation
size_t orcd_sparse_prove(int kind, size_t C, size_t log_m, size_t log_r, const uint64_t* indices, size_t n, const uint64_t* r,
                         const uint64_t* stream, size_t n_points, void* transcript, void* tape, uint8_t* out, size_t cap,
                         uint8_t* comm_out, size_t comm_cap, uint64_t* claim_out) {
  try {
    const Strategy S{kind, C, log_m, log_r};
    std::vector<std::vector<size_t>> idx(n, std::vector<size_t>(C));
    for (size_t j = 0; j < n; j++)
      for (size_t i = 0; i < C; i++) idx[j][i] = indices[j * C + i];
    DensifiedRepresentation dense = DensifiedRepresentation::from_lookup_indices(idx, C, log_m);
    if (n_points < SparsePolyCommitmentGens::needs_points(C, dense.s, S.num_memories(), log_m)) return 0;
    SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(C, dense.s, S.num_memories(), log_m, ldstream(stream, n_points));
    const std::vector<uint8_t> cb = serialize_commitment(densified_commit(dense, pg));
    const SparsePolynomialEvaluationProof p = SparsePolynomialEvaluationProof::prove(
        S, dense, ldvec(r, ark_log2(dense.s)), pg, *(Transcript*)transcript, *(RandomTape*)tape);
    const std::vector<uint8_t> b = serialize_proof(p);
    if (b.size() > cap || cb.size() > comm_cap) return 0;
    memcpy(out, b.data(), b.size());
    memcpy(comm_out, cb.data(), cb.size());
    stfr(claim_out, p.claimed_evaluation);
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_sparse_prove: %s\n", e.what());
    return 0;
  }
}
// SparsePolynomialEvaluationProof::verify of serialised bytes against serialised commitment bytes, on a caller's
// transcript: 0 accepted, 1 rejected, 2 the bytes do not parse or the generator stream is too short
int orcd_sparse_verify(int kind, size_t C, size_t log_m, size_t log_r, const uint64_t* stream, size_t n_points,
                       const uint8_t* comm, size_t comm_len, const uint8_t* proof, size_t proof_len, const uint64_t* r,
                       void* transcript) {
  const Strategy S{kind, C, log_m, log_r};
  SparsePolynomialCommitment c;
  SparsePolynomialEvaluationProof p;
  if (!read_sparse_commitment(comm, comm_len, c) || !read_sparse_proof(proof, proof_len, S.num_memories(), C, p)) return 2;
  if (n_points < SparsePolyCommitmentGens::needs_points(C, c.s, S.num_memories(), log_m)) return 2;
  SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(C, c.s, S.num_memories(), log_m, ldstream(stream, n_points));
  return p.verify(S, c, ldvec(r, ark_log2(c.s)), pg, *(Transcript*)transcript) ? 0 : 1;
}


// ---- polynomials derived from a caller's: k sequential calls of the oracle's bound_poly_var_top / bound_poly_var_bot
// (dense_mlpoly.rs:209-225), r[0] first; split (dense_mlpoly.rs:101-107) as the two copies it makes; new_padded
// (dense_mlpoly.rs:75-87).  out receives the result's evaluations in natural order.
void orcd_poly_bind_top(const uint64_t* Z, size_t len, const uint64_t* r, size_t k, uint64_t* out) {
  DensePolynomial p(ldvec(Z, len));
  for (size_t j = 0; j < k; j++) p.bound_poly_var_top(ldfr(r + 4 * j));
  for (size_t i = 0; i < p.len; i++) stfr(out + 4 * i, p[i]);
}
void orcd_poly_bind_bot(const uint64_t* Z, size_t len, const uint64_t* r, size_t k, uint64_t* out) {
  DensePolynomial p(ldvec(Z, len));
  for (size_t j = 0; j < k; j++) p.bound_poly_var_bot(ldfr(r + 4 * j));
  for (size_t i = 0; i < p.len; i++) stfr(out + 4 * i, p[i]);
}
void orcd_poly_split(const uint64_t* Z, size_t len, size_t idx, uint64_t* lo, uint64_t* hi) {
  const DensePolynomial p(ldvec(Z, len));
  const DensePolynomial a(std::vector<Fr>(p.Z.begin(), p.Z.begin() + idx)), b(std::vector<Fr>(p.Z.begin() + idx, p.Z.begin() + 2 * idx));
  for (size_t i = 0; i < idx; i++) {
    stfr(lo + 4 * i, a[i]);
    stfr(hi + 4 * i, b[i]);
  }
}
// -> the padded length; out has room for it
size_t orcd_poly_new_padded(const uint64_t* Z, size_t len, uint64_t* out) {
  const DensePolynomial p = DensePolynomial::new_padded(ldvec(Z, len));
  for (size_t i = 0; i < p.len; i++) stfr(out + 4 * i, p[i]);
  return p.len;
}

// ---- MemoryCheckingProof on a caller's transcript and tape (memory_checking.rs:26-147), built-in strategies.
// indices: n x C; the densified representation, its commitment (comm_out, serialize_commitment's bytes) and the
// combined-table commitment to the lookup polynomials (derefs_out, a PolyCommitment) are made as
// SparsePolynomialEvaluationProof::prove makes them.  r == null: MemoryCheckingProof::prove at (gamma, tau) on the
// transcript as it is.  r != null: gamma and tau are ignored, and the steps of surge.rs:129-186 run first on the
// transcript and the tape (the proof's prefix, not returned), with (gamma, tau) = challenge_vector("challenge_r_hash", 2)
// as surge.rs:188 draws them.  Returns the length of the serialised proof in out (0 on error); *comm_len and
// *derefs_len receive the commitments' lengths.
size_t orcd_memory_check_prove(int kind, size_t C, size_t log_m, size_t log_r, const uint64_t* indices, size_t n,
                               const uint64_t* gamma, const uint64_t* tau, const uint64_t* r, const uint64_t* stream,
                               size_t n_points, void* transcript, void* tape, uint8_t* out, size_t cap, uint8_t* comm_out,
                               size_t comm_cap, size_t* comm_len, uint8_t* derefs_out, size_t derefs_cap,
                               size_t* derefs_len) {
  try {
    const Strategy S{kind, C, log_m, log_r};
    std::vector<std::vector<size_t>> idx(n, std::vector<size_t>(C));
    for (size_t j = 0; j < n; j++)
      for (size_t i = 0; i < C; i++) idx[j][i] = indices[j * C + i];
    DensifiedRepresentation dense = DensifiedRepresentation::from_lookup_indices(idx, C, log_m);
    if (n_points < SparsePolyCommitmentGens::needs_points(C, dense.s, S.num_memories(), log_m)) return 0;
    SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(C, dense.s, S.num_memories(), log_m, ldstream(stream, n_points));
    const std::vector<uint8_t> cb = serialize_commitment(densified_commit(dense, pg));
    Subtables subtables(S, dense.dim_usize, dense.s);
    const PolyCommitment comm_derefs = subtables.commit(pg.gens_derefs);
    const std::vector<uint8_t> db = ser_commitment(comm_derefs);
    Transcript& T = *(Transcript*)transcript;
    RandomTape& tp = *(RandomTape*)tape;
    Fr g = ldfr(gamma), t = ldfr(tau);
    if (r) {  // surge.rs:129-188 with the oracle's own steps, as SparsePolynomialEvaluationProof::prove runs them
      T.append_protocol_name("Lasso SparsePolynomialEvaluationProof");
      append_combined_table_commitment(comm_derefs, "comm_poly_row_col_ops_val", T);
      EqPolynomial eq(ldvec(r, ark_log2(dense.s)));
      T.append_scalar("claim_eval_scalar_product", subtables.compute_sumcheck_claim(eq));
      std::vector<DensePolynomial> combined;
      for (auto& p : subtables.lookup_polys) combined.push_back(p.clone());
      combined.emplace_back(eq.evals());
      std::vector<Fr> r_z, final_evals, eval_derefs;
      SumcheckInstanceProof::prove_arbitrary(
          log_2(dense.s), combined, [&](const Fr* v) { return S.combine_lookups_eq(v); }, S.sumcheck_poly_degree(), T,
          r_z, final_evals);
      for (auto& p : subtables.lookup_polys) eval_derefs.push_back(p.evaluate(r_z));
      CombinedTableEvalProof::prove(subtables.combined_poly, eval_derefs, r_z, pg.gens_derefs, T, tp);
      const std::vector<Fr> r_hash = T.challenge_vector("challenge_r_hash", 2);
      g = r_hash[0];
      t = r_hash[1];
    }
    const MemoryCheckingProof mc = MemoryCheckingProof::prove(dense, g, t, subtables, pg, T, tp);
    ByteWriter w;  // field order: memory_checking.rs:26-37, 655-660, 313-329
    for (auto& e : mc.proof_prod_layer.grand_product_evals)
      for (int k = 0; k < 4; k++) w.fr(e[k]);
    ser(w, mc.proof_prod_layer.proof_mem);
    ser(w, mc.proof_prod_layer.proof_ops);
    const auto& hl = mc.proof_hash_layer;
    w.arr_fr(hl.eval_dim);
    w.arr_fr(hl.eval_read);
    w.arr_fr(hl.eval_final);
    w.arr_fr(hl.eval_derefs);
    ser(w, hl.proof_ops.proof);
    ser(w, hl.proof_mem.proof);
    ser(w, hl.proof_derefs.proof_table_eval.proof);
    if (w.b.size() > cap || cb.size() > comm_cap || db.size() > derefs_cap) return 0;
    memcpy(out, w.b.data(), w.b.size());
    memcpy(comm_out, cb.data(), cb.size());
    memcpy(derefs_out, db.data(), db.size());
    *comm_len = cb.size();
    *derefs_len = db.size();
    return w.b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_memory_check_prove: %s\n", e.what());
    return 0;
  }
}
// MemoryCheckingProof::verify (memory_checking.rs:85-147) of serialised bytes at (gamma, tau) against the two
// commitments orcd_memory_check_prove returns, on a caller's transcript: 0 accepted, 1 rejected, 2 the bytes do not
// parse or the generator stream is too short
int orcd_memory_check_verify(int kind, size_t C, size_t log_m, size_t log_r, const uint64_t* stream, size_t n_points,
                             const uint8_t* comm, size_t comm_len, const uint8_t* derefs, size_t derefs_len,
                             const uint8_t* proof, size_t proof_len, const uint64_t* gamma, const uint64_t* tau,
                             void* transcript) {
  const Strategy S{kind, C, log_m, log_r};
  const size_t alpha = S.num_memories();
  SparsePolynomialCommitment c;
  if (!read_sparse_commitment(comm, comm_len, c)) return 2;
  Reader rc{derefs, derefs_len};
  PolyCommitment comm_derefs;
  comm_derefs.C = rc.points();
  if (!rc.ok || rc.at != derefs_len) return 2;
  Reader rd{proof, proof_len};
  MemoryCheckingProof mc;
  auto& pl = mc.proof_prod_layer;
  for (size_t i = 0; rd.ok && i < alpha; i++) {
    std::array<Fr, 4> e;
    for (int k = 0; k < 4; k++) e[k] = rd.fr();
    pl.grand_product_evals.push_back(e);
  }
  pl.proof_mem = read_gpa(rd);
  pl.proof_ops = read_gpa(rd);
  auto& hl = mc.proof_hash_layer;
  hl.eval_dim = read_frs(rd, C);
  hl.eval_read = read_frs(rd, C);
  hl.eval_final = read_frs(rd, C);
  hl.eval_derefs = read_frs(rd, alpha);
  hl.proof_ops.proof = read_dpl(rd);
  hl.proof_mem.proof = read_dpl(rd);
  hl.proof_derefs.proof_table_eval.proof = read_dpl(rd);
  if (!rd.ok || rd.at != proof_len) return 2;
  if (n_points < SparsePolyCommitmentGens::needs_points(C, c.s, alpha, log_m)) return 2;
  SparsePolyCommitmentGens pg = SparsePolyCommitmentGens::make(C, c.s, alpha, log_m, ldstream(stream, n_points));
  return mc.verify(S, c, comm_derefs, pg, ldfr(gamma), ldfr(tau), c.s, *(Transcript*)transcript) ? 0 : 1;
}

// ---- zero-knowledge sumchecks.  A MultiCommitGens is (G: n affine points, h: one), 64 bytes per point.
// Commitments::batch_commit (commitments.rs:84-93) -> out (32 bytes compressed)
void orcd_mc_commit(const uint64_t* G, size_t n, const uint64_t* h, const uint64_t* scalars, const uint64_t* blind,
                    uint8_t* out) {
  const std::vector<Fr> s = ldvec(scalars, n);
  batch_commit(s.data(), n, ldfr(blind), ldgens(G, n, h)).compress(out);
}
// DotProductProof::prove (dot_product.rs:31-93) on a caller's transcript and tape: returns the proof's length (0 on
// error); Cx_out, Cy_out = the compressed commitments returned alongside
size_t orcd_dot_prove(const uint64_t* G1, const uint64_t* h1, const uint64_t* Gn, size_t n, const uint64_t* hn,
                      void* transcript, void* tape, const uint64_t* x, const uint64_t* blind_x, const uint64_t* a,
                      const uint64_t* y, const uint64_t* blind_y, uint8_t* out, size_t cap, uint8_t* Cx_out,
                      uint8_t* Cy_out) {
  try {
    Point Cx, Cy;
    const DotProductProof p = dot_prove(ldgens(G1, 1, h1), ldgens(Gn, n, hn), *(Transcript*)transcript,
                                        *(RandomTape*)tape, ldvec(x, n), ldfr(blind_x), ldvec(a, n), ldfr(y),
                                        ldfr(blind_y), Cx, Cy);
    std::vector<uint8_t> b;
    ser_dot(b, p);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    Cx.compress(Cx_out);
    Cy.compress(Cy_out);
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_dot_prove: %s\n", e.what());
    return 0;
  }
}
// DotProductProof::verify (dot_product.rs:95-136) of serialised bytes: 0 accepted, 1 rejected, 2 the bytes or a
// commitment do not parse
int orcd_dot_verify(const uint64_t* G1, const uint64_t* h1, const uint64_t* Gn, size_t n, const uint64_t* hn,
                    const uint8_t* proof, size_t proof_len, const uint64_t* a, const uint8_t* Cx, const uint8_t* Cy,
                    void* transcript) {
  Reader rd{proof, proof_len};
  const DotProductProof p = read_dot(rd);
  Point cx, cy;
  if (!rd.ok || rd.at != proof_len || !ldpoint(Cx, cx) || !ldpoint(Cy, cy)) return 2;
  return dot_verify(p, ldgens(G1, 1, h1), ldgens(Gn, n, hn), *(Transcript*)transcript, ldvec(a, n), cx, cy) ? 0 : 1;
}
// The ZK sumcheck prover of zk_prove on copies of polys (k x len Montgomery elements, row-major) with the program
// interpreted on the host; gens_n has degree + 1 points.  out: the serialised ZKSumcheckInstanceProof (returns its
// length, 0 on error); r_out: num_rounds challenges; final_out: k values; claim_out; comm_claim_out (32 bytes);
// blind_eval_out.
size_t orcd_zk_prove(const uint64_t* polys, size_t k, size_t len, size_t num_rounds, const int32_t* prog, size_t n_ops,
                     const uint64_t* K, size_t n_k, size_t degree, const uint64_t* blind_claim, const uint64_t* G1,
                     const uint64_t* h1, const uint64_t* Gn, const uint64_t* hn, void* transcript, void* tape,
                     uint8_t* out, size_t cap, uint64_t* r_out, uint64_t* final_out, uint64_t* claim_out,
                     uint8_t* comm_claim_out, uint64_t* blind_eval_out) {
  try {
    std::vector<DensePolynomial> ps;
    for (size_t j = 0; j < k; j++) ps.emplace_back(ldvec(polys + 4 * len * j, len));
    const Program g{k, std::vector<int32_t>(prog, prog + 3 * n_ops), ldvec(K, n_k)};
    std::vector<Fr> r, final_evals;
    Fr claim, blind_eval;
    Point comm_claim;
    const ZKSumcheckInstanceProof p =
        zk_prove(ps, g, degree, num_rounds, ldfr(blind_claim), ldgens(G1, 1, h1), ldgens(Gn, degree + 1, hn),
                 *(Transcript*)transcript, *(RandomTape*)tape, r, final_evals, claim, comm_claim, blind_eval);
    const std::vector<uint8_t> b = ser_zk(p);
    if (b.size() > cap) return 0;
    memcpy(out, b.data(), b.size());
    for (size_t j = 0; j < num_rounds; j++) stfr(r_out + 4 * j, r[j]);
    for (size_t j = 0; j < k; j++) stfr(final_out + 4 * j, final_evals[j]);
    stfr(claim_out, claim);
    comm_claim.compress(comm_claim_out);
    stfr(blind_eval_out, blind_eval);
    return b.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "orcd_zk_prove: %s\n", e.what());
    return 0;
  }
}
// ZKSumcheckInstanceProof::verify (sumcheck.rs:347-446) of serialised bytes against a compressed comm_claim, gens_n of
// degree_bound + 1 points: 0 accepted (e_out = the compressed last comm_eval, r_out = num_rounds challenges),
// 1 rejected, 2 the bytes or comm_claim do not parse
int orcd_zk_verify(const uint8_t* bytes, size_t nbytes, const uint8_t* comm_claim, size_t num_rounds, size_t degree_bound,
                   const uint64_t* G1, const uint64_t* h1, const uint64_t* Gn, const uint64_t* hn, void* transcript,
                   uint8_t* e_out, uint64_t* r_out) {
  Reader rd{bytes, nbytes};
  ZKSumcheckInstanceProof p;
  for (auto* v : {&p.comm_polys, &p.comm_evals}) {
    const uint64_t m = rd.u64();
    if (m > nbytes / 32) rd.ok = false;
    for (uint64_t i = 0; rd.ok && i < m; i++) v->push_back(rd.point());
  }
  const uint64_t m = rd.u64();
  if (m > nbytes / 136) rd.ok = false;
  for (uint64_t i = 0; rd.ok && i < m; i++) p.proofs.push_back(read_dot(rd));
  Point cc;
  if (!rd.ok || rd.at != nbytes || !ldpoint(comm_claim, cc)) return 2;
  Point e;
  std::vector<Fr> r;
  if (!zk_verify(p, cc, num_rounds, degree_bound, ldgens(G1, 1, h1), ldgens(Gn, degree_bound + 1, hn),
                 *(Transcript*)transcript, e, r))
    return 1;
  e.compress(e_out);
  for (size_t j = 0; j < num_rounds; j++) stfr(r_out + 4 * j, r[j]);
  return 0;
}

// ---- Σ-protocols of committed scalars (gens: G1 one affine point, h1 one).  The provers return the proof's length (0 on
// error) and the compressed commitments the reference returns alongside; the verifiers return 0 accepted, 1 rejected,
// 2 the bytes or a commitment do not parse.
size_t orcd_knowledge_prove(const uint64_t* G1, const uint64_t* h1, void* transcript, void* tape, const uint64_t* x,
                            const uint64_t* r, uint8_t* out, uint8_t* C_out) {
  Point C;
  const KnowledgeProof p =
      knowledge_prove(ldgens(G1, 1, h1), *(Transcript*)transcript, *(RandomTape*)tape, ldfr(x), ldfr(r), C);
  std::vector<uint8_t> b;
  put_point(b, p.alpha);
  put_fr(b, p.z1);
  put_fr(b, p.z2);
  memcpy(out, b.data(), b.size());
  C.compress(C_out);
  return b.size();
}
int orcd_knowledge_verify(const uint64_t* G1, const uint64_t* h1, const uint8_t* proof, size_t proof_len,
                          const uint8_t* C, void* transcript) {
  Reader rd{proof, proof_len};
  KnowledgeProof p;
  p.alpha = rd.point();
  p.z1 = rd.fr();
  p.z2 = rd.fr();
  Point c;
  if (!rd.ok || rd.at != proof_len || !ldpoint(C, c)) return 2;
  return knowledge_verify(p, ldgens(G1, 1, h1), *(Transcript*)transcript, c) ? 0 : 1;
}
size_t orcd_equality_prove(const uint64_t* G1, const uint64_t* h1, void* transcript, void* tape, const uint64_t* v1,
                           const uint64_t* s1, const uint64_t* v2, const uint64_t* s2, uint8_t* out, uint8_t* C1_out,
                           uint8_t* C2_out) {
  Point C1, C2;
  const EqualityProof p = equality_prove(ldgens(G1, 1, h1), *(Transcript*)transcript, *(RandomTape*)tape, ldfr(v1),
                                         ldfr(s1), ldfr(v2), ldfr(s2), C1, C2);
  std::vector<uint8_t> b;
  put_point(b, p.alpha);
  put_fr(b, p.z);
  memcpy(out, b.data(), b.size());
  C1.compress(C1_out);
  C2.compress(C2_out);
  return b.size();
}
int orcd_equality_verify(const uint64_t* G1, const uint64_t* h1, const uint8_t* proof, size_t proof_len,
                         const uint8_t* C1, const uint8_t* C2, void* transcript) {
  Reader rd{proof, proof_len};
  EqualityProof p;
  p.alpha = rd.point();
  p.z = rd.fr();
  Point c1, c2;
  if (!rd.ok || rd.at != proof_len || !ldpoint(C1, c1) || !ldpoint(C2, c2)) return 2;
  return equality_verify(p, ldgens(G1, 1, h1), *(Transcript*)transcript, c1, c2) ? 0 : 1;
}
size_t orcd_product_prove(const uint64_t* G1, const uint64_t* h1, void* transcript, void* tape, const uint64_t* x,
                          const uint64_t* rX, const uint64_t* y, const uint64_t* rY, const uint64_t* z,
                          const uint64_t* rZ, uint8_t* out, uint8_t* X_out, uint8_t* Y_out, uint8_t* Z_out) {
  Point X, Y, Z;
  const ProductProof p = product_prove(ldgens(G1, 1, h1), *(Transcript*)transcript, *(RandomTape*)tape, ldfr(x), ldfr(rX),
                                       ldfr(y), ldfr(rY), ldfr(z), ldfr(rZ), X, Y, Z);
  std::vector<uint8_t> b;
  put_point(b, p.alpha);
  put_point(b, p.beta);
  put_point(b, p.delta);
  for (const Fr& f : p.z) put_fr(b, f);  // [F; 5]: no length prefix
  memcpy(out, b.data(), b.size());
  X.compress(X_out);
  Y.compress(Y_out);
  Z.compress(Z_out);
  return b.size();
}
int orcd_product_verify(const uint64_t* G1, const uint64_t* h1, const uint8_t* proof, size_t proof_len, const uint8_t* X,
                        const uint8_t* Y, const uint8_t* Z, void* transcript) {
  Reader rd{proof, proof_len};
  ProductProof p;
  p.alpha = rd.point();
  p.beta = rd.point();
  p.delta = rd.point();
  for (Fr& f : p.z) f = rd.fr();
  Point x, y, z;
  if (!rd.ok || rd.at != proof_len || !ldpoint(X, x) || !ldpoint(Y, y) || !ldpoint(Z, z)) return 2;
  return product_verify(p, ldgens(G1, 1, h1), *(Transcript*)transcript, x, y, z) ? 0 : 1;
}
// sum_i scalars[i] points[i] of n compressed points -> out (compressed): a verifier's homomorphic combination of
// commitments.  0, or 2 when a point does not decompress.
int orcd_point_lincomb(const uint8_t* points, size_t n, const uint64_t* scalars, uint8_t* out) {
  Point acc = Point::zero();
  for (size_t i = 0; i < n; i++) {
    Point p;
    if (!ldpoint(points + 32 * i, p)) return 2;
    acc += p * ldfr(scalars + 4 * i);
  }
  acc.compress(out);
  return 0;
}

}  // extern "C"
