// lasso_b200 — twisted-Edwards group of curve25519 (-x^2 + y^2 = 1 + d x^2 y^2) on sm_90a.
//
// Replaces ark-ec's `twisted_edwards::{Affine, Projective}` under the reference's MSM
// (src/msm/mod.rs:127-163: `buckets[..] += base`, running sums, window doublings) and
// Pedersen commitments (src/poly/commitments.rs:78-93).  Extended coordinates (X:Y:Z:T),
// a = -1, complete unified formulas (add-2008-hwcd-3 / dbl-2008-hwcd), so identity and
// equal inputs need no special-casing.  Any formula yields the same group element; outputs
// are compared after affine normalisation, as the reference's transcript sees them
// (src/utils/transcript.rs:47-51).
#pragma once
#include "fq.cuh"

namespace lb {

struct pt_ext {  // 128 B, internal (non-Montgomery) Fq limbs
  fq_t X, Y, Z, T;
};
// affine point prepared for mixed addition: (y+x, y-x, 2d*x*y), 96 B
struct pt_niels {
  fq_t yplusx, yminusx, t2d;
};

LB_HD fq_t fq_d2() {  // 2d mod q, internal form
  fq_t r = {{0x26b2f159u, 0xebd69b94u, 0x8283b156u, 0x00e0149au, 0xeef3d130u, 0x198e80f2u, 0x56dffce7u, 0x2406d9dcu}};
  return r;
}

LB_HD pt_ext pt_identity() {
  pt_ext p;
  p.X = fq_zero();
  p.Y = fq_one();
  p.Z = fq_one();
  p.T = fq_zero();
  return p;
}
LB_HD pt_niels niels_identity() {
  pt_niels n;
  n.yplusx = fq_one();
  n.yminusx = fq_one();
  n.t2d = fq_zero();
  return n;
}
// from internal affine (x, y)
LB_HD pt_niels niels_from_affine(const fq_t& x, const fq_t& y) {
  pt_niels n;
  n.yplusx = fq_add(y, x);
  n.yminusx = fq_sub(y, x);
  n.t2d = fq_mul(fq_mul(x, y), fq_d2());
  return n;
}
LB_HD pt_niels niels_neg(const pt_niels& n) {
  pt_niels r;
  r.yplusx = n.yminusx;
  r.yminusx = n.yplusx;
  r.t2d = fq_neg(n.t2d);
  return r;
}
LB_HD pt_ext pt_neg(const pt_ext& p) {
  pt_ext r = p;
  r.X = fq_neg(p.X);
  r.T = fq_neg(p.T);
  return r;
}

// P + Q, Q affine-niels: 7 M
LB_HD pt_ext pt_madd(const pt_ext& p, const pt_niels& q) {
  fq_t A = fq_mul(fq_sub(p.Y, p.X), q.yminusx);
  fq_t B = fq_mul(fq_add(p.Y, p.X), q.yplusx);
  fq_t C = fq_mul(p.T, q.t2d);
  fq_t D = fq_dbl(p.Z);
  fq_t E = fq_sub(B, A), F = fq_sub(D, C), G = fq_add(D, C), H = fq_add(B, A);
  pt_ext r;
  r.X = fq_mul(E, F);
  r.Y = fq_mul(G, H);
  r.T = fq_mul(E, H);
  r.Z = fq_mul(F, G);
  return r;
}
// P - Q
LB_HD pt_ext pt_msub(const pt_ext& p, const pt_niels& q) {
  fq_t A = fq_mul(fq_sub(p.Y, p.X), q.yplusx);
  fq_t B = fq_mul(fq_add(p.Y, p.X), q.yminusx);
  fq_t C = fq_mul(p.T, q.t2d);
  fq_t D = fq_dbl(p.Z);
  fq_t E = fq_sub(B, A), F = fq_add(D, C), G = fq_sub(D, C), H = fq_add(B, A);
  pt_ext r;
  r.X = fq_mul(E, F);
  r.Y = fq_mul(G, H);
  r.T = fq_mul(E, H);
  r.Z = fq_mul(F, G);
  return r;
}
// P + Q, both extended: 9 M
LB_HD pt_ext pt_add(const pt_ext& p, const pt_ext& q) {
  fq_t A = fq_mul(fq_sub(p.Y, p.X), fq_sub(q.Y, q.X));
  fq_t B = fq_mul(fq_add(p.Y, p.X), fq_add(q.Y, q.X));
  fq_t C = fq_mul(fq_mul(p.T, q.T), fq_d2());
  fq_t D = fq_dbl(fq_mul(p.Z, q.Z));
  fq_t E = fq_sub(B, A), F = fq_sub(D, C), G = fq_add(D, C), H = fq_add(B, A);
  pt_ext r;
  r.X = fq_mul(E, F);
  r.Y = fq_mul(G, H);
  r.T = fq_mul(E, H);
  r.Z = fq_mul(F, G);
  return r;
}
// 2P: 4 S + 4 M
LB_HD pt_ext pt_dbl(const pt_ext& p) {
  fq_t A = fq_sqr(p.X), B = fq_sqr(p.Y), C = fq_dbl(fq_sqr(p.Z));
  fq_t D = fq_neg(A);
  fq_t E = fq_sub(fq_sub(fq_sqr(fq_add(p.X, p.Y)), A), B);
  fq_t G = fq_add(D, B), F = fq_sub(G, C), H = fq_sub(D, B);
  pt_ext r;
  r.X = fq_mul(E, F);
  r.Y = fq_mul(G, H);
  r.T = fq_mul(E, H);
  r.Z = fq_mul(F, G);
  return r;
}
LB_HD pt_ext pt_from_niels(const pt_niels& n) { return pt_madd(pt_identity(), n); }

// arkworks TE Affine {x, y} (Montgomery limbs, 64 B) -> niels
LB_HD pt_niels niels_from_ark_affine(const fq_t& xm, const fq_t& ym) {
  return niels_from_affine(fq_from_ark(xm), fq_from_ark(ym));
}
// canonical affine coordinates (plain integers < q)
LB_HD void pt_to_affine_canonical(const pt_ext& p, fq_t& x, fq_t& y) {
  fq_t zi = fq_inv(p.Z);
  x = fq_canonical(fq_mul(p.X, zi));
  y = fq_canonical(fq_mul(p.Y, zi));
}
// ark-serialize compressed TE point from canonical affine coords: 32-byte LE y, top bit set
// iff x > -x as integers, i.e. x > (q-1)/2   [SURVEY Appendix C]
LB_HD void pt_compress_canonical(const fq_t& x, const fq_t& y, uint32_t out[8]) {
  // x > (q-1)/2 = 2^254 - 10  <=>  x + 9 >= 2^254
  uint64_t c = 9;
  uint32_t top = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t u = (uint64_t)x.v[i] + c;
    top = (uint32_t)u;
    c = u >> 32;
  }
  bool neg = (top >> 30) != 0;
#pragma unroll
  for (int i = 0; i < 8; i++) out[i] = y.v[i];
  if (neg) out[7] |= 0x80000000u;
}

}  // namespace lb
