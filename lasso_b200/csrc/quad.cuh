// lasso_b200 — quad-lane point arithmetic on the twisted-Edwards group of curve25519: FOUR lanes of a warp hold
// X, Y, Z, T of one extended point (role = lane & 3) and run the 4-way parallel forms of the group law, exchanging
// coordinates with quad shuffles.  Used wherever a chain of dependent point operations is on the critical path
// (the short MSMs of the opening proofs, the window combination of the large MSM): a lone thread is bound by
// instruction issue (~2000 instructions per addition), a quad is 3-4x faster.
// Included after the translation unit has chosen its fq_mul attributes (LB_FQ_MUL_ATTR).
#pragma once
#include "common.cuh"

namespace lb {

// ---------------------------------------------------------------- quad-lane point addition
// The latency of one extended addition on one thread is 9 dependent Fq multiplications; the short MSMs of the opening proofs (two rows, a few thousand terms) are nothing but a chain of
// ~30 of them.  Here the FOUR lanes of a quad hold X, Y, Z, T of the accumulator (role = lane & 3) and run
// the 4-way parallel form of add-2008-hwcd-3 (Hisil et al. sect. 4.2): A, B, D, C side by side, then
// E*F, G*H, F*G, E*H side by side -> 2 multiplication levels (+1 on the T lane for 2d*T2), the coordinates
// exchanged with quad shuffles.  `q` = X2, Y2, Z2, T2 of the other point (global or shared memory).
__device__ __forceinline__ fq_t shfl_fq(unsigned mask, const fq_t& v, int src_lane) {
  fq_t r;
#pragma unroll
  for (int l = 0; l < 8; l++) r.v[l] = __shfl_sync(mask, v.v[l], src_lane);
  return r;
}
// second half of the 4-way addition: v = (A, B, D, C) on the four lanes -> (X3, Y3, Z3, T3)
__device__ __forceinline__ fq_t quad_tail(unsigned mask, int lane, const fq_t& v) {  // v = A, B, D, C
  const int role = lane & 3, qb = lane & ~3;
  const fq_t o = shfl_fq(mask, v, lane ^ 1);  // B, A, C, D
  fq_t p1, p2 = fq_zero();
  if (role == 0) p1 = fq_sub(o, v);           // E = B - A
  else if (role == 1) p1 = fq_add(v, o);      // H = B + A
  else if (role == 2) { p1 = fq_sub(v, o); p2 = fq_add(v, o); }  // F = D - C, G = D + C
  else p1 = fq_add(o, v);                     // G
  const int src_a = qb + (role == 0 ? 2 : role == 1 ? 3 : role == 2 ? 2 : 0);
  fq_t a = shfl_fq(mask, p1, src_a);
  const fq_t b = shfl_fq(mask, p1, qb + 1);
  if (role == 2) a = p2;
  return fq_mul(role == 3 ? a : p1, role == 3 ? b : a);  // X3 = E F, Y3 = H G, Z3 = F G, T3 = E H
}
__device__ __forceinline__ fq_t quad_add(unsigned mask, int lane, const fq_t& mine, const fq_t* q) {
  const int role = lane & 3;
  const fq_t partner = shfl_fq(mask, mine, lane ^ 1);  // X <-> Y (Z <-> T unused)
  fq_t s1, m;
  if (role == 0) {
    s1 = fq_sub(partner, mine);  // Y1 - X1
    m = fq_sub(q[1], q[0]);
  } else if (role == 1) {
    s1 = fq_add(mine, partner);  // Y1 + X1
    m = fq_add(q[1], q[0]);
  } else if (role == 2) {
    s1 = mine;
    m = fq_dbl(q[2]);  // D = Z1 * 2 Z2
  } else {
    s1 = mine;
    m = fq_mul(q[3], fq_d2());  // C = T1 * (2d T2)
  }
  return quad_tail(mask, lane, fq_mul(s1, m));  // A, B, D, C -> X3, Y3, Z3, T3
}
// mixed quad addition: the quad's accumulator + one affine-niels entry; lane 0 / 1 / 3 hold the entry's
// (y-x | y+x) / (y+x | y-x) / (+-2dxy) already selected for the sign of the digit
__device__ __forceinline__ fq_t quad_madd(unsigned mask, int lane, const fq_t& mine, const fq_t& operand) {
  const int role = lane & 3;
  const fq_t partner = shfl_fq(mask, mine, lane ^ 1);
  fq_t v;
  if (role == 0) v = fq_mul(fq_sub(partner, mine), operand);       // A = (Y1 - X1)(y2 - x2)
  else if (role == 1) v = fq_mul(fq_add(mine, partner), operand);  // B = (Y1 + X1)(y2 + x2)
  else if (role == 2) v = fq_dbl(mine);                            // D = 2 Z1
  else v = fq_mul(mine, operand);                                  // C = T1 * 2d x2 y2
  return quad_tail(mask, lane, v);
}

// 2P (dbl-2008-hwcd, a = -1): 4 squarings side by side, then E*F, G*H, F*G, E*H side by side — two multiplication
// levels.  `mine` = X, Y, Z, T on the four lanes of the quad.
__device__ __forceinline__ fq_t quad_dbl(unsigned mask, int lane, const fq_t& mine) {
  const int role = lane & 3, qb = lane & ~3;
  const fq_t x = shfl_fq(mask, mine, qb), y = shfl_fq(mask, mine, qb + 1);
  fq_t s;
  if (role == 0) s = fq_mul(mine, mine);                 // A = X^2
  else if (role == 1) s = fq_mul(mine, mine);            // B = Y^2
  else if (role == 2) s = fq_dbl(fq_mul(mine, mine));    // C = 2 Z^2
  else { const fq_t xy = fq_add(x, y); s = fq_mul(xy, xy); }  // (X + Y)^2
  const fq_t A = shfl_fq(mask, s, qb), B = shfl_fq(mask, s, qb + 1), C = shfl_fq(mask, s, qb + 2), Q = shfl_fq(mask, s, qb + 3);
  const fq_t E = fq_sub(fq_sub(Q, A), B), G = fq_sub(B, A), F = fq_sub(G, C), H = fq_neg(fq_add(A, B));
  if (role == 0) return fq_mul(E, F);
  if (role == 1) return fq_mul(G, H);
  if (role == 2) return fq_mul(F, G);
  return fq_mul(E, H);
}

}  // namespace lb
