// lasso_b200 — curve25519 base field Fq = GF(2^255 - 19) on sm_90a.
//
// Replaces what the reference gets from ark-ff (generic 4x64 Montgomery Fq) underneath
// ark-ec's twisted-Edwards group in src/msm/mod.rs:127-163 and src/poly/commitments.rs:84-93.
// Inside kernels an element is a plain (non-Montgomery) 256-bit integer x, only loosely
// reduced (any x < 2^256 with the right residue): q is pseudo-Mersenne, so a product
// reduces with one multiplication by 38 instead of a Montgomery pass.  The boundary format
// stays arkworks': 4 x u64 limbs of x * 2^256 mod q = 38 x mod q; fq_from_ark / fq_to_ark
// convert, and every group output is compared / serialised after canonical reduction.
#pragma once
#include "fr.cuh"

namespace lb {

struct alignas(32) fq_t {
  uint32_t v[8];
};

LB_HD fq_t fq_zero() {
  fq_t r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = 0;
  return r;
}
LB_HD fq_t fq_one() {
  fq_t r = fq_zero();
  r.v[0] = 1;
  return r;
}

// x + 38*c for a small c (the wrap-around of 2^256 = 38 mod q), twice: the second wrap
// can only happen when the value is already tiny, so it cannot ripple.
LB_HD void fq_fold_carry(uint32_t t[8], uint32_t c) {
  LB_CF_DECL
  uint32_t k = c * 38u, c2;
  LB_ADD_CC(t[0], t[0], k);
  LB_ADDC_CC(t[1], t[1], 0u);
  LB_ADDC_CC(t[2], t[2], 0u);
  LB_ADDC_CC(t[3], t[3], 0u);
  LB_ADDC_CC(t[4], t[4], 0u);
  LB_ADDC_CC(t[5], t[5], 0u);
  LB_ADDC_CC(t[6], t[6], 0u);
  LB_ADDC_CC(t[7], t[7], 0u);
  LB_ADDC(c2, 0u, 0u);
  t[0] += c2 * 38u;
}

LB_HD fq_t fq_add(const fq_t& a, const fq_t& b) {
  LB_CF_DECL
  fq_t r;
  uint32_t c;
  LB_ADD_CC(r.v[0], a.v[0], b.v[0]);
  LB_ADDC_CC(r.v[1], a.v[1], b.v[1]);
  LB_ADDC_CC(r.v[2], a.v[2], b.v[2]);
  LB_ADDC_CC(r.v[3], a.v[3], b.v[3]);
  LB_ADDC_CC(r.v[4], a.v[4], b.v[4]);
  LB_ADDC_CC(r.v[5], a.v[5], b.v[5]);
  LB_ADDC_CC(r.v[6], a.v[6], b.v[6]);
  LB_ADDC_CC(r.v[7], a.v[7], b.v[7]);
  LB_ADDC(c, 0u, 0u);
  fq_fold_carry(r.v, c);
  return r;
}

LB_HD fq_t fq_sub(const fq_t& a, const fq_t& b) {
  LB_CF_DECL
  fq_t r;
  uint32_t bw, bw2;
  LB_SUB_CC(r.v[0], a.v[0], b.v[0]);
  LB_SUBC_CC(r.v[1], a.v[1], b.v[1]);
  LB_SUBC_CC(r.v[2], a.v[2], b.v[2]);
  LB_SUBC_CC(r.v[3], a.v[3], b.v[3]);
  LB_SUBC_CC(r.v[4], a.v[4], b.v[4]);
  LB_SUBC_CC(r.v[5], a.v[5], b.v[5]);
  LB_SUBC_CC(r.v[6], a.v[6], b.v[6]);
  LB_SUBC_CC(r.v[7], a.v[7], b.v[7]);
  LB_SUBC(bw, 0u, 0u);  // all-ones iff borrow: the wrapped value is 2^256 too big = 38 too big mod q
  LB_SUB_CC(r.v[0], r.v[0], bw & 38u);
  LB_SUBC_CC(r.v[1], r.v[1], 0u);
  LB_SUBC_CC(r.v[2], r.v[2], 0u);
  LB_SUBC_CC(r.v[3], r.v[3], 0u);
  LB_SUBC_CC(r.v[4], r.v[4], 0u);
  LB_SUBC_CC(r.v[5], r.v[5], 0u);
  LB_SUBC_CC(r.v[6], r.v[6], 0u);
  LB_SUBC_CC(r.v[7], r.v[7], 0u);
  LB_SUBC(bw2, 0u, 0u);
  r.v[0] -= bw2 & 38u;  // second wrap only when the value is within 38 of 2^256: cannot ripple
  return r;
}
LB_HD fq_t fq_neg(const fq_t& a) { return fq_sub(fq_zero(), a); }
LB_HD fq_t fq_dbl(const fq_t& a) { return fq_add(a, a); }

// 8x8 -> 16 limb product on the even/odd split accumulator (see fr.cuh), then 2^256 = 38 fold.
// The MSM kernels compile this as a real (non-inlined) function: a bucket kernel inlines ~50 field
// multiplications otherwise (>100 KB of SASS) and, with 3 warps per scheduler each in a different
// phase, stalls on instruction fetch (ncu: stalled_no_instruction was the top stall reason).
#ifndef LB_FQ_MUL_ATTR
#define LB_FQ_MUL_ATTR LB_HD
#endif
#ifdef LB_FQ_MUL_BYVALUE
LB_FQ_MUL_ATTR fq_t fq_mul(const fq_t A, const fq_t B) {
#else
LB_FQ_MUL_ATTR fq_t fq_mul(const fq_t& A, const fq_t& B) {
#endif
  const uint32_t* a = A.v;
  const uint32_t* b = B.v;
  uint32_t ev[18], od[18];  // value = sum ev[k] 2^(32k) + sum od[k] 2^(32(k+1))
#pragma unroll
  for (int k = 0; k < 18; k++) ev[k] = od[k] = 0;
  {
    uint64_t t;
    t = (uint64_t)a[0] * b[0]; ev[0] = (uint32_t)t; ev[1] = (uint32_t)(t >> 32);
    t = (uint64_t)a[2] * b[0]; ev[2] = (uint32_t)t; ev[3] = (uint32_t)(t >> 32);
    t = (uint64_t)a[4] * b[0]; ev[4] = (uint32_t)t; ev[5] = (uint32_t)(t >> 32);
    t = (uint64_t)a[6] * b[0]; ev[6] = (uint32_t)t; ev[7] = (uint32_t)(t >> 32);
    t = (uint64_t)a[1] * b[0]; od[0] = (uint32_t)t; od[1] = (uint32_t)(t >> 32);
    t = (uint64_t)a[3] * b[0]; od[2] = (uint32_t)t; od[3] = (uint32_t)(t >> 32);
    t = (uint64_t)a[5] * b[0]; od[4] = (uint32_t)t; od[5] = (uint32_t)(t >> 32);
    t = (uint64_t)a[7] * b[0]; od[6] = (uint32_t)t; od[7] = (uint32_t)(t >> 32);
  }
#pragma unroll
  for (int i = 1; i < 8; i++) {
    LB_CF_DECL
    if (i & 1) {
      // odd row: a_even * b_i lands at odd limbs -> od[i-1 ..], a_odd * b_i at even limbs -> ev[i+1 ..]
      LB_PAIR_MAD(od[i - 1], od[i], a[0], b[i]);
      LB_PAIR_MADC(od[i + 1], od[i + 2], a[2], b[i]);
      LB_PAIR_MADC(od[i + 3], od[i + 4], a[4], b[i]);
      LB_PAIR_MADC(od[i + 5], od[i + 6], a[6], b[i]);
      LB_ADDC(od[i + 7], od[i + 7], 0u);
      LB_PAIR_MAD(ev[i + 1], ev[i + 2], a[1], b[i]);
      LB_PAIR_MADC(ev[i + 3], ev[i + 4], a[3], b[i]);
      LB_PAIR_MADC(ev[i + 5], ev[i + 6], a[5], b[i]);
      LB_PAIR_MADC(ev[i + 7], ev[i + 8], a[7], b[i]);
      LB_ADDC(ev[i + 9], ev[i + 9], 0u);
    } else {
      LB_PAIR_MAD(ev[i], ev[i + 1], a[0], b[i]);
      LB_PAIR_MADC(ev[i + 2], ev[i + 3], a[2], b[i]);
      LB_PAIR_MADC(ev[i + 4], ev[i + 5], a[4], b[i]);
      LB_PAIR_MADC(ev[i + 6], ev[i + 7], a[6], b[i]);
      LB_ADDC(ev[i + 8], ev[i + 8], 0u);
      LB_PAIR_MAD(od[i], od[i + 1], a[1], b[i]);
      LB_PAIR_MADC(od[i + 2], od[i + 3], a[3], b[i]);
      LB_PAIR_MADC(od[i + 4], od[i + 5], a[5], b[i]);
      LB_PAIR_MADC(od[i + 6], od[i + 7], a[7], b[i]);
      LB_ADDC(od[i + 8], od[i + 8], 0u);
    }
  }
  // p[k] = ev[k] + od[k-1] (+ carry), 16 limbs (the product is < 2^512 so nothing above)
  uint32_t p[16];
  {
    LB_CF_DECL
    p[0] = ev[0];
    LB_ADD_CC(p[1], ev[1], od[0]);
    LB_ADDC_CC(p[2], ev[2], od[1]);
    LB_ADDC_CC(p[3], ev[3], od[2]);
    LB_ADDC_CC(p[4], ev[4], od[3]);
    LB_ADDC_CC(p[5], ev[5], od[4]);
    LB_ADDC_CC(p[6], ev[6], od[5]);
    LB_ADDC_CC(p[7], ev[7], od[6]);
    LB_ADDC_CC(p[8], ev[8], od[7]);
    LB_ADDC_CC(p[9], ev[9], od[8]);
    LB_ADDC_CC(p[10], ev[10], od[9]);
    LB_ADDC_CC(p[11], ev[11], od[10]);
    LB_ADDC_CC(p[12], ev[12], od[11]);
    LB_ADDC_CC(p[13], ev[13], od[12]);
    LB_ADDC_CC(p[14], ev[14], od[13]);
    LB_ADDC(p[15], ev[15], od[14]);
  }
  // r = lo + 38 * hi  (9 limbs), then fold the 9th limb
  fq_t r;
  uint64_t c = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    uint64_t t = (uint64_t)p[8 + k] * 38u + p[k] + c;
    r.v[k] = (uint32_t)t;
    c = t >> 32;
  }
  fq_fold_carry(r.v, (uint32_t)c);
  return r;
}
LB_HD fq_t fq_sqr(const fq_t& a) { return fq_mul(a, a); }

// small-constant multiply (c < 2^26 or so)
LB_HD fq_t fq_mul_small(const fq_t& a, uint32_t k) {
  fq_t r;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t t = (uint64_t)a.v[i] * k + c;
    r.v[i] = (uint32_t)t;
    c = t >> 32;
  }
  // c < 2^26: fold c * 38 (may exceed 32 bits) in two steps
  uint64_t f = c * 38u;
  uint32_t t2[8];
#pragma unroll
  for (int i = 0; i < 8; i++) t2[i] = r.v[i];
  {
    uint64_t s = (uint64_t)t2[0] + (uint32_t)f;
    t2[0] = (uint32_t)s;
    uint64_t cc = (s >> 32) + (f >> 32);
#pragma unroll
    for (int i = 1; i < 8; i++) {
      s = (uint64_t)t2[i] + cc;
      t2[i] = (uint32_t)s;
      cc = s >> 32;
    }
    t2[0] += (uint32_t)cc * 38u;
  }
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t2[i];
  return r;
}

// fully reduce to the canonical representative in [0, q)
LB_HD fq_t fq_canonical(const fq_t& a) {
  uint32_t t[8];
#pragma unroll
  for (int i = 0; i < 8; i++) t[i] = a.v[i];
  // fold bit 255: x = (x mod 2^255) + 19 * (x >> 255)
#pragma unroll
  for (int rep = 0; rep < 2; rep++) {
    uint32_t top = t[7] >> 31;
    t[7] &= 0x7fffffffu;
    uint64_t c = (uint64_t)top * 19u;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint64_t s = (uint64_t)t[i] + c;
      t[i] = (uint32_t)s;
      c = s >> 32;
    }
  }
  // now t < 2^255; subtract q if t >= q  (q = 2^255 - 19): t >= q  <=>  t + 19 >= 2^255
  uint32_t s[8];
  uint64_t c = 19;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t u = (uint64_t)t[i] + c;
    s[i] = (uint32_t)u;
    c = u >> 32;
  }
  bool ge = (s[7] >> 31) != 0;
  s[7] &= 0x7fffffffu;
  fq_t r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = ge ? s[i] : t[i];
  return r;
}
LB_HD bool fq_is_zero(const fq_t& a) {
  fq_t c = fq_canonical(a);
  uint32_t x = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) x |= c.v[i];
  return x == 0;
}
LB_HD bool fq_equal(const fq_t& a, const fq_t& b) { return fq_is_zero(fq_sub(a, b)); }

// a^(2^n)
LB_HD fq_t fq_sqr_n(fq_t a, int n) {
  for (int i = 0; i < n; i++) a = fq_sqr(a);
  return a;
}
// a^(q-2) = a^(2^255 - 21), the standard curve25519 addition chain (254 S + 11 M)
LB_HD fq_t fq_inv(const fq_t& z) {
  fq_t z2 = fq_sqr(z);
  fq_t z9 = fq_mul(fq_sqr_n(z2, 2), z);
  fq_t z11 = fq_mul(z9, z2);
  fq_t z2_5_0 = fq_mul(fq_sqr(z11), z9);
  fq_t z2_10_0 = fq_mul(fq_sqr_n(z2_5_0, 5), z2_5_0);
  fq_t z2_20_0 = fq_mul(fq_sqr_n(z2_10_0, 10), z2_10_0);
  fq_t z2_40_0 = fq_mul(fq_sqr_n(z2_20_0, 20), z2_20_0);
  fq_t z2_50_0 = fq_mul(fq_sqr_n(z2_40_0, 10), z2_10_0);
  fq_t z2_100_0 = fq_mul(fq_sqr_n(z2_50_0, 50), z2_50_0);
  fq_t z2_200_0 = fq_mul(fq_sqr_n(z2_100_0, 100), z2_100_0);
  fq_t z2_250_0 = fq_mul(fq_sqr_n(z2_200_0, 50), z2_50_0);
  return fq_mul(fq_sqr_n(z2_250_0, 5), z11);
}

// arkworks Montgomery limbs (38 x mod q) -> internal x : multiply by 38^-1 mod q
LB_HD fq_t fq_from_ark(const fq_t& m) {
  // 38^-1 mod q
  const fq_t inv38 = {{0x9435e50au, 0x435e50d7u, 0x35e50d79u, 0x5e50d794u, 0xe50d7943u, 0x50d79435u, 0x0d79435eu, 0x179435e5u}};
  return fq_mul(m, inv38);
}
// internal x -> arkworks Montgomery limbs, canonical
LB_HD fq_t fq_to_ark(const fq_t& x) { return fq_canonical(fq_mul_small(x, 38u)); }

}  // namespace lb
