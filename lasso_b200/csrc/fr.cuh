// lasso_b200 — curve25519 scalar field Fr on sm_90a (and on the host, for the prover's
// Fiat–Shamir / interpolation glue).
//
// Replaces what the reference gets from ark-ff's `Fp<MontBackend<_,4>,4>` under
// DensePolynomial / EqPolynomial / sumcheck (src/poly/dense_mlpoly.rs:209-235,
// src/poly/eq_poly.rs:21-38, src/subprotocols/sumcheck.rs:179-218).  Memory format is
// bit-identical to ark-ff: 4 x u64 little-endian limbs of a*2^256 mod l, viewed here as
// 8 x u32.  All results are canonical residues (< l), so values are bit-exact against
// the reference no matter how the arithmetic is scheduled.
//
// Multiplication: 32-bit CIOS Montgomery with the accumulator split into an "even" and an
// "odd" limb array so every 32x32 product is one mad.lo.cc/madc.hi.cc pair on an aligned
// register pair (ptxas fuses the pair into one IMAD.WIDE with carry-in/out).  The modulus
// l = 2^252 + c (c < 2^125) has limbs {p0,p1,p2,p3,0,0,0,2^28}: the reduction step costs four
// products and a shift instead of eight products.
#pragma once
#include <cstdint>
#if !defined(__CUDA_ARCH__)
#include "host_modinv.hpp"
#endif

#if defined(__CUDACC__)
#define LB_HD __host__ __device__ __forceinline__
#else
#define LB_HD inline
#endif

namespace lb {

struct alignas(32) fr_t {
  uint32_t v[8];
};

#define LB_FR_P0 0x5cf5d3edu
#define LB_FR_P1 0x5812631au
#define LB_FR_P2 0xa2f79cd6u
#define LB_FR_P3 0x14def9deu
#define LB_FR_P7 0x10000000u
#define LB_FR_INV 0x12547e1bu  // -l^-1 mod 2^32

// ---- carry-chain primitives: PTX on the device, emulated with a local flag `cf` on the host
#if defined(__CUDA_ARCH__)
#define LB_CF_DECL
#define LB_ADD_CC(d, a, b) asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define LB_ADDC_CC(d, a, b) asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define LB_ADDC(d, a, b) asm volatile("addc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define LB_SUB_CC(d, a, b) asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define LB_SUBC_CC(d, a, b) asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define LB_SUBC(d, a, b) asm volatile("subc.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b))
#define LB_MAD_LO_CC(d, a, b, c) asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c))
#define LB_MADC_LO_CC(d, a, b, c) asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c))
#define LB_MADC_HI_CC(d, a, b, c) asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c))
#define LB_MADC_HI(d, a, b, c) asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c))
// (lo,hi) += a*b as ONE asm statement on a read-write pair: the shape ptxas fuses into IMAD.WIDE.U32[.X]
#define LB_PAIR_MAD(lo, hi, a, b) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b))
#define LB_PAIR_MADC(lo, hi, a, b) asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b))
#define LB_PAIR_MADC_END(lo, hi, a, b) asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b))
#else
#define LB_PAIR_MAD(lo, hi, a, b) { LB_MAD_LO_CC(lo, a, b, lo); LB_MADC_HI_CC(hi, a, b, hi); }
#define LB_PAIR_MADC(lo, hi, a, b) { LB_MADC_LO_CC(lo, a, b, lo); LB_MADC_HI_CC(hi, a, b, hi); }
#define LB_PAIR_MADC_END(lo, hi, a, b) { LB_MADC_LO_CC(lo, a, b, lo); LB_MADC_HI(hi, a, b, hi); }
#define LB_CF_DECL uint32_t cf = 0; (void)cf;
#define LB_ADD_CC(d, a, b) { uint64_t t_ = (uint64_t)(a) + (b); d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32); }
#define LB_ADDC_CC(d, a, b) { uint64_t t_ = (uint64_t)(a) + (b) + cf; d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32); }
#define LB_ADDC(d, a, b) { d = (uint32_t)((a) + (b) + cf); }
#define LB_SUB_CC(d, a, b) { uint64_t t_ = (uint64_t)(a) - (b); d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32) & 1; }
#define LB_SUBC_CC(d, a, b) { uint64_t t_ = (uint64_t)(a) - (b) - cf; d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32) & 1; }
#define LB_SUBC(d, a, b) { d = (uint32_t)((a) - (b) - cf); }
#define LB_MAD_LO_CC(d, a, b, c) { uint64_t t_ = (uint64_t)(uint32_t)((uint64_t)(a) * (b)) + (c); d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32); }
#define LB_MADC_LO_CC(d, a, b, c) { uint64_t t_ = (uint64_t)(uint32_t)((uint64_t)(a) * (b)) + (c) + cf; d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32); }
#define LB_MADC_HI_CC(d, a, b, c) { uint64_t t_ = (((uint64_t)(a) * (b)) >> 32) + (c) + cf; d = (uint32_t)t_; cf = (uint32_t)(t_ >> 32); }
#define LB_MADC_HI(d, a, b, c) { d = (uint32_t)((((uint64_t)(a) * (b)) >> 32) + (c) + cf); }
#endif
// NOTE on the device: PTX's sub.cc sets CF = 1 on NO borrow?  No: PTX defines the borrow in
// CC.CF the same way as the host emulation above (subc subtracts CC.CF), so a final
// `subc d, 0, 0` yields 0xffffffff iff the chain borrowed.

LB_HD fr_t fr_zero() {
  fr_t r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = 0;
  return r;
}
// Montgomery form of 1: R mod l
LB_HD fr_t fr_one() {
  fr_t r = {{0x8d98951du, 0xd6ec3174u, 0x737dcf70u, 0xc6ef5bf4u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0x0fffffffu}};
  return r;
}
// R^2 mod l (Montgomery form of R): multiply by it to enter Montgomery form
LB_HD fr_t fr_r2() {
  fr_t r = {{0x449c0f01u, 0xa40611e3u, 0x68859347u, 0xd00e1ba7u, 0x17f5be65u, 0xceec73d2u, 0x7c309a3du, 0x0399411bu}};
  return r;
}
LB_HD bool fr_is_zero(const fr_t& a) {
  uint32_t x = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) x |= a.v[i];
  return x == 0;
}
LB_HD bool fr_eq(const fr_t& a, const fr_t& b) {
  uint32_t x = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) x |= a.v[i] ^ b.v[i];
  return x == 0;
}

// r = t - l if t >= l else t   (t < 2l)
LB_HD fr_t fr_reduce_once(const uint32_t t[8]) {
  LB_CF_DECL
  uint32_t s[8], bw;
  LB_SUB_CC(s[0], t[0], LB_FR_P0);
  LB_SUBC_CC(s[1], t[1], LB_FR_P1);
  LB_SUBC_CC(s[2], t[2], LB_FR_P2);
  LB_SUBC_CC(s[3], t[3], LB_FR_P3);
  LB_SUBC_CC(s[4], t[4], 0u);
  LB_SUBC_CC(s[5], t[5], 0u);
  LB_SUBC_CC(s[6], t[6], 0u);
  LB_SUBC_CC(s[7], t[7], LB_FR_P7);
  LB_SUBC(bw, 0u, 0u);  // 0xffffffff iff t < l
  fr_t r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = bw ? t[i] : s[i];
  return r;
}

LB_HD fr_t fr_add(const fr_t& a, const fr_t& b) {
  LB_CF_DECL
  uint32_t t[8];
  LB_ADD_CC(t[0], a.v[0], b.v[0]);
  LB_ADDC_CC(t[1], a.v[1], b.v[1]);
  LB_ADDC_CC(t[2], a.v[2], b.v[2]);
  LB_ADDC_CC(t[3], a.v[3], b.v[3]);
  LB_ADDC_CC(t[4], a.v[4], b.v[4]);
  LB_ADDC_CC(t[5], a.v[5], b.v[5]);
  LB_ADDC_CC(t[6], a.v[6], b.v[6]);
  LB_ADDC(t[7], a.v[7], b.v[7]);  // a, b < l < 2^253: no carry out
  return fr_reduce_once(t);
}

LB_HD fr_t fr_sub(const fr_t& a, const fr_t& b) {
  LB_CF_DECL
  uint32_t t[8], bw;
  LB_SUB_CC(t[0], a.v[0], b.v[0]);
  LB_SUBC_CC(t[1], a.v[1], b.v[1]);
  LB_SUBC_CC(t[2], a.v[2], b.v[2]);
  LB_SUBC_CC(t[3], a.v[3], b.v[3]);
  LB_SUBC_CC(t[4], a.v[4], b.v[4]);
  LB_SUBC_CC(t[5], a.v[5], b.v[5]);
  LB_SUBC_CC(t[6], a.v[6], b.v[6]);
  LB_SUBC_CC(t[7], a.v[7], b.v[7]);
  LB_SUBC(bw, 0u, 0u);  // all-ones iff a < b
  fr_t r;
  LB_ADD_CC(r.v[0], t[0], bw & LB_FR_P0);
  LB_ADDC_CC(r.v[1], t[1], bw & LB_FR_P1);
  LB_ADDC_CC(r.v[2], t[2], bw & LB_FR_P2);
  LB_ADDC_CC(r.v[3], t[3], bw & LB_FR_P3);
  LB_ADDC_CC(r.v[4], t[4], 0u);
  LB_ADDC_CC(r.v[5], t[5], 0u);
  LB_ADDC_CC(r.v[6], t[6], 0u);
  LB_ADDC(r.v[7], t[7], bw & LB_FR_P7);
  return r;
}
LB_HD fr_t fr_neg(const fr_t& a) { return fr_sub(fr_zero(), a); }
LB_HD fr_t fr_dbl(const fr_t& a) { return fr_add(a, a); }

// one CIOS row: acc += a * bi ; acc += m * l ; acc >>= 32, on the even/odd split accumulator.
// value(acc) = sum e[k] 2^(32k) + sum o[k] 2^(32(k+1)) + stray   (see header comment)
LB_HD void fr_mul_row(uint32_t e[9], uint32_t o[8], uint32_t& stray, const uint32_t a[8], uint32_t bi, bool first) {
  LB_CF_DECL
  if (first) {
    uint64_t t;
    t = (uint64_t)a[0] * bi; e[0] = (uint32_t)t; e[1] = (uint32_t)(t >> 32);
    t = (uint64_t)a[2] * bi; e[2] = (uint32_t)t; e[3] = (uint32_t)(t >> 32);
    t = (uint64_t)a[4] * bi; e[4] = (uint32_t)t; e[5] = (uint32_t)(t >> 32);
    t = (uint64_t)a[6] * bi; e[6] = (uint32_t)t; e[7] = (uint32_t)(t >> 32);
    e[8] = 0;
    t = (uint64_t)a[1] * bi; o[0] = (uint32_t)t; o[1] = (uint32_t)(t >> 32);
    t = (uint64_t)a[3] * bi; o[2] = (uint32_t)t; o[3] = (uint32_t)(t >> 32);
    t = (uint64_t)a[5] * bi; o[4] = (uint32_t)t; o[5] = (uint32_t)(t >> 32);
    t = (uint64_t)a[7] * bi; o[6] = (uint32_t)t; o[7] = (uint32_t)(t >> 32);
  } else {
    // the carry of (limb 0 += stray) has weight 2^32 = the odd chain's first limb
    LB_ADD_CC(e[0], e[0], stray);
    LB_PAIR_MADC(o[0], o[1], a[1], bi);
    LB_PAIR_MADC(o[2], o[3], a[3], bi);
    LB_PAIR_MADC(o[4], o[5], a[5], bi);
    LB_PAIR_MADC_END(o[6], o[7], a[7], bi);  // value bound (< 2^255 after the shift) => no carry out
    LB_PAIR_MAD(e[0], e[1], a[0], bi);
    LB_PAIR_MADC(e[2], e[3], a[2], bi);
    LB_PAIR_MADC(e[4], e[5], a[4], bi);
    LB_PAIR_MADC(e[6], e[7], a[6], bi);
    LB_ADDC(e[8], e[8], 0u);
  }
  uint32_t m = e[0] * LB_FR_INV;
  const uint32_t p0 = LB_FR_P0, p1 = LB_FR_P1, p2 = LB_FR_P2, p3 = LB_FR_P3;
  LB_PAIR_MAD(e[0], e[1], m, p0);  // e[0] -> 0
  LB_PAIR_MADC(e[2], e[3], m, p2);
  LB_ADDC_CC(e[4], e[4], 0u);
  LB_ADDC_CC(e[5], e[5], 0u);
  LB_ADDC_CC(e[6], e[6], 0u);
  LB_ADDC_CC(e[7], e[7], 0u);
  LB_ADDC(e[8], e[8], 0u);
  LB_PAIR_MAD(o[0], o[1], m, p1);
  LB_PAIR_MADC(o[2], o[3], m, p3);
  LB_ADDC_CC(o[4], o[4], 0u);
  LB_ADDC_CC(o[5], o[5], 0u);
  LB_ADDC_CC(o[6], o[6], m << 28);  // m * p7 = m * 2^28 sits on the (o6, o7) pair
  LB_ADDC(o[7], o[7], m >> 4);
  // divide by 2^32: e[0] == 0 now; e[1] becomes the stray limb-0 addend, the arrays swap roles
  stray = e[1];
  uint32_t ne[9], no[8];
#pragma unroll
  for (int k = 0; k < 8; k++) ne[k] = o[k];
  ne[8] = 0;
#pragma unroll
  for (int k = 0; k < 7; k++) no[k] = e[k + 2];
  no[7] = 0;
#pragma unroll
  for (int k = 0; k < 9; k++) e[k] = ne[k];
#pragma unroll
  for (int k = 0; k < 8; k++) o[k] = no[k];
}

#if !defined(__CUDA_ARCH__)
// Host fast path (the prover's Fiat-Shamir glue: interpolation, challenge arithmetic, u^-1): 4 x 64-bit CIOS with
// unsigned __int128; the Montgomery step uses the shape of l (limbs {p0, p1, 0, 2^60}): two products and a shift
// per row instead of four products.  ~3x faster than the generic 64-bit loop it replaced, ~30x faster than emulating
// the 32-bit carry chains.
namespace frh {
typedef unsigned __int128 u128;
struct w4 {
  uint64_t v[4];
};
static const uint64_t kP0 = 0x5812631a5cf5d3edULL, kP1 = 0x14def9dea2f79cd6ULL, kP3 = 0x1000000000000000ULL;
static const uint64_t kInv = 0xd2b51da312547e1bULL;
inline w4 mul(const w4& a, const w4& b) {
  uint64_t t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0, t5;
  for (int i = 0; i < 4; i++) {
    const uint64_t bi = b.v[i];
    u128 c = (u128)a.v[0] * bi + t0;
    t0 = (uint64_t)c;
    c = (c >> 64) + (u128)a.v[1] * bi + t1;
    t1 = (uint64_t)c;
    c = (c >> 64) + (u128)a.v[2] * bi + t2;
    t2 = (uint64_t)c;
    c = (c >> 64) + (u128)a.v[3] * bi + t3;
    t3 = (uint64_t)c;
    c = (c >> 64) + t4;
    t4 = (uint64_t)c;
    t5 = (uint64_t)(c >> 64);
    // t += m * l, then shift one limb: m * l = m*p0 + m*p1*2^64 + m*2^252
    const uint64_t m = t0 * kInv;
    c = ((u128)m * kP0 + t0) >> 64;
    c += (u128)m * kP1 + t1;
    t0 = (uint64_t)c;
    c = (c >> 64) + t2;
    t1 = (uint64_t)c;
    c = (c >> 64) + (u128)t3 + ((u128)m << 60);  // m * 2^60 at limb 3 (spills into limb 4)
    t2 = (uint64_t)c;
    c = (c >> 64) + t4;
    t3 = (uint64_t)c;
    t4 = t5 + (uint64_t)(c >> 64);
  }
  // t < 2l: one conditional subtraction
  uint64_t s0, s1, s2, s3;
  u128 d = (u128)t0 - kP0;
  s0 = (uint64_t)d;
  d = (u128)t1 - kP1 - (uint64_t)((d >> 64) & 1);
  s1 = (uint64_t)d;
  d = (u128)t2 - (uint64_t)((d >> 64) & 1);
  s2 = (uint64_t)d;
  d = (u128)t3 - kP3 - (uint64_t)((d >> 64) & 1);
  s3 = (uint64_t)d;
  const bool ge = t4 != 0 || ((d >> 64) & 1) == 0;
  w4 r;
  r.v[0] = ge ? s0 : t0;
  r.v[1] = ge ? s1 : t1;
  r.v[2] = ge ? s2 : t2;
  r.v[3] = ge ? s3 : t3;
  return r;
}
inline w4 load(const fr_t& a) {
  w4 r;
  for (int i = 0; i < 4; i++) r.v[i] = (uint64_t)a.v[2 * i] | ((uint64_t)a.v[2 * i + 1] << 32);
  return r;
}
inline fr_t store(const w4& a) {
  fr_t r;
  for (int i = 0; i < 4; i++) {
    r.v[2 * i] = (uint32_t)a.v[i];
    r.v[2 * i + 1] = (uint32_t)(a.v[i] >> 32);
  }
  return r;
}
}  // namespace frh
#endif
#if !defined(__CUDA_ARCH__)
inline fr_t fr_mul_host64(const fr_t& A, const fr_t& B) { return frh::store(frh::mul(frh::load(A), frh::load(B))); }
#endif

// the even/odd carry-chain multiplication (device path; also runs on the host for validation)
LB_HD fr_t fr_mul_chain(const fr_t& a, const fr_t& b) {
  uint32_t e[9], o[8], stray = 0;
  fr_mul_row(e, o, stray, a.v, b.v[0], true);
#pragma unroll
  for (int i = 1; i < 8; i++) fr_mul_row(e, o, stray, a.v, b.v[i], false);
  LB_CF_DECL
  uint32_t t[8];
  LB_ADD_CC(t[0], e[0], stray);
  LB_ADDC_CC(t[1], e[1], o[0]);
  LB_ADDC_CC(t[2], e[2], o[1]);
  LB_ADDC_CC(t[3], e[3], o[2]);
  LB_ADDC_CC(t[4], e[4], o[3]);
  LB_ADDC_CC(t[5], e[5], o[4]);
  LB_ADDC_CC(t[6], e[6], o[5]);
  LB_ADDC(t[7], e[7], o[6]);
  return fr_reduce_once(t);
}
// a * b * 2^-256 mod l
LB_HD fr_t fr_mul(const fr_t& a, const fr_t& b) {
#if defined(__CUDA_ARCH__)
  return fr_mul_chain(a, b);
#else
  return fr_mul_host64(a, b);
#endif
}
LB_HD fr_t fr_sqr(const fr_t& a) { return fr_mul(a, a); }

// a * 2^k mod l for 0 <= k <= 31, without a Montgomery multiplication (the weights of combine_lookups are powers of
// two: and.rs:45-53, range_check.rs:78-86).  With l = 2^252 + c, c < 2^125:  a 2^k = top 2^252 + low  ==  low - top c,
// top < 2^(k+1), top c < 2^157 < l — one conditional addition of l makes the result canonical.  The same residue as
// fr_mul(a, fr_from_u64(1 << k)), hence the same bits.
LB_HD fr_t fr_mul_pow2(const fr_t& a, int k) {
  if (k == 0) return a;
  LB_CF_DECL
  uint32_t y[8];
  y[0] = a.v[0] << k;
#pragma unroll
  for (int i = 1; i < 7; i++) y[i] = (a.v[i] << k) | (a.v[i - 1] >> (32 - k));
  const uint64_t y78 = ((uint64_t)a.v[7] << k) | (a.v[6] >> (32 - k));  // a.v[7] < 2^29: below 2^60
  const uint32_t top = (uint32_t)(y78 >> 28);
  y[7] = (uint32_t)y78 & 0x0fffffffu;
  uint32_t m[5];
  uint64_t t = (uint64_t)top * LB_FR_P0;
  m[0] = (uint32_t)t;
  t = (t >> 32) + (uint64_t)top * LB_FR_P1;
  m[1] = (uint32_t)t;
  t = (t >> 32) + (uint64_t)top * LB_FR_P2;
  m[2] = (uint32_t)t;
  t = (t >> 32) + (uint64_t)top * LB_FR_P3;
  m[3] = (uint32_t)t;
  m[4] = (uint32_t)(t >> 32);
  uint32_t d[8], bw;
  LB_SUB_CC(d[0], y[0], m[0]);
  LB_SUBC_CC(d[1], y[1], m[1]);
  LB_SUBC_CC(d[2], y[2], m[2]);
  LB_SUBC_CC(d[3], y[3], m[3]);
  LB_SUBC_CC(d[4], y[4], m[4]);
  LB_SUBC_CC(d[5], y[5], 0u);
  LB_SUBC_CC(d[6], y[6], 0u);
  LB_SUBC_CC(d[7], y[7], 0u);
  LB_SUBC(bw, 0u, 0u);  // all-ones iff low < top c
  fr_t r;
  LB_ADD_CC(r.v[0], d[0], bw & LB_FR_P0);
  LB_ADDC_CC(r.v[1], d[1], bw & LB_FR_P1);
  LB_ADDC_CC(r.v[2], d[2], bw & LB_FR_P2);
  LB_ADDC_CC(r.v[3], d[3], bw & LB_FR_P3);
  LB_ADDC_CC(r.v[4], d[4], 0u);
  LB_ADDC_CC(r.v[5], d[5], 0u);
  LB_ADDC_CC(r.v[6], d[6], 0u);
  LB_ADDC(r.v[7], d[7], bw & LB_FR_P7);
  return r;
}

// F::from(u64): v * R mod l
LB_HD fr_t fr_from_u64(uint64_t x) {
  fr_t t = fr_zero();
  t.v[0] = (uint32_t)x;
  t.v[1] = (uint32_t)(x >> 32);
  return fr_mul(t, fr_r2());
}
// into_bigint: canonical integer limbs
LB_HD fr_t fr_to_canonical(const fr_t& a) {
  fr_t one = fr_zero();
  one.v[0] = 1;
  return fr_mul(a, one);
}
// from a raw < 2^256 integer to Montgomery form
LB_HD fr_t fr_from_raw_int(const fr_t& raw) { return fr_mul(raw, fr_r2()); }


#if !defined(__CUDA_ARCH__)
namespace frh {
// Inversion by exponentiation on 64-bit limbs; l - 2 = 2^252 + (125 bits) is walked with a fixed 4-bit window
// (252 squarings + ~32 multiplications).  The comparator of the binary-GCD inversion below.
inline fr_t inv_fermat(const fr_t& A) {
  // l - 2 = 2^252 + 0x14def9dea2f79cd65812631a5cf5d3eb
  static const uint64_t E[4] = {0x5812631a5cf5d3ebULL, 0x14def9dea2f79cd6ULL, 0x0ULL, 0x1000000000000000ULL};
  w4 tab[16];
  tab[1] = load(A);
  tab[2] = mul(tab[1], tab[1]);
  for (int i = 3; i < 16; i++) tab[i] = mul(tab[i - 1], tab[1]);
  w4 acc = tab[1];  // the top window (bits 252..255) is 1
  for (int w = 62; w >= 0; w--) {
    acc = mul(acc, acc);
    acc = mul(acc, acc);
    acc = mul(acc, acc);
    acc = mul(acc, acc);
    const unsigned d = (unsigned)(E[w >> 4] >> (4 * (w & 15))) & 15u;
    if (d) acc = mul(acc, tab[d]);
  }
  return store(acc);
}
// Inversion on the critical path (u^-1 of every Bulletproofs round, the batching coefficients of a grand-product
// layer): binary extended GCD on the residue (host_modinv.hpp, ~1.8 us against ~7 us for the exponentiation).
// A = a R; the GCD returns A^-1 = a^-1 R^-1 as a plain residue; one Montgomery product with R^3 gives a^-1 R.
inline fr_t inv(const fr_t& A) {
  static const uint64_t kL[4] = {kP0, kP1, 0, kP3};
  static const modinv::Modulus M = modinv::make_modulus(kL);
  static const w4 r3 = mul(load(fr_r2()), load(fr_r2()));  // R^2 * R^2 * R^-1
  w4 y = load(A), x;
  if (!modinv::inverse(y.v, M, x.v)) return inv_fermat(A);
  return store(mul(x, r3));
}
}  // namespace frh
#endif

// a^(l-2)
LB_HD fr_t fr_inv(const fr_t& a) {
#if !defined(__CUDA_ARCH__)
  return frh::inv(a);
#else
  // l - 2 = 2^252 + 0x14def9dea2f79cd65812631a5cf5d3eb
  const uint32_t E[8] = {0x5cf5d3ebu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0, 0, 0, 0x10000000u};
  fr_t acc = fr_one();
  for (int i = 252; i >= 0; i--) {
    acc = fr_sqr(acc);
    if ((E[i >> 5] >> (i & 31)) & 1) acc = fr_mul(acc, a);
  }
  return acc;
#endif
}
// the bitwise square-and-multiply on the portable multiplication (reference for the host fast path)
LB_HD fr_t fr_inv_chain(const fr_t& a) {
  const uint32_t E[8] = {0x5cf5d3ebu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0, 0, 0, 0x10000000u};
  fr_t acc = fr_one();
  for (int i = 252; i >= 0; i--) {
    acc = fr_mul_chain(acc, acc);
    if ((E[i >> 5] >> (i & 31)) & 1) acc = fr_mul_chain(acc, a);
  }
  return acc;
}

}  // namespace lb
