// The field and group primitives of fr.cuh, fq.cuh and ed25519.cuh, one operation per element, for comparison with
// plain integers (tests/test_gpu_arith.py on the device, tests/test_arith_host.py compiled with g++ on the host).
// The bodies are LB_HD, so the same source runs on both sides; the quad-lane forms of quad.cuh use warp shuffles and
// live in arith_kernels.cuh only.
//
// Element layout: a, b and out are 32 u32 (128 B) per element, k one u64.  A field element is 8 u32 (fr_t: Montgomery
// limbs; fq_t: the internal, loosely reduced integer), a point its coordinates in order: pt_ext X, Y, Z, T; pt_niels
// y+x, y-x, 2dxy; affine x, y.  A boolean result is out[0].
#pragma once
#include "../../lasso_b200/csrc/ed25519.cuh"

// X(name): operations applied by one thread to one element
#define KH_ARITH_THREAD_OPS(X)                                                                                      \
  X(fr_add) X(fr_sub) X(fr_neg) X(fr_dbl) X(fr_mul) X(fr_mul_chain) X(fr_sqr) X(fr_mul_pow2) X(fr_from_u64)           \
  X(fr_to_canonical) X(fr_eq) X(fr_is_zero) X(fr_from_raw_int) X(fr_inv)                                             \
  X(fq_add) X(fq_sub) X(fq_neg) X(fq_dbl) X(fq_mul) X(fq_sqr) X(fq_mul_small) X(fq_canonical) X(fq_is_zero)           \
  X(fq_equal) X(fq_inv) X(fq_from_ark) X(fq_to_ark)                                                                  \
  X(niels_from_affine) X(niels_from_ark_affine) X(niels_neg) X(pt_madd) X(pt_msub) X(pt_add) X(pt_dbl) X(pt_neg)    \
  X(pt_from_niels) X(pt_to_affine_canonical) X(pt_compress_canonical)
// operations applied by the four lanes of a quad to one element (device only)
#define KH_ARITH_QUAD_OPS(X) X(quad_add) X(quad_madd) X(quad_dbl)

namespace arith {

enum Op {
#define KH_ARITH_ENUM(name) OP_##name,
  KH_ARITH_THREAD_OPS(KH_ARITH_ENUM) KH_ARITH_QUAD_OPS(KH_ARITH_ENUM)
#undef KH_ARITH_ENUM
  OP_COUNT
};

inline const char* op_name(int op) {
  static const char* const names[] = {
#define KH_ARITH_NAME(name) #name,
      KH_ARITH_THREAD_OPS(KH_ARITH_NAME) KH_ARITH_QUAD_OPS(KH_ARITH_NAME)
#undef KH_ARITH_NAME
  };
  return op >= 0 && op < OP_COUNT ? names[op] : nullptr;
}

using lb::fq_t;
using lb::fr_t;
using lb::pt_ext;
using lb::pt_niels;

// element-wise copies: the host side reads numpy buffers, which need not have fq_t's 32-byte alignment
LB_HD fq_t ldq(const uint32_t* p, int i) {
  fq_t r;
#pragma unroll
  for (int l = 0; l < 8; l++) r.v[l] = p[8 * i + l];
  return r;
}
LB_HD void stq(uint32_t* p, int i, const fq_t& x) {
#pragma unroll
  for (int l = 0; l < 8; l++) p[8 * i + l] = x.v[l];
}
LB_HD fr_t ldr(const uint32_t* p) {
  fr_t r;
#pragma unroll
  for (int l = 0; l < 8; l++) r.v[l] = p[l];
  return r;
}
LB_HD void str(uint32_t* p, const fr_t& x) {
#pragma unroll
  for (int l = 0; l < 8; l++) p[l] = x.v[l];
}
LB_HD pt_ext ldp(const uint32_t* p) {
  pt_ext r;
  r.X = ldq(p, 0);
  r.Y = ldq(p, 1);
  r.Z = ldq(p, 2);
  r.T = ldq(p, 3);
  return r;
}
LB_HD void stp(uint32_t* p, const pt_ext& r) {
  stq(p, 0, r.X);
  stq(p, 1, r.Y);
  stq(p, 2, r.Z);
  stq(p, 3, r.T);
}
LB_HD pt_niels ldn(const uint32_t* p) {
  pt_niels n;
  n.yplusx = ldq(p, 0);
  n.yminusx = ldq(p, 1);
  n.t2d = ldq(p, 2);
  return n;
}
LB_HD void stn(uint32_t* p, const pt_niels& n) {
  stq(p, 0, n.yplusx);
  stq(p, 1, n.yminusx);
  stq(p, 2, n.t2d);
}

// one thread operation on one element; `op` is a compile-time constant in the device kernels, so each one inlines
// a single case
LB_HD void apply(int op, const uint32_t* a, const uint32_t* b, uint64_t k, uint32_t* o) {
  using namespace lb;
  switch (op) {
    case OP_fr_add: str(o, fr_add(ldr(a), ldr(b))); break;
    case OP_fr_sub: str(o, fr_sub(ldr(a), ldr(b))); break;
    case OP_fr_neg: str(o, fr_neg(ldr(a))); break;
    case OP_fr_dbl: str(o, fr_dbl(ldr(a))); break;
    case OP_fr_mul: str(o, fr_mul(ldr(a), ldr(b))); break;
    case OP_fr_mul_chain: str(o, fr_mul_chain(ldr(a), ldr(b))); break;
    case OP_fr_sqr: str(o, fr_sqr(ldr(a))); break;
    case OP_fr_mul_pow2: str(o, fr_mul_pow2(ldr(a), (int)k)); break;
    case OP_fr_from_u64: str(o, fr_from_u64(k)); break;
    case OP_fr_to_canonical: str(o, fr_to_canonical(ldr(a))); break;
    case OP_fr_eq: o[0] = fr_eq(ldr(a), ldr(b)) ? 1u : 0u; break;
    case OP_fr_is_zero: o[0] = fr_is_zero(ldr(a)) ? 1u : 0u; break;
    case OP_fr_from_raw_int: str(o, fr_from_raw_int(ldr(a))); break;
    case OP_fr_inv: str(o, fr_inv(ldr(a))); break;
    case OP_fq_add: stq(o, 0, fq_add(ldq(a, 0), ldq(b, 0))); break;
    case OP_fq_sub: stq(o, 0, fq_sub(ldq(a, 0), ldq(b, 0))); break;
    case OP_fq_neg: stq(o, 0, fq_neg(ldq(a, 0))); break;
    case OP_fq_dbl: stq(o, 0, fq_dbl(ldq(a, 0))); break;
    case OP_fq_mul: stq(o, 0, fq_mul(ldq(a, 0), ldq(b, 0))); break;
    case OP_fq_sqr: stq(o, 0, fq_sqr(ldq(a, 0))); break;
    case OP_fq_mul_small: stq(o, 0, fq_mul_small(ldq(a, 0), (uint32_t)k)); break;
    case OP_fq_canonical: stq(o, 0, fq_canonical(ldq(a, 0))); break;
    case OP_fq_is_zero: o[0] = fq_is_zero(ldq(a, 0)) ? 1u : 0u; break;
    case OP_fq_equal: o[0] = fq_equal(ldq(a, 0), ldq(b, 0)) ? 1u : 0u; break;
    case OP_fq_inv: stq(o, 0, fq_inv(ldq(a, 0))); break;
    case OP_fq_from_ark: stq(o, 0, fq_from_ark(ldq(a, 0))); break;
    case OP_fq_to_ark: stq(o, 0, fq_to_ark(ldq(a, 0))); break;
    case OP_niels_from_affine: stn(o, niels_from_affine(ldq(a, 0), ldq(a, 1))); break;
    case OP_niels_from_ark_affine: stn(o, niels_from_ark_affine(ldq(a, 0), ldq(a, 1))); break;
    case OP_niels_neg: stn(o, niels_neg(ldn(a))); break;
    case OP_pt_madd: stp(o, pt_madd(ldp(a), ldn(b))); break;
    case OP_pt_msub: stp(o, pt_msub(ldp(a), ldn(b))); break;
    case OP_pt_add: stp(o, pt_add(ldp(a), ldp(b))); break;
    case OP_pt_dbl: stp(o, pt_dbl(ldp(a))); break;
    case OP_pt_neg: stp(o, pt_neg(ldp(a))); break;
    case OP_pt_from_niels: stp(o, pt_from_niels(ldn(a))); break;
    case OP_pt_to_affine_canonical: {
      fq_t x, y;
      pt_to_affine_canonical(ldp(a), x, y);
      stq(o, 0, x);
      stq(o, 1, y);
      break;
    }
    case OP_pt_compress_canonical: pt_compress_canonical(ldq(a, 0), ldq(a, 1), o); break;
    default: break;
  }
}

}  // namespace arith
