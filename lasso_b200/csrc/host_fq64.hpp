// lasso_b200 — host-side Fq = GF(2^255 - 19) on 4 x 64-bit limbs (unsigned __int128), used only to
// normalise / compress the one or two group elements a Bulletproofs round sends to the transcript:
// a single Fq inversion is ~2 us on a CPU core (binary GCD) against a 265-step serial chain on one GPU thread.
// Values are plain (non-Montgomery) integers, loosely reduced below 2^256 like the device code (fq.cuh).
#pragma once
#include <cstdint>
#include <cstring>

#include "host_modinv.hpp"

namespace lb {
namespace h64 {

typedef unsigned __int128 u128;
struct fe {
  uint64_t v[4];
};

inline fe from_limbs32(const uint32_t* p) {
  fe r;
  memcpy(r.v, p, 32);
  return r;
}
inline void fold(uint64_t t[4], uint64_t c) {  // t += 38 * c, twice
  u128 acc = (u128)c * 38;
  for (int i = 0; i < 4; i++) {
    acc += t[i];
    t[i] = (uint64_t)acc;
    acc >>= 64;
  }
  t[0] += (uint64_t)acc * 38;  // second wrap cannot ripple (value is tiny when it happens)
}
inline fe mul(const fe& a, const fe& b) {
  uint64_t p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    u128 c = 0;
    for (int j = 0; j < 4; j++) {
      c += (u128)a.v[j] * b.v[i] + p[i + j];
      p[i + j] = (uint64_t)c;
      c >>= 64;
    }
    p[i + 4] = (uint64_t)c;
  }
  fe r;
  u128 c = 0;
  for (int k = 0; k < 4; k++) {
    c += (u128)p[4 + k] * 38 + p[k];
    r.v[k] = (uint64_t)c;
    c >>= 64;
  }
  fold(r.v, (uint64_t)c);
  return r;
}
inline fe sqr_n(fe a, int n) {
  for (int i = 0; i < n; i++) a = mul(a, a);
  return a;
}
inline fe inv_fermat(const fe& z) {  // z^(2^255 - 21): the comparator of inv() below
  fe z2 = mul(z, z);
  fe z9 = mul(sqr_n(z2, 2), z);
  fe z11 = mul(z9, z2);
  fe z2_5_0 = mul(mul(z11, z11), z9);
  fe z2_10_0 = mul(sqr_n(z2_5_0, 5), z2_5_0);
  fe z2_20_0 = mul(sqr_n(z2_10_0, 10), z2_10_0);
  fe z2_40_0 = mul(sqr_n(z2_20_0, 20), z2_20_0);
  fe z2_50_0 = mul(sqr_n(z2_40_0, 10), z2_10_0);
  fe z2_100_0 = mul(sqr_n(z2_50_0, 50), z2_50_0);
  fe z2_200_0 = mul(sqr_n(z2_100_0, 100), z2_100_0);
  fe z2_250_0 = mul(sqr_n(z2_200_0, 50), z2_50_0);
  return mul(sqr_n(z2_250_0, 5), z11);
}
inline fe canonical(const fe& a);
// z^-1 as a canonical residue by binary extended GCD (host_modinv.hpp): ~1.8 us against ~6 us for the exponentiation
inline fe inv(const fe& z) {
  static const uint64_t kQ[4] = {0xffffffffffffffedULL, 0xffffffffffffffffULL, 0xffffffffffffffffULL, 0x7fffffffffffffffULL};
  static const modinv::Modulus M = modinv::make_modulus(kQ);
  fe r;
  if (!modinv::inverse(z.v, M, r.v)) return canonical(inv_fermat(z));
  return r;
}
inline fe canonical(const fe& a) {
  uint64_t t[4] = {a.v[0], a.v[1], a.v[2], a.v[3]};
  for (int rep = 0; rep < 2; rep++) {
    uint64_t top = t[3] >> 63;
    t[3] &= 0x7fffffffffffffffULL;
    u128 c = (u128)top * 19;
    for (int i = 0; i < 4; i++) {
      c += t[i];
      t[i] = (uint64_t)c;
      c >>= 64;
    }
  }
  uint64_t s[4];
  u128 c = 19;
  for (int i = 0; i < 4; i++) {
    c += t[i];
    s[i] = (uint64_t)c;
    c >>= 64;
  }
  bool ge = (s[3] >> 63) != 0;
  s[3] &= 0x7fffffffffffffffULL;
  fe r;
  for (int i = 0; i < 4; i++) r.v[i] = ge ? s[i] : t[i];
  return r;
}
// Whether a 32-byte ark-serialize compressed point decompresses (get_point_from_y_unchecked): y below q, and
// x^2 = (y^2 - 1) / (d y^2 + 1) a square (Euler's criterion), d = -121665/121666.  Not a subgroup check.
inline bool decompresses(const uint8_t in[32]) {
  static const uint64_t kQm1[4] = {0xffffffffffffffecULL, 0xffffffffffffffffULL, 0xffffffffffffffffULL, 0x7fffffffffffffffULL};
  static const fe kD = {{0x75eb4dca135978a3ULL, 0x00700a4d4141d8abULL, 0x8cc740797779e898ULL, 0x52036cee2b6ffe73ULL}};
  fe y;
  memcpy(y.v, in, 32);
  y.v[3] &= 0x7fffffffffffffffULL;
  for (int i = 3; i >= 0; i--) {  // y < q = (q - 1) + 1
    if (y.v[i] != kQm1[i]) {
      if (y.v[i] > kQm1[i]) return false;
      break;
    }
    if (i == 0) return false;
  }
  auto add = [](const fe& a, const uint64_t* b) {  // a, b < 2^255: the sum fits 256 bits
    fe r;
    u128 c = 0;
    for (int i = 0; i < 4; i++) {
      c += (u128)a.v[i] + b[i];
      r.v[i] = (uint64_t)c;
      c >>= 64;
    }
    return canonical(r);
  };
  const uint64_t one[4] = {1, 0, 0, 0};
  const fe y2 = canonical(mul(y, y));
  const fe num = add(y2, kQm1), den = add(canonical(mul(kD, y2)), one);
  if (!(den.v[0] | den.v[1] | den.v[2] | den.v[3])) return false;
  const fe x2 = mul(num, inv(den));
  fe e = {{1, 0, 0, 0}}, b = x2;  // x2^((q - 1) / 2), the exponent 2^254 - 10 taken bit by bit
  static const uint64_t kE[4] = {0xfffffffffffffff6ULL, 0xffffffffffffffffULL, 0xffffffffffffffffULL, 0x3fffffffffffffffULL};
  for (int i = 0; i < 256; i++) {
    if ((kE[i / 64] >> (i % 64)) & 1) e = mul(e, b);
    b = mul(b, b);
  }
  e = canonical(e);
  return e.v[1] == 0 && e.v[2] == 0 && e.v[3] == 0 && e.v[0] <= 1;
}
// (X, Y, Z) internal limbs (3 x 8 u32) -> ark-serialize compressed point (32 bytes)
inline void compress_xyz(const uint32_t* xyz, uint8_t out[32]) {
  fe X = from_limbs32(xyz), Y = from_limbs32(xyz + 8), Z = from_limbs32(xyz + 16);
  fe zi = inv(Z);
  fe x = canonical(mul(X, zi)), y = canonical(mul(Y, zi));
  // x > (q-1)/2  <=>  x + 9 >= 2^254
  u128 c = 9;
  uint64_t top = 0;
  for (int i = 0; i < 4; i++) {
    c += x.v[i];
    top = (uint64_t)c;
    c >>= 64;
  }
  bool neg = (top >> 62) != 0;
  memcpy(out, y.v, 32);
  if (neg) out[31] |= 0x80;
}
// Two points at once (L and R of a Bulletproofs round): one inversion for both (Montgomery's trick)
inline void compress_xyz_pair(const uint32_t* xyz_a, const uint32_t* xyz_b, uint8_t out_a[32], uint8_t out_b[32]) {
  const fe Za = from_limbs32(xyz_a + 16), Zb = from_limbs32(xyz_b + 16);
  const fe zi = inv(mul(Za, Zb));
  const fe zia = mul(zi, Zb), zib = mul(zi, Za);
  const uint32_t* src[2] = {xyz_a, xyz_b};
  const fe* z[2] = {&zia, &zib};
  uint8_t* dst[2] = {out_a, out_b};
  for (int k = 0; k < 2; k++) {
    const fe x = canonical(mul(from_limbs32(src[k]), *z[k])), y = canonical(mul(from_limbs32(src[k] + 8), *z[k]));
    u128 c = 9;  // x > (q-1)/2  <=>  x + 9 >= 2^254
    uint64_t top = 0;
    for (int i = 0; i < 4; i++) {
      c += x.v[i];
      top = (uint64_t)c;
      c >>= 64;
    }
    memcpy(dst[k], y.v, 32);
    if ((top >> 62) != 0) dst[k][31] |= 0x80;
  }
}
// k <= 8 points (k x 24 words) at once (the rows of one short MSM): one inversion for all of them (Montgomery's trick)
inline void compress_xyz_batch(const uint32_t* xyz, int k, uint8_t* out /* k x 32 */) {
  fe pre[8], zi[8];  // pre[i] = Z_0 .. Z_{i-1}
  fe acc = {{1, 0, 0, 0}};
  for (int i = 0; i < k; i++) {
    pre[i] = acc;
    acc = mul(acc, from_limbs32(xyz + 24 * i + 16));
  }
  fe inv_acc = inv(acc);  // 1 / (Z_0 .. Z_{i})
  for (int i = k - 1; i >= 0; i--) {
    zi[i] = mul(inv_acc, pre[i]);
    inv_acc = mul(inv_acc, from_limbs32(xyz + 24 * i + 16));
  }
  for (int i = 0; i < k; i++) {
    const fe x = canonical(mul(from_limbs32(xyz + 24 * i), zi[i])), y = canonical(mul(from_limbs32(xyz + 24 * i + 8), zi[i]));
    u128 c = 9;  // x > (q-1)/2  <=>  x + 9 >= 2^254
    uint64_t top = 0;
    for (int l = 0; l < 4; l++) {
      c += x.v[l];
      top = (uint64_t)c;
      c >>= 64;
    }
    memcpy(out + 32 * i, y.v, 32);
    if ((top >> 62) != 0) out[32 * i + 31] |= 0x80;
  }
}

}  // namespace h64
}  // namespace lb
