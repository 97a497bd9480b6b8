"""The product's host-side pieces that need no GPU, compiled with g++ straight from the headers:
Merlin transcript (host_transcript.hpp) against the published vector, the 64-bit host field code against the
32-bit carry-chain code that also runs on the device (fr.cuh / fq.cuh / host_fq64.hpp), the wire format of the
tagged device -> host publication (pub_codec.hpp)."""
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lasso_b200", "csrc")

PROG = r'''
#include "host_transcript.hpp"
#include "ed25519.cuh"
#include "host_fq64.hpp"
#include "pub_codec.hpp"
#include <cstdio>
#include <random>
using namespace lb;
int main() {
  // 1. Merlin's published vector
  Transcript t("test protocol");
  t.append_message("some label", std::string("some data"));
  uint8_t o[32];
  t.challenge_bytes("challenge", o, 32);
  for (int i = 0; i < 32; i++) printf("%02x", o[i]);
  printf("\n");
  int bad = 0;
  // 1b. block-wise absorb: random framed messages of every length (0 .. 400 bytes, crossing the 166-byte rate
  // several times) against a byte-at-a-time STROBE written out here
  {
    struct SlowStrobe {
      uint64_t lanes[25];
      int pos = 0, pos_begin = 0;
      uint8_t* b() { return reinterpret_cast<uint8_t*>(lanes); }
      void run_f() {
        b()[pos] ^= (uint8_t)pos_begin; b()[pos + 1] ^= 0x04; b()[167] ^= 0x80;
        KeccakF1600::permute(lanes); pos = 0; pos_begin = 0;
      }
      void absorb(const uint8_t* d, size_t n) { for (size_t i = 0; i < n; i++) { b()[pos] ^= d[i]; if (++pos == 166) run_f(); } }
      void op(uint8_t flags, bool more) {
        if (more) return;
        uint8_t hdr[2] = {(uint8_t)pos_begin, flags};
        pos_begin = pos + 1;
        absorb(hdr, 2);
        if ((flags & (4 | 32)) && pos != 0) run_f();
      }
      explicit SlowStrobe(const std::string& proto) {
        memset(lanes, 0, sizeof(lanes));
        const uint8_t head[6] = {1, 168, 1, 0, 1, 96};
        memcpy(b(), head, 6); memcpy(b() + 6, "STROBEv1.0.2", 12);
        KeccakF1600::permute(lanes);
        op(16 | 2, false); absorb((const uint8_t*)proto.data(), proto.size());
      }
      void msg(const char* label, const uint8_t* m, uint32_t n) {
        op(16 | 2, false); absorb((const uint8_t*)label, strlen(label));
        op(16 | 2, true); absorb((const uint8_t*)&n, 4);
        op(2, false); absorb(m, n);
      }
      void chal(const char* label, uint8_t* out, uint32_t n) {
        op(16 | 2, false); absorb((const uint8_t*)label, strlen(label));
        op(16 | 2, true); absorb((const uint8_t*)&n, 4);
        op(1 | 2 | 4, false);
        for (uint32_t i = 0; i < n; i++) { out[i] = b()[pos]; b()[pos] = 0; if (++pos == 166) run_f(); }
      }
    };
    std::mt19937_64 gg(99);
    Transcript tf("blockwise");  // Transcript's constructor: STROBE("Merlin v1.0") + the "dom-sep" message
    SlowStrobe ts("Merlin v1.0");
    ts.msg("dom-sep", (const uint8_t*)"blockwise", 9);
    int mism = 0;
    std::vector<uint8_t> m(400);
    for (int it = 0; it < 600; it++) {
      uint32_t n = (uint32_t)(gg() % 401);
      for (auto& x : m) x = (uint8_t)gg();
      tf.append_message("lbl", m.data(), n);
      ts.msg("lbl", m.data(), n);
      if (it % 7 == 0) {
        uint8_t o1[64], o2[64];
        tf.challenge_bytes("ch", o1, 64);
        ts.chal("ch", o2, 64);
        if (memcmp(o1, o2, 64)) mism++;
      }
    }
    if (mism) printf("blockwise absorb mismatches: %d\n", mism);
    bad += mism;
  }
  // 1c. the run-time-dispatched permutation (x86-64-v3 build of the same source where the CPU has it) == the
  // portable build, on random states and on the all-zero state iterated
  {
    std::mt19937_64 gk(11);
    int km = 0;
    uint64_t z1[25] = {0}, z2[25] = {0};
    for (int i = 0; i < 2000; i++) {
      uint64_t a1[25], a2[25];
      for (int k = 0; k < 25; k++) a1[k] = a2[k] = gk();
      KeccakF1600::permute(a1);
      KeccakF1600::permute_portable(a2);
      KeccakF1600::permute(z1);
      KeccakF1600::permute_portable(z2);
      if (memcmp(a1, a2, 200) || memcmp(z1, z2, 200)) km++;
    }
    // Keccak-f[1600] of the zero state (first lane of the published KAT)
    uint64_t z[25] = {0};
    KeccakF1600::permute(z);
    if (z[0] != 0xF1258F7940E1DDE7ull) km++;
    if (km) printf("keccak dispatch mismatches: %d\n", km);
    bad += km;
  }
  // 2. fast host Fr (64-bit limbs) == even/odd carry-chain multiplication (the device algorithm)
  std::mt19937_64 g(7);
  fr_t a = fr_from_u64(g()), b = fr_from_u64(g());
  for (int i = 0; i < 20000; i++) {
    fr_t m1 = fr_mul(a, b), m2 = fr_mul_chain(a, b);
    if (!fr_eq(m1, m2)) bad++;
    a = fr_add(m1, b);
    b = fr_sub(m2, fr_from_u64(g()));
  }
  // fr_inv (host: 64-bit limbs, 4-bit window) == bitwise square-and-multiply on the carry-chain multiplication
  for (int i = 0; i < 300; i++) {
    fr_t x = fr_add(fr_mul(a, fr_from_u64(g())), fr_from_u64(g()));
    fr_t i1 = fr_inv(x), i2 = fr_inv_chain(x);
    if (!fr_eq(i1, i2) || !fr_eq(fr_mul(x, i1), fr_one())) bad++;
    a = x;
  }
  {
    fr_t one = fr_one(), m1 = fr_sub(fr_zero(), one);
    if (!fr_eq(fr_inv(one), one) || !fr_eq(fr_inv(m1), m1)) bad++;
  }
  // 2c. a * 2^k by shift-and-fold == Montgomery multiplication by F::from(1 << k), every k the weights of
  // combine_lookups can take, on random elements and on the edges 0, 1, -1, l - 2^j
  {
    int pm = 0;
    std::vector<fr_t> xs = {fr_zero(), fr_one(), fr_sub(fr_zero(), fr_one()), fr_from_u64(1), fr_sub(fr_zero(), fr_from_u64(1))};
    fr_t x = a;
    for (int i = 0; i < 3000; i++) {
      x = fr_add(fr_mul(x, b), fr_from_u64(g()));
      xs.push_back(x);
    }
    for (int j = 0; j < 64; j++) xs.push_back(fr_sub(fr_zero(), fr_from_u64(1ull << j)));
    for (const fr_t& v : xs)
      for (int k = 0; k <= 31; k++)
        if (!fr_eq(fr_mul_pow2(v, k), fr_mul(v, fr_from_u64(1ull << k)))) pm++;
    // also on raw residues just below l and at 2^252 (Montgomery form is just another residue)
    fr_t top = {{LB_FR_P0 - 1, LB_FR_P1, LB_FR_P2, LB_FR_P3, 0, 0, 0, LB_FR_P7}}, mid = {{0, 0, 0, 0, 0, 0, 0, 0x10000000u}};
    for (int k = 0; k <= 31; k++) {
      if (!fr_eq(fr_mul_pow2(top, k), fr_mul(top, fr_from_u64(1ull << k)))) pm++;
      if (!fr_eq(fr_mul_pow2(mid, k), fr_mul(mid, fr_from_u64(1ull << k)))) pm++;
    }
    if (pm) printf("fr_mul_pow2 mismatches: %d\n", pm);
    bad += pm;
  }
  // 2d. binary-GCD inversion (host_modinv.hpp) == the exponentiation, for both fields: zero, +-1, +-2^j, small values,
  // non-canonical Fq inputs (q, q + 1, 2^256 - 1) and random elements
  {
    int im = 0;
    auto chk_fr = [&](const fr_t& v) {
      const fr_t i1 = fr_inv(v), i2 = frh::inv_fermat(v);
      if (!fr_eq(i1, i2)) im++;
      if (!fr_is_zero(v) && !fr_eq(fr_mul(v, i1), fr_one())) im++;
    };
    chk_fr(fr_zero());
    chk_fr(fr_one());
    chk_fr(fr_sub(fr_zero(), fr_one()));
    for (int j = 0; j < 64; j++) {
      chk_fr(fr_from_u64(1ull << j));
      chk_fr(fr_sub(fr_zero(), fr_from_u64(1ull << j)));
    }
    for (int j = 0; j < 252; j++) {  // raw residues 2^j (any residue below l is an element in memory format)
      fr_t t = fr_zero();
      t.v[j >> 5] = 1u << (j & 31);
      chk_fr(t);
    }
    for (uint64_t k = 1; k < 300; k++) chk_fr(fr_from_u64(k));
    fr_t x = a;
    for (int i = 0; i < 20000; i++) {
      x = fr_add(fr_mul(x, b), fr_from_u64(g()));
      chk_fr(x);
    }
    auto chk_fq = [&](const uint64_t y[4]) {
      h64::fe Y;
      memcpy(Y.v, y, 32);
      const h64::fe i1 = h64::inv(Y), i2 = h64::canonical(h64::inv_fermat(Y));
      if (memcmp(i1.v, i2.v, 32)) im++;
    };
    const uint64_t q[4] = {0xffffffffffffffedULL, 0xffffffffffffffffULL, 0xffffffffffffffffULL, 0x7fffffffffffffffULL};
    uint64_t y[4] = {0, 0, 0, 0};
    chk_fq(y);
    chk_fq(q);
    memcpy(y, q, 32);
    y[0] += 1;
    chk_fq(y);
    for (int i = 0; i < 4; i++) y[i] = ~0ULL;
    chk_fq(y);
    for (int j = 0; j < 256; j++) {
      uint64_t t[4] = {0, 0, 0, 0};
      t[j >> 6] = 1ULL << (j & 63);
      chk_fq(t);
      t[0] |= 1;
      chk_fq(t);
    }
    for (uint64_t k = 1; k < 300; k++) {
      uint64_t t[4] = {k, 0, 0, 0};
      chk_fq(t);
    }
    for (int i = 0; i < 20000; i++) {
      uint64_t t[4] = {g(), g(), g(), g()};
      if (i & 1) t[3] >>= (i % 64);
      chk_fq(t);
    }
    if (im) printf("modinv mismatches: %d\n", im);
    bad += im;
  }
  // 3. host Fq64 normalisation == device-code normalisation + ark compression
  fq_t bx = {{0x8f25d51au, 0xc9562d60u, 0x9525a7b2u, 0x692cc760u, 0xfdd6dc5cu, 0xc0a4e231u, 0xcd6e53feu, 0x216936d3u}};
  fq_t by = {{0x66666658u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u}};
  pt_niels n = niels_from_affine(bx, by);
  pt_ext acc = pt_identity();
  for (int i = 0; i < 100; i++) {
    acc = pt_madd(pt_dbl(acc), n);
    fq_t x, y;
    pt_to_affine_canonical(acc, x, y);
    uint32_t c[8];
    pt_compress_canonical(x, y, c);
    uint32_t xyz[32];
    memcpy(xyz, acc.X.v, 32); memcpy(xyz + 8, acc.Y.v, 32); memcpy(xyz + 16, acc.Z.v, 32); memcpy(xyz + 24, acc.T.v, 32);
    uint8_t h[32];
    h64::compress_xyz(xyz, h);
    if (memcmp(h, c, 32)) bad++;
    // pair version (one inversion for two points) against the single one: this point and its double
    pt_ext dbl = pt_dbl(acc);
    uint32_t xyz2[32];
    memcpy(xyz2, dbl.X.v, 32); memcpy(xyz2 + 8, dbl.Y.v, 32); memcpy(xyz2 + 16, dbl.Z.v, 32); memcpy(xyz2 + 24, dbl.T.v, 32);
    uint8_t h2[32], pa[32], pb[32];
    h64::compress_xyz(xyz2, h2);
    h64::compress_xyz_pair(xyz, xyz2, pa, pb);
    if (memcmp(pa, h, 32) || memcmp(pb, h2, 32)) bad++;
  }
  // 4. wire format of a tagged publication (pub_codec.hpp): encode -> five self-identifying words -> decode, for
  // random values below 2^255, every tag class, and the edge values; a word of another message is never accepted
  {
    std::mt19937_64 g(99);
    for (int it = 0; it < 20000; it++) {
      uint32_t x[8], y[8];
      for (int l = 0; l < 8; l++) x[l] = (uint32_t)g();
      if (it == 0) for (int l = 0; l < 8; l++) x[l] = 0;
      if (it == 1) for (int l = 0; l < 8; l++) x[l] = 0xffffffffu;
      x[7] &= 0x7fffffffu;  // < 2^255
      const uint32_t tag = 1 + (uint32_t)(g() % 8191);
      unsigned long long w[5], v[5];
      pub_encode(x, tag, w);
      for (int k = 0; k < 5; k++) {
        if (pub_tag_of(w[k]) != tag || pub_tag_of(w[k]) == 0) bad++;
        if (pub_tag_of(w[k]) == (tag % 8191) + 1) bad++;  // the next message's tag differs in every word
        v[k] = w[k] & kPubValueMask;
      }
      pub_decode(v, y);
      if (memcmp(x, y, 32)) bad++;
    }
  }
  printf("bad=%d\n", bad);
  return bad;
}
'''


def test_host_transcript_and_field_code():
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "t.cpp")
        open(src, "w").write(PROG)
        exe = os.path.join(d, "t")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wno-psabi", "-I", CSRC, src, "-o", exe])
        out = subprocess.run([exe], capture_output=True, text=True)
        lines = out.stdout.strip().splitlines()
        assert lines[0] == "d5a21972d0d5fe320c0d263fac7fffb8145aa640af6e9bca177c03c7efcf0615"
        assert lines[1] == "bad=0" and out.returncode == 0


def test_portable_build_of_the_host_code():
    """The same program with the run-time dispatch compiled out (LB_KECCAK_NO_DISPATCH: what a non-x86 host or a CPU
    without AVX2 / BMI2 runs): same Merlin vector, same checks."""
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "t.cpp")
        open(src, "w").write(PROG)
        exe = os.path.join(d, "t")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wno-psabi", "-DLB_KECCAK_NO_DISPATCH", "-I", CSRC, src, "-o", exe])
        out = subprocess.run([exe], capture_output=True, text=True)
        lines = out.stdout.strip().splitlines()
        assert lines[0] == "d5a21972d0d5fe320c0d263fac7fffb8145aa640af6e9bca177c03c7efcf0615"
        assert lines[1] == "bad=0" and out.returncode == 0


def test_host_microbenchmark_builds():
    """tools/hostbench/host_bench.cpp (the host-side microbenchmark) keeps compiling from the headers."""
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "hb")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-psabi", "-I", CSRC,
                               os.path.join(ROOT, "tools", "hostbench", "host_bench.cpp"), "-o", exe])
        assert os.path.exists(exe)


def test_kernel_microbenchmark_builds():
    """tools/ubench (the kernel microbenchmarks, linked against the library's kernel objects) keeps compiling against the
    current launcher interfaces."""
    objs = [os.path.join(ROOT, "lasso_b200", "_build", o) for o in ("poly_kernels.o", "msm_kernels.o")]
    if shutil.which("nvcc") is None or not all(os.path.exists(o) for o in objs):
        pytest.skip("needs nvcc and the library objects under lasso_b200/_build (run build() first)")
    subprocess.check_call(["make", "-s", "-B", "-C", os.path.join(ROOT, "tools", "ubench")])
    assert os.path.exists(os.path.join(ROOT, "tools", "ubench", "kbench"))
