// lasso_b200 — host-side Fiat–Shamir transcript for the prover: Merlin (STROBE-128 over
// Keccak-f[1600]) with the reference's ProofTranscript conventions
// (/root/reference/src/utils/transcript.rs:20-72) and RandomTape (utils/random.rs:9-39).
// BASELINE's north star keeps the transcript on the host; the GPU only ever sees challenges.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "fr.cuh"

namespace lb {

// The permutation is the host's largest single cost inside a proof (a 2^20-lookup proof absorbs ~0.7 MB through
// 4337 permutations: four 2048-scalar `a` vectors, the commitments, every round message and challenge), and it is
// on the critical path between kernel launches.  On x86-64 the same source (keccak_f1600_body.inc) is compiled a
// second time for x86-64-v3 (ANDN for chi, RORX for rho, three-operand forms: -35 % on an absorb) and chosen at run time.
#if defined(__x86_64__) && defined(__GNUC__) && !defined(__CUDA_ARCH__) && !defined(LB_KECCAK_NO_DISPATCH)
#define LB_KECCAK_DISPATCH 1
#else
#define LB_KECCAK_DISPATCH 0
#endif
class KeccakF1600 {
 public:
  static void permute(uint64_t s[25]) {
#if LB_KECCAK_DISPATCH
    static const bool fast = __builtin_cpu_supports("avx2") && __builtin_cpu_supports("bmi") &&
                             __builtin_cpu_supports("bmi2") && __builtin_cpu_supports("fma");
    if (fast) {
      permute_v3(s);
      return;
    }
#endif
    permute_portable(s);
  }
  static void permute_portable(uint64_t s[25]) {  // baseline x86-64 / any other host (and the tests' comparator)
#include "keccak_f1600_body.inc"
  }

 private:
#if LB_KECCAK_DISPATCH
  __attribute__((target("arch=x86-64-v3"), noinline)) static void permute_v3(uint64_t s[25]) {
#include "keccak_f1600_body.inc"
  }
#endif
};

// STROBE-128/1600 restricted to the operations Merlin uses (AD, meta-AD, PRF).
class Strobe {
 public:
  explicit Strobe(const std::string& proto) {
    memset(lanes_, 0, sizeof(lanes_));
    uint8_t* s = bytes();
    const uint8_t head[6] = {1, kRate + 2, 1, 0, 1, 96};
    memcpy(s, head, 6);
    memcpy(s + 6, "STROBEv1.0.2", 12);
    KeccakF1600::permute(lanes_);
    op(kFlagM | kFlagA, false);
    absorb(reinterpret_cast<const uint8_t*>(proto.data()), proto.size());
  }
  void meta_ad(const void* d, size_t n, bool more) {
    op(kFlagM | kFlagA, more);
    absorb(static_cast<const uint8_t*>(d), n);
  }
  void ad(const void* d, size_t n) {
    op(kFlagA, false);
    absorb(static_cast<const uint8_t*>(d), n);
  }
  void prf(uint8_t* out, size_t n) {
    op(kFlagI | kFlagA | kFlagC, false);
    uint8_t* s = bytes();
    for (size_t i = 0; i < n; i++) {
      out[i] = s[pos_];
      s[pos_] = 0;
      if (++pos_ == kRate) run_f();
    }
  }

 private:
  static constexpr int kRate = 166;
  static constexpr uint8_t kFlagI = 1, kFlagA = 2, kFlagC = 4, kFlagT = 8, kFlagM = 16, kFlagK = 32;
  uint64_t lanes_[25];
  int pos_ = 0, pos_begin_ = 0;
  uint8_t cur_flags_ = 0;
  uint8_t* bytes() { return reinterpret_cast<uint8_t*>(lanes_); }
  void run_f() {
    uint8_t* s = bytes();
    s[pos_] ^= (uint8_t)pos_begin_;
    s[pos_ + 1] ^= 0x04;
    s[kRate + 1] ^= 0x80;
    KeccakF1600::permute(lanes_);
    pos_ = 0;
    pos_begin_ = 0;
  }
  // XOR the message into the rate portion, a block at a time (the 64 KB `a` vector of every opening goes through
  // here as 2048 framed messages: 8 bytes per step instead of one)
  void absorb(const uint8_t* d, size_t n) {
    uint8_t* s = bytes();
    while (n) {
      size_t take = (size_t)(kRate - pos_);
      if (take > n) take = n;
      uint8_t* dst = s + pos_;
      size_t i = 0;
      for (; i + 8 <= take; i += 8) {
        uint64_t a, b;
        memcpy(&a, dst + i, 8);
        memcpy(&b, d + i, 8);
        a ^= b;
        memcpy(dst + i, &a, 8);
      }
      for (; i < take; i++) dst[i] ^= d[i];
      pos_ += (int)take;
      d += take;
      n -= take;
      if (pos_ == kRate) run_f();
    }
  }
  void op(uint8_t flags, bool more) {
    if (more) return;  // continuation of the previous operation
    uint8_t hdr[2] = {(uint8_t)pos_begin_, flags};
    pos_begin_ = pos_ + 1;
    cur_flags_ = flags;
    absorb(hdr, 2);
    if ((flags & (kFlagC | kFlagK)) && pos_ != 0) run_f();
  }
};

inline void fr_to_bytes(const fr_t& a, uint8_t out[32]) {  // ark serialize_compressed: 32 B LE canonical
  fr_t c = fr_to_canonical(a);
  memcpy(out, c.v, 32);
}
// PrimeField::from_le_bytes_mod_order over 64 bytes: lo + hi * 2^256 mod l
inline fr_t fr_from_bytes64(const uint8_t in[64]) {
  fr_t lo, hi;
  memcpy(lo.v, in, 32);
  memcpy(hi.v, in + 32, 32);
  fr_t r2 = fr_r2();
  return fr_add(fr_mul(lo, r2), fr_mul(fr_mul(hi, r2), r2));
}

class Transcript {
 public:
  explicit Transcript(const std::string& label) : strobe_("Merlin v1.0") { append_message("dom-sep", label); }
  void append_message(const char* label, const void* msg, size_t n) {
    uint32_t len = (uint32_t)n;
    strobe_.meta_ad(label, strlen(label), false);
    strobe_.meta_ad(&len, 4, true);  // little-endian host
    strobe_.ad(msg, n);
  }
  void append_message(const char* label, const std::string& msg) { append_message(label, msg.data(), msg.size()); }
  void challenge_bytes(const char* label, uint8_t* out, size_t n) {
    uint32_t len = (uint32_t)n;
    strobe_.meta_ad(label, strlen(label), false);
    strobe_.meta_ad(&len, 4, true);
    strobe_.prf(out, n);
  }
  void append_u64(const char* label, uint64_t x) {  // merlin: the 8 little-endian bytes
    uint8_t b[8];
    for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i));
    append_message(label, b, 8);
  }
  void append_protocol_name(const char* name) { append_message("protocol-name", std::string(name)); }
  void append_scalar(const char* label, const fr_t& s) {
    uint8_t b[32];
    fr_to_bytes(s, b);
    append_message(label, b, 32);
  }
  void append_scalars(const char* label, const fr_t* v, size_t n) {
    append_message(label, std::string("begin_append_vector"));
    for (size_t i = 0; i < n; i++) append_scalar(label, v[i]);
    append_message(label, std::string("end_append_vector"));
  }
  // canonical scalars already serialised (32 B each), e.g. read back from the device
  void append_scalars_bytes(const char* label, const uint8_t* bytes32, size_t n) {
    append_message(label, std::string("begin_append_vector"));
    for (size_t i = 0; i < n; i++) append_message(label, bytes32 + 32 * i, 32);
    append_message(label, std::string("end_append_vector"));
  }
  void append_point_compressed(const char* label, const uint8_t comp[32]) { append_message(label, comp, 32); }
  fr_t challenge_scalar(const char* label) {
    uint8_t buf[64];
    challenge_bytes(label, buf, 64);
    fr_t c = fr_from_bytes64(buf);
    if (trace) trace->push_back(c);
    return c;
  }
  std::vector<fr_t> challenge_vector(const char* label, size_t n) {
    std::vector<fr_t> v(n);
    for (size_t i = 0; i < n; i++) v[i] = challenge_scalar(label);
    return v;
  }
  std::vector<fr_t>* trace = nullptr;  // optional: every challenge in order (parity tests)

 private:
  Strobe strobe_;
};

// utils/random.rs:9-39; the seed scalar (F::rand(test_rng()) in the reference) is an explicit input
class RandomTape {
 public:
  RandomTape(const std::string& name, const fr_t& init_randomness) : tape_(name) {
    tape_.append_scalar("init_randomness", init_randomness);
  }
  fr_t random_scalar(const char* label) { return tape_.challenge_scalar(label); }
  std::vector<fr_t> random_vector(const char* label, size_t n) { return tape_.challenge_vector(label, n); }

 private:
  Transcript tape_;
};

}  // namespace lb
