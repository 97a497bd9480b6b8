// Test harness for the launchers of the caller-polynomial paths: the combining-function interpreter (sumcheck rounds,
// fused bind + round, bind, final evaluations, pointwise map), layer 0 of a caller's grand product, the ingest of a
// caller's dense polynomial and the eq tables.  The conventions of harness.cu: host inputs copied in, ONE launcher on a
// stream of its own (twice with `repeat`), every output and every array the launch may write copied back.  Field
// elements are 4 x u64 Montgomery limbs.
//
// Programs come in lasso_comb_create's SSA format (3 x int32 per instruction) and go through the library's own checker
// and slot allocator (program_check.hpp), so the instructions launched here are the ones the library would launch.
// Input tables: `src_of` (may be null) maps input k to the host array it reads, src_of[k] <= k; an input with
// src_of[k] < k shares that array (the same polynomial passed twice).  Host arrays are k x len elements whatever the map;
// the rows of shared inputs are ignored and only the arrays in use are copied back.
// Publishing wrappers with repeat != 0 launch twice on the same Finalize, with tags 1 and 2, after restoring what the
// first launch wrote in place: the second launch publishes only if the first left the ticket counter at 0, and both
// must publish the same values (else -5).
#include <cstring>

#include "../../lasso_b200/csrc/program_check.hpp"
#include "harness_common.cuh"

using namespace lb;
using kh::ck;
using kh::fr_of;
using kh::guarded;
using kh::HarnessError;
using kh::make_fin;
using kh::Pub;
using kh::Scope;

namespace {

constexpr size_t kPartialElems = 65536;  // >= (kCustomMaxDegree + 1) x the largest comb grid (132 x 8 CTAs)

bool check_program(int n_inputs, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts, int degree,
                   std::vector<CustomIns>& ins, int* n_slots) {
  if (n_inputs < 1 || n_inputs > kCombMaxInputs || !prog) return false;
  const std::string why = program_check(n_inputs, prog, n_ops, consts, n_consts, degree, "degree", ins, n_slots);
  if (!why.empty()) fprintf(stderr, "kernel harness: program rejected: %s\n", why.c_str());
  return why.empty();
}

CombProgram upload_program(Scope& s, int n_inputs, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts,
                           int degree) {
  std::vector<CustomIns> ins;
  int n_slots = 0;
  if (!check_program(n_inputs, prog, n_ops, consts, n_consts, degree, ins, &n_slots)) throw HarnessError{-4};
  const CustomIns* d_ops = s.up<CustomIns>(ins.data(), ins.size());
  const fr_t* d_consts = s.up<fr_t>(consts, n_consts);
  return CombProgram{n_inputs, degree, n_ops, n_consts, n_slots, d_ops, d_consts};
}

bool valid_map(const int* src_of, int n) {
  if (n < 1 || n > 65) return false;
  for (int k = 0; src_of && k < n; k++)
    if (src_of[k] < 0 || src_of[k] > k || src_of[src_of[k]] != src_of[k]) return false;
  return true;
}
bool shares(const int* src_of, int n) {
  for (int k = 0; src_of && k < n; k++)
    if (src_of[k] != k) return true;
  return false;
}

// n device arrays of len elements from host[k * len ..], input k reading array src_of[k]
struct Arrays {
  std::vector<fr_t*> p;
  std::vector<bool> own;
  Arrays(Scope& s, const uint64_t* host, const int* src_of, int n, size_t len) : p(n), own(n) {
    for (int k = 0; k < n; k++) {
      own[k] = !src_of || src_of[k] == k;
      p[k] = own[k] ? s.up<fr_t>(host + (size_t)k * len * 4, len) : p[src_of[k]];
    }
  }
  CombPtrs ptrs() const {
    CombPtrs c{};
    for (size_t k = 0; k < p.size() && k < (size_t)kCombMaxInputs; k++) c.p[k] = p[k];
    return c;
  }
  void down(Scope& s, uint64_t* host, size_t len) const {
    for (size_t k = 0; k < p.size(); k++)
      if (own[k]) s.down(host + k * len * 4, p[k], len);
  }
  // device copies of the arrays in use, to undo an in-place launch before it is repeated
  std::vector<fr_t*> backup(Scope& s, size_t len) const {
    std::vector<fr_t*> b(p.size(), nullptr);
    for (size_t k = 0; k < p.size(); k++)
      if (own[k]) {
        b[k] = s.alloc<fr_t>(len);
        ck(cudaMemcpyAsync(b[k], p[k], len * sizeof(fr_t), cudaMemcpyDeviceToDevice, s.st));
      }
    return b;
  }
  void restore(Scope& s, const std::vector<fr_t*>& b, size_t len) const {
    for (size_t k = 0; k < p.size(); k++)
      if (own[k]) ck(cudaMemcpyAsync(p[k], b[k], len * sizeof(fr_t), cudaMemcpyDeviceToDevice, s.st));
  }
};

// Runs launch(fin) once, or twice with tags 1 and 2 (before_second() in between); out: the npub published values.
// launch returns whether it launched anything: when the first call does not, nothing may have been published and
// publish_run returns false.
template <class Launch, class Between>
bool publish_run(Scope& s, int npub, int repeat, uint64_t* out, Launch launch, Between before_second) {
  Pub pub(s);
  Finalize fin = make_fin(s, pub, kPartialElems);
  const bool launched = launch(fin);
  s.sync();
  if (!launched) {
    pub.expect_empty(0, npub);
    return false;
  }
  if (!repeat) {
    pub.decode(0, npub, out);
    return true;
  }
  std::vector<uint64_t> first((size_t)npub * 4);
  pub.decode(0, npub, first.data());
  before_second();
  pub.set_tag(2);
  fin.pub = pub.dst;
  if (!launch(fin)) throw HarnessError{-1};
  s.sync();
  pub.decode(0, npub, out);
  if (memcmp(first.data(), out, first.size() * 8) != 0) throw HarnessError{-5};
  return true;
}

}  // namespace

extern "C" {

// program_check on its own (no GPU): ins_out receives 4 x n_ops ints (op, dst, a, b after slot allocation), *n_slots
// the physical slot count.  -4: the program is rejected (the reason goes to stderr).
int kh_comb_program(int n_inputs, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts, int degree,
                    int32_t* ins_out, int* n_slots) {
  std::vector<CustomIns> ins;
  if (!check_program(n_inputs, prog, n_ops, consts, n_consts, degree, ins, n_slots)) return -4;
  for (int j = 0; j < n_ops; j++) {
    const int32_t v[4] = {ins[j].op, ins[j].dst, ins[j].a, ins[j].b};
    memcpy(ins_out + 4 * j, v, sizeof v);
  }
  return 0;
}

// launch_sumcheck_eval_comb over in: n_inputs x 2 half elements (copied back); out: the degree + 1 published sums
int kh_comb_eval(int n_inputs, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts, int degree,
                 const int* src_of, uint64_t* in, size_t half, int repeat, uint64_t* out) {
  if (!valid_map(src_of, n_inputs) || half < 1) return -4;
  return guarded([&] {
    Scope s;
    const CombProgram g = upload_program(s, n_inputs, prog, n_ops, consts, n_consts, degree);
    const Arrays a(s, in, src_of, n_inputs, 2 * half);
    publish_run(s, degree + 1, repeat, out, [&](const Finalize& f) {
                  launch_sumcheck_eval_comb(g, a.ptrs(), half, f, s.st);
                  return true;
                },
                [] {});
    a.down(s, in, 2 * half);
    s.sync();
  });
}

// launch_sumcheck_bind_eval_comb with the given min_q (0: the library's default threshold): src is n_inputs x 4q
// elements.  in_place: dst = src (src_of must not share arrays), dst_io unused.  Else dst_io (n_inputs x 4q, uploaded
// first so that the caller can check what the launch must not write) receives the whole dst arrays.  src is copied back
// either way.  *launched: what the launcher returned (0: q below the threshold, nothing launched or published).
int kh_comb_bind_eval(int n_inputs, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts, int degree,
                      const int* src_of, uint64_t* src, size_t q, const uint64_t* r, size_t min_q, int in_place, int repeat,
                      uint64_t* dst_io, uint64_t* out, int* launched) {
  if (!valid_map(src_of, n_inputs) || q < 1 || (in_place && shares(src_of, n_inputs)) || (!in_place && !dst_io)) return -4;
  return guarded([&] {
    Scope s;
    const CombProgram g = upload_program(s, n_inputs, prog, n_ops, consts, n_consts, degree);
    const size_t len = 4 * q;
    const Arrays a(s, src, src_of, n_inputs, len);
    const Arrays d = in_place ? a : Arrays(s, dst_io, nullptr, n_inputs, len);
    const std::vector<fr_t*> saved = repeat && in_place ? a.backup(s, len) : std::vector<fr_t*>();
    *launched = publish_run(
        s, degree + 1, repeat, out,
        [&](const Finalize& f) { return launch_sumcheck_bind_eval_comb(g, a.ptrs(), d.ptrs(), q, fr_of(r), f, min_q, s.st); },
        [&] {
          if (in_place) a.restore(s, saved, len);
        });
    a.down(s, src, len);
    if (!in_place) d.down(s, dst_io, len);
    s.sync();
  });
}

// launch_bind_comb over n arrays of 2 half elements: src copied back; out of place, dst_io (n x 2 half, uploaded
// first) receives the whole dst arrays
int kh_bind_comb(int n, const int* src_of, uint64_t* src, size_t half, const uint64_t* r, int in_place, uint64_t* dst_io) {
  if (!valid_map(src_of, n) || n > kCombMaxInputs || half < 1 || (in_place && shares(src_of, n)) || (!in_place && !dst_io))
    return -4;
  return guarded([&] {
    Scope s;
    const Arrays a(s, src, src_of, n, 2 * half);
    const Arrays d = in_place ? a : Arrays(s, dst_io, nullptr, n, 2 * half);
    launch_bind_comb(a.ptrs(), d.ptrs(), n, half, fr_of(r), s.st);
    s.sync();
    a.down(s, src, 2 * half);
    if (!in_place) d.down(s, dst_io, 2 * half);
    s.sync();
  });
}

// launch_final_comb over n arrays of 2 half elements (copied back); out: the n published values
int kh_final_comb(int n, uint64_t* src, size_t half, const uint64_t* r, int repeat, uint64_t* out) {
  if (n < 1 || n > kCombMaxInputs || half < 1) return -4;
  return guarded([&] {
    Scope s;
    const Arrays a(s, src, nullptr, n, 2 * half);
    publish_run(
        s, n, repeat, out,
        [&](const Finalize& f) {
          launch_final_comb(a.ptrs(), n, half, fr_of(r), f, s.st);
          return true;
        },
        [] {});
    a.down(s, src, 2 * half);
    s.sync();
  });
}

// launch_comb_map over in: n_inputs x n elements (copied back); out_io: n + guard elements, uploaded first and copied
// back whole (the map writes the first n only)
int kh_comb_map(int n_inputs, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts, int degree,
                const int* src_of, uint64_t* in, size_t n, uint64_t* out_io, size_t guard) {
  if (!valid_map(src_of, n_inputs) || n < 1) return -4;
  return guarded([&] {
    Scope s;
    const CombProgram g = upload_program(s, n_inputs, prog, n_ops, consts, n_consts, degree);
    const Arrays a(s, in, src_of, n_inputs, n);
    fr_t* d_out = s.up<fr_t>(out_io, n + guard);
    launch_comb_map(g, a.ptrs(), n, d_out, s.st);
    s.sync();
    a.down(s, in, n);
    s.down(out_io, d_out, n + guard);
    s.sync();
  });
}

// launch_product_layer1: P (2 half elements, copied back); out_io: half + guard elements, uploaded first, copied back
int kh_product_layer1(uint64_t* P, size_t half, uint64_t* out_io, size_t guard) {
  if (half < 1) return -4;
  return guarded([&] {
    Scope s;
    fr_t* dP = s.up<fr_t>(P, 2 * half);
    fr_t* dout = s.up<fr_t>(out_io, half + guard);
    launch_product_layer1(dP, dout, half, s.st);
    s.sync();
    s.down(P, dP, 2 * half);
    s.down(out_io, dout, half + guard);
    s.sync();
  });
}

// launch_bind_ptrs over n <= 65 pointer pairs: src (n x 2 half, shared arrays allowed) copied back, dst_io (n x 2 half,
// uploaded first) copied back whole
int kh_bind_ptrs(int n, const int* src_of, uint64_t* src, size_t half, const uint64_t* r, uint64_t* dst_io) {
  if (!valid_map(src_of, n) || half < 1) return -4;
  return guarded([&] {
    Scope s;
    const Arrays a(s, src, src_of, n, 2 * half);
    const Arrays d(s, dst_io, nullptr, n, 2 * half);
    fr_t* const* dsrc = s.up<fr_t*>(a.p.data(), n);
    fr_t* const* ddst = s.up<fr_t*>(d.p.data(), n);
    launch_bind_ptrs(dsrc, ddst, n, half, fr_of(r), s.st);
    s.sync();
    a.down(s, src, 2 * half);
    d.down(s, dst_io, 2 * half);
    s.sync();
  });
}

// launch_poly_ingest: src holds (n - 1) * row_stride + 4 u64 (row i at i * row_stride; from a 256-byte aligned
// allocation, so rows are 8-byte aligned and, for row_stride 5..7, mostly not 32-byte aligned).  dst: n elements;
// flags: the two flag words (zeroed before the launch).
int kh_poly_ingest(const uint64_t* src, size_t row_stride, size_t n, uint64_t* dst, uint32_t* flags) {
  if (row_stride < 4 || n < 1) return -4;
  return guarded([&] {
    Scope s;
    const uint64_t* dsrc = s.up<uint64_t>(src, (n - 1) * row_stride + 4);
    fr_t* ddst = s.alloc<fr_t>(n);
    unsigned* dflags = s.alloc<unsigned>(2);
    launch_poly_ingest(dsrc, row_stride, n, ddst, dflags, s.st);
    s.sync();
    s.down(dst, ddst, n);
    s.down(flags, dflags, 2);
    s.sync();
  });
}

int kh_poly_mirror_u32(const uint64_t* in, size_t n, uint32_t* out) {
  if (n < 1) return -4;
  return guarded([&] {
    Scope s;
    const fr_t* din = s.up<fr_t>(in, n);
    uint32_t* dout = s.alloc<uint32_t>(n);
    launch_poly_mirror_u32(din, n, dout, s.st);
    s.sync();
    s.down(out, dout, n);
    s.sync();
  });
}

// launch_eq_evals(r, ell) into 2^ell elements followed by a guard of kGuard elements, with a scratch of exactly
// kEqScratchElems elements followed by a guard.  The output and both guards start as 0xA5 bytes, a non-canonical value
// no entry can take, so an entry the launch never wrote cannot pass for any expected value.  ranges: n_ranges (start, count)
// pairs of entries to copy back, concatenated in out.  guards[0] / guards[1]: 1 when the output's / the scratch's
// guard changed.
int kh_eq_evals(int ell, const uint64_t* r, const uint64_t* ranges, size_t n_ranges, uint64_t* out, int* guards) {
  constexpr size_t kGuard = 4096;
  if (ell < 0 || ell > 28) return -4;
  const size_t n = (size_t)1 << ell;
  for (size_t j = 0; j < n_ranges; j++)
    if (ranges[2 * j] > n || ranges[2 * j + 1] > n - ranges[2 * j]) return -4;
  return guarded([&] {
    Scope s;
    FrVec rv{};
    for (int j = 0; j < ell; j++) rv.v[j] = fr_of(r + 4 * j);
    fr_t* dout = s.alloc<fr_t>(n + kGuard);
    fr_t* scratch = s.alloc<fr_t>(kEqScratchElems + kGuard);
    ck(cudaMemsetAsync(dout, 0xA5, (n + kGuard) * sizeof(fr_t), s.st));
    ck(cudaMemsetAsync(scratch + kEqScratchElems, 0xA5, kGuard * sizeof(fr_t), s.st));
    launch_eq_evals(rv, ell, dout, scratch, s.st);
    s.sync();
    size_t o = 0;
    for (size_t j = 0; j < n_ranges; j++) {
      s.down(out + 4 * o, dout + ranges[2 * j], ranges[2 * j + 1]);
      o += ranges[2 * j + 1];
    }
    std::vector<uint8_t> g(2 * kGuard * sizeof(fr_t));
    s.down(g.data(), (const uint8_t*)(dout + n), kGuard * sizeof(fr_t));
    s.down(g.data() + kGuard * sizeof(fr_t), (const uint8_t*)(scratch + kEqScratchElems), kGuard * sizeof(fr_t));
    s.sync();
    guards[0] = guards[1] = 0;
    for (size_t i = 0; i < g.size(); i++)
      if (g[i] != 0xA5) guards[i < kGuard * sizeof(fr_t) ? 0 : 1] = 1;
  });
}

}  // extern "C"
