// Test harness: one extern "C" wrapper per launcher of kernels.cuh / msm.cuh that the C ABI does not expose on its own.
// Linked from the library's own kernel objects (lasso_b200/_build/poly_kernels.o, msm_kernels.o), so the tests run
// exactly the code the prover runs.  Every wrapper copies its host inputs to the device, calls ONE launcher on a stream
// of its own, synchronises, copies every output (in-place arrays included) back and frees what it allocated.  Field
// elements are 4 x u64 Montgomery limbs (the fr_t layout), points arkworks affine (x, y) Montgomery limbs.
// Return codes: 0 ok, -1 a launcher threw (std::runtime_error), -2 a CUDA error, -3 a publication slot did not carry
// the message's tag, -4 bad arguments.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "../../lasso_b200/csrc/kernels.cuh"
#include "../../lasso_b200/csrc/msm.cuh"
#include "../../lasso_b200/csrc/pub_codec.hpp"

using namespace lb;

namespace {

struct HarnessError {
  int code;
};

void ck(cudaError_t e) {
  if (e != cudaSuccess) {
    fprintf(stderr, "kernel harness: CUDA error %s\n", cudaGetErrorString(e));
    throw HarnessError{-2};
  }
}

// every device allocation of one call; freed when the call returns, whatever happens
struct Scope {
  std::vector<void*> dev, host;
  cudaStream_t st = nullptr;
  Scope() { ck(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); }
  ~Scope() {
    if (st) cudaStreamSynchronize(st);
    for (void* p : dev) cudaFree(p);
    for (void* p : host) cudaFreeHost(p);
    if (st) cudaStreamDestroy(st);
  }
  template <class T>
  T* alloc(size_t count) {
    void* p = nullptr;
    ck(cudaMalloc(&p, count * sizeof(T) + 16));
    dev.push_back(p);
    ck(cudaMemsetAsync(p, 0, count * sizeof(T) + 16, st));
    return (T*)p;
  }
  template <class T>
  T* up(const void* h, size_t count) {
    T* d = alloc<T>(count);
    if (count) ck(cudaMemcpyAsync(d, h, count * sizeof(T), cudaMemcpyHostToDevice, st));
    return d;
  }
  template <class T>
  void down(void* h, const T* d, size_t count) {
    if (count) ck(cudaMemcpyAsync(h, d, count * sizeof(T), cudaMemcpyDeviceToHost, st));
  }
  // an array of device pointers to n arrays of `len` elements each, filled from host[k * len ..]
  fr_t* const* ptr_array(const uint64_t* host, int n, size_t len, std::vector<fr_t*>& ptrs) {
    ptrs.resize(n);
    for (int k = 0; k < n; k++) ptrs[k] = up<fr_t>(host + (size_t)k * len * 4, len);
    return up<fr_t*>(ptrs.data(), n);
  }
  void sync() {
    ck(cudaStreamSynchronize(st));
    ck(cudaGetLastError());
  }
};

// one publication region in mapped pinned host memory (as the prover's Ctx), tag 1
struct Pub {
  unsigned long long* h = nullptr;
  PubDst dst = {};
  static constexpr uint32_t kTag = 1;
  explicit Pub(Scope& s) {
    const size_t bytes = (size_t)kPubElems * kPubSlotWords * 8;
    ck(cudaHostAlloc((void**)&h, bytes, cudaHostAllocMapped));
    s.host.push_back(h);
    memset(h, 0, bytes);
    unsigned long long* d = nullptr;
    ck(cudaHostGetDevicePointer((void**)&d, h, 0));
    dst.dst[0] = d;
    dst.ndst = 1;
    dst.tag = kTag;
  }
  // elements [v0, v0 + count) -> out (4 x u64 each); every word must carry the tag
  void decode(int v0, int count, uint64_t* out) const {
    for (int v = v0; v < v0 + count; v++) {
      unsigned long long w[5];
      for (int k = 0; k < 5; k++) {
        const unsigned long long word = h[(size_t)v * kPubSlotWords + k];
        if (pub_tag_of(word) != kTag) throw HarnessError{-3};
        w[k] = word & kPubValueMask;
      }
      uint32_t x[8];
      pub_decode(w, x);
      memcpy(out + 4 * (size_t)(v - v0), x, 32);
    }
  }
  // elements [v0, v0 + count) must not have been written
  void expect_empty(int v0, int count) const {
    for (size_t i = (size_t)v0 * kPubSlotWords; i < (size_t)(v0 + count) * kPubSlotWords; i++)
      if (h[i] != 0) throw HarnessError{-3};
  }
};

Finalize make_fin(Scope& s, const Pub& p, size_t partial_elems) {
  Finalize f;
  f.partial = s.alloc<fr_t>(partial_elems);
  f.counter = s.alloc<unsigned>(1);
  f.pub = p.dst;
  return f;
}

fr_t fr_of(const uint64_t* x) {
  fr_t r;
  memcpy(r.v, x, 32);
  return r;
}

bool g_inited = false;
void init() {
  if (g_inited) return;
  poly_init_device();
  msm_init_device();
  g_inited = true;
}

template <class F>
int guarded(F f) {
  try {
    init();
    f();
    return 0;
  } catch (const HarnessError& e) {
    return e.code;
  } catch (const std::runtime_error& e) {
    fprintf(stderr, "kernel harness: %s\n", e.what());
    return -1;
  }
}

}  // namespace

// ---------------------------------------------------------------- window + digit-multiples tables of a generator set
// Built once per test module with the library's launchers (launch_build_table, launch_build_multiples, optionally
// launch_build_multiples16 for ncols16 local columns, column jl <-> generator jl * col_mul + col_add) and kept on the
// device until kh_tables_destroy: rebuilding ~1 GB per launch under test would dominate the suite.
struct KhTables {
  size_t npts = 0, ncols16 = 0;
  pt_niels *T = nullptr, *M = nullptr, *M16 = nullptr;
};

extern "C" {

int kh_tables_create(const uint64_t* gens_affine, size_t npts, size_t ncols16, size_t col_mul, size_t col_add, KhTables** out) {
  *out = nullptr;
  KhTables* t = new KhTables();
  int rc = guarded([&] {
    Scope s;
    t->npts = npts;
    t->ncols16 = ncols16;
    ck(cudaMalloc(&t->T, (size_t)kMsmFullWindows * npts * sizeof(pt_niels)));
    ck(cudaMalloc(&t->M, (size_t)kMsmFullWindows * npts * 128 * sizeof(pt_niels)));
    if (ncols16) ck(cudaMalloc(&t->M16, ncols16 * 32768 * sizeof(pt_niels)));
    const fq_t* d_bases = s.up<fq_t>(gens_affine, npts * 2);
    launch_build_table(d_bases, npts, t->T, npts, kMsmFullWindows, s.st);
    launch_build_multiples(t->T, npts, npts, kMsmFullWindows, t->M, s.st);
    if (ncols16) launch_build_multiples16(t->T, t->M, npts, ncols16, col_mul, col_add, t->M16, s.st);
    s.sync();
  });
  if (rc != 0) {
    cudaFree(t->T);
    cudaFree(t->M);
    cudaFree(t->M16);
    delete t;
    return rc;
  }
  *out = t;
  return 0;
}

void kh_tables_destroy(KhTables* t) {
  if (!t) return;
  cudaFree(t->T);
  cudaFree(t->M);
  cudaFree(t->M16);
  delete t;
}

// ---------------------------------------------------------------- K3: batched cubic rounds
// bind == 0: launch_sumcheck_eval_cubic_comb over arrays of len = 2 * half elements.
// bind != 0: launch_sumcheck_bind_eval_cubic_comb over arrays of len = 2 * h elements (h = bound length); Cout: h elements.
// A, B (ncirc x len) and Cin (len) are copied back after the launch; out3: the three published values.
int kh_cubic(int bind, int ncirc, size_t len, uint64_t* A, uint64_t* B, uint64_t* Cin, uint64_t* Cout, const uint64_t* r,
             const uint64_t* coeffs, int scale, uint64_t* out3) {
  if (ncirc < 1 || ncirc > 32 || len < 2) return -4;
  return guarded([&] {
    Scope s;
    Pub pub(s);
    std::vector<fr_t*> pa, pb;
    fr_t* const* dA = s.ptr_array(A, ncirc, len, pa);
    fr_t* const* dB = s.ptr_array(B, ncirc, len, pb);
    fr_t* dC = s.up<fr_t>(Cin, len);
    fr_t* dCout = s.alloc<fr_t>(len / 2);
    CubicCoeffs cf;
    memset(&cf, 0, sizeof cf);
    memcpy(cf.v, coeffs, (size_t)ncirc * 32);
    const Finalize fin = make_fin(s, pub, 3 * 65536);
    if (bind)
      launch_sumcheck_bind_eval_cubic_comb(dA, dB, dC, dCout, ncirc, len / 2, fr_of(r), cf, scale, fin, s.st);
    else
      launch_sumcheck_eval_cubic_comb(dA, dB, dC, ncirc, len / 2, cf, scale, fin, s.st);
    s.sync();
    for (int k = 0; k < ncirc; k++) {
      s.down(A + (size_t)k * len * 4, pa[k], len);
      s.down(B + (size_t)k * len * 4, pb[k], len);
    }
    s.down(Cin, dC, len);
    if (bind) s.down(Cout, dCout, len / 2);
    s.sync();
    pub.decode(0, 3, out3);
  });
}

// ---------------------------------------------------------------- product trees
// trees: ntrees x (2N) elements, layer 0 in the first N; every layer is copied back.  tops: ntrees * stop_len
// published elements (values stop_len * (slot0 + t) + j); the slots below are checked to stay empty.
int kh_product_trees(int ntrees, size_t N, int slot0, int stop_len, uint64_t* trees, uint64_t* tops) {
  if (ntrees < 1 || ntrees > 32 || (stop_len != 1 && stop_len != 2) || stop_len * (slot0 + ntrees) > kPubElems) return -4;
  return guarded([&] {
    Scope s;
    Pub pub(s);
    std::vector<fr_t*> pt;
    s.ptr_array(trees, ntrees, 2 * N, pt);
    TreePtrs tp;
    memset(&tp, 0, sizeof tp);
    for (int t = 0; t < ntrees; t++) tp.p[t] = pt[t];
    const Finalize fin = make_fin(s, pub, 1);
    launch_product_trees(tp, ntrees, N, slot0, stop_len, fin, s.st);
    s.sync();
    for (int t = 0; t < ntrees; t++) s.down(trees + (size_t)t * 2 * N * 4, pt[t], 2 * N);
    s.sync();
    pub.expect_empty(0, stop_len * slot0);
    pub.decode(stop_len * slot0, stop_len * ntrees, tops);
  });
}

// heads: n x 2 elements (each pair its own device array); copied back; out: the n published values
int kh_bind_heads(int n, uint64_t* heads, const uint64_t* r, uint64_t* out) {
  if (n < 1 || n > 64) return -4;
  return guarded([&] {
    Scope s;
    Pub pub(s);
    std::vector<fr_t*> ph;
    fr_t* const* d = s.ptr_array(heads, n, 2, ph);
    launch_bind_heads(d, n, fr_of(r), make_fin(s, pub, 1), s.st);
    s.sync();
    for (int k = 0; k < n; k++) s.down(heads + (size_t)k * 8, ph[k], 2);
    s.sync();
    pub.decode(0, n, out);
  });
}

// ---------------------------------------------------------------- u32-mirror reductions
int kh_bound_u32(const uint32_t* Z, const uint64_t* L, size_t L_size, size_t R_size, uint64_t* out) {
  return guarded([&] {
    Scope s;
    const uint32_t* dZ = s.up<uint32_t>(Z, L_size * R_size);
    const fr_t* dL = s.up<fr_t>(L, L_size);
    fr_t* partial = s.alloc<fr_t>((size_t)bound_max_chunks() * R_size);
    fr_t* dout = s.alloc<fr_t>(R_size);
    launch_bound_u32(dZ, dL, L_size, R_size, partial, dout, s.st);
    s.sync();
    s.down(out, dout, R_size);
    s.sync();
  });
}

// base: npolys x stride u32 (the first n of each row are used)
int kh_multi_dot_u32(const uint32_t* base, size_t stride, int npolys, const uint64_t* eq, size_t n, uint64_t* out) {
  return guarded([&] {
    Scope s;
    const uint32_t* dz = s.up<uint32_t>(base, (size_t)npolys * stride);
    const fr_t* deq = s.up<fr_t>(eq, n);
    fr_t* partial = s.alloc<fr_t>((size_t)sumcheck_max_blocks() * npolys);
    fr_t* dout = s.alloc<fr_t>(npolys);
    launch_multi_dot_u32(dz, stride, npolys, deq, n, partial, dout, s.st);
    s.sync();
    s.down(out, dout, npolys);
    s.sync();
  });
}

// ---------------------------------------------------------------- fingerprints
// table: M_local * G elements (the full table), final_fr: M_local
int kh_fingerprints_mem(const uint64_t* table, const uint64_t* final_fr, size_t M_local, int G, int g, const uint64_t* gamma,
                        const uint64_t* tau, uint64_t* out_init, uint64_t* out_final) {
  return guarded([&] {
    Scope s;
    const fr_t* dt = s.up<fr_t>(table, M_local * G);
    const fr_t* df = s.up<fr_t>(final_fr, M_local);
    fr_t* oi = s.alloc<fr_t>(M_local);
    fr_t* of = s.alloc<fr_t>(M_local);
    launch_gp_fingerprints_mem(dt, df, M_local, G, g, fr_of(gamma), fr_of(tau), oi, of, s.st);
    s.sync();
    s.down(out_init, oi, M_local);
    s.down(out_final, of, M_local);
    s.sync();
  });
}

int kh_fingerprints_ops(const uint64_t* dim, const uint64_t* E, const uint64_t* read, size_t n, const uint64_t* gamma,
                        const uint64_t* tau, uint64_t* out_read, uint64_t* out_write) {
  return guarded([&] {
    Scope s;
    const fr_t* dd = s.up<fr_t>(dim, n);
    const fr_t* dE = s.up<fr_t>(E, n);
    const fr_t* dr = s.up<fr_t>(read, n);
    fr_t* orr = s.alloc<fr_t>(n);
    fr_t* ow = s.alloc<fr_t>(n);
    launch_gp_fingerprints_ops(dd, dE, dr, n, fr_of(gamma), fr_of(tau), orr, ow, s.st);
    s.sync();
    s.down(out_read, orr, n);
    s.down(out_write, ow, n);
    s.sync();
  });
}

// ---------------------------------------------------------------- Bulletproofs scalar helpers
// a, b: 2h elements each, folded in place (copied back whole)
int kh_fold_ab(uint64_t* a, uint64_t* b, size_t h, const uint64_t* u, const uint64_t* uinv) {
  return guarded([&] {
    Scope s;
    fr_t* da = s.up<fr_t>(a, 2 * h);
    fr_t* db = s.up<fr_t>(b, 2 * h);
    launch_fold_ab(da, db, h, fr_of(u), fr_of(uinv), s.st);
    s.sync();
    s.down(a, da, 2 * h);
    s.down(b, db, 2 * h);
    s.sync();
  });
}

int kh_cross_inner_products(const uint64_t* a, const uint64_t* b, size_t h, uint64_t* out2) {
  return guarded([&] {
    Scope s;
    const fr_t* da = s.up<fr_t>(a, 2 * h);
    const fr_t* db = s.up<fr_t>(b, 2 * h);
    fr_t* partial = s.alloc<fr_t>(2 * 64);
    fr_t* dout = s.alloc<fr_t>(2);
    launch_cross_inner_products(da, db, h, partial, dout, s.st);
    s.sync();
    s.down(out2, dout, 2);
    s.sync();
  });
}

int kh_expand_weights(const uint64_t* w, size_t n_in, const uint64_t* u, const uint64_t* uinv, uint64_t* w_out) {
  return guarded([&] {
    Scope s;
    const fr_t* dw = s.up<fr_t>(w, n_in);
    fr_t* dout = s.alloc<fr_t>(2 * n_in);
    launch_expand_weights(dw, dout, n_in, fr_of(u), fr_of(uinv), s.st);
    s.sync();
    s.down(w_out, dout, 2 * n_in);
    s.sync();
  });
}

// a: a_len elements, w: w_len elements; sL, sR: n_loc elements each
int kh_bullet_scalars(const uint64_t* a, size_t a_len, const uint64_t* w, size_t w_len, size_t n_loc, size_t m, int G, int g,
                      int a_rep, uint64_t* sL, uint64_t* sR) {
  return guarded([&] {
    Scope s;
    const fr_t* da = s.up<fr_t>(a, a_len);
    const fr_t* dw = s.up<fr_t>(w, w_len);
    fr_t* dl = s.alloc<fr_t>(n_loc);
    fr_t* dr = s.alloc<fr_t>(n_loc);
    launch_bullet_scalars(da, dw, n_loc, m, G, g, a_rep, dl, dr, s.st);
    s.sync();
    s.down(sL, dl, n_loc);
    s.down(sR, dr, n_loc);
    s.sync();
  });
}

// t: t00, t01, t10, t11; out: 2 x (n + 2) canonical integers
int kh_two_row_scalars(const uint64_t* v, int scale, const uint64_t* k, const uint64_t* t, size_t n, uint64_t* out) {
  return guarded([&] {
    Scope s;
    const fr_t* dv = s.up<fr_t>(v, n);
    fr_t* dout = s.alloc<fr_t>(2 * (n + 2));
    launch_two_row_scalars(dv, scale, fr_of(k), fr_of(t), fr_of(t + 4), fr_of(t + 8), fr_of(t + 12), n, dout, s.st);
    s.sync();
    s.down(out, dout, 2 * (n + 2));
    s.sync();
  });
}

// ---------------------------------------------------------------- MSMs over the multiples table
// scalars: 2 x len canonical integers (8 x u32 each); out: 6 x 4 u64, canonical (X, Y, Z) of row 0 then row 1
int kh_msm_direct(const KhTables* t, const uint32_t* scalars, int len, uint64_t* out) {
  if (!t || (size_t)len > t->npts) return -4;
  return guarded([&] {
    Scope s;
    Pub pub(s);
    const uint32_t* ds = s.up<uint32_t>(scalars, (size_t)2 * len * 8);
    pt_ext* part = s.alloc<pt_ext>(2 * (size_t)msm_direct_chunks(len, 1));
    launch_msm_direct(t->M, t->npts, ds, len, part, pub.dst, s.st);
    s.sync();
    pub.decode(0, 6, out);
  });
}

// One Bulletproofs round over generators 0 .. n+1 (G_0..G_{n-1}, Q, h) of the tables (npts >= n + 2).
// a_in / b_in: 2m (fold) or m elements; w_in: n / (2m) (fold) or n / m; a_out / b_out: m, w_out: n / m (fold only).
// out: 6 x 4 u64, canonical (X, Y, Z) of L then R.
int kh_bullet_fused(const KhTables* t, const uint64_t* a_in, const uint64_t* b_in, const uint64_t* w_in, size_t n, size_t m,
                    int fold, const uint64_t* u, const uint64_t* uinv, const uint64_t* blind_L, const uint64_t* blind_R,
                    uint64_t* a_out, uint64_t* b_out, uint64_t* w_out, uint64_t* out) {
  if (!t || n + 2 > t->npts || m < 2 || n < m) return -4;
  return guarded([&] {
    Scope s;
    Pub pub(s);
    const size_t ab_len = fold ? 2 * m : m, w_len = fold ? n / (2 * m) : n / m;
    const fr_t* da = s.up<fr_t>(a_in, ab_len);
    const fr_t* db = s.up<fr_t>(b_in, ab_len);
    const fr_t* dw = s.up<fr_t>(w_in, w_len);
    fr_t* dao = s.alloc<fr_t>(m);
    fr_t* dbo = s.alloc<fr_t>(m);
    fr_t* dwo = s.alloc<fr_t>(n / m);
    const int chunks = bullet_fused_chunks((int)n);
    pt_ext* part = s.alloc<pt_ext>(2 * (size_t)chunks);
    fr_t* ip = s.alloc<fr_t>(2 * (size_t)chunks);
    unsigned* counter = s.alloc<unsigned>(1);
    launch_bullet_fused(t->M, t->npts, da, db, dw, dao, dbo, dwo, n, m, fold, fr_of(u), fr_of(uinv), fr_of(blind_L),
                        fr_of(blind_R), part, ip, counter, pub.dst, s.st);
    s.sync();
    if (fold) {
      s.down(a_out, dao, m);
      s.down(b_out, dbo, m);
      s.down(w_out, dwo, n / m);
    }
    s.sync();
    pub.decode(0, 6, out);
  });
}

// nrows x ncols u32 scalars (row stride ncols); use16: with the tables' M16 (built for exactly this ncols and column
// map) and K16 from launch_centre_constant, else M16 = nullptr.  out: nrows x 16 u64 (x, y, t, z) arkworks limbs.
int kh_msm_rows_direct_u32(const KhTables* t, const uint32_t* scalars, int nrows, int ncols, int nw, int col_mul, int col_add,
                           int use16, uint64_t* out) {
  if (!t || (size_t)(ncols - 1) * col_mul + col_add >= t->npts || (use16 && (!t->M16 || t->ncols16 != (size_t)ncols)))
    return -4;
  return guarded([&] {
    Scope s;
    const uint32_t* ds = s.up<uint32_t>(scalars, (size_t)nrows * ncols);
    pt_ext* part = s.alloc<pt_ext>(nrows);
    fq_t* dout = s.alloc<fq_t>((size_t)nrows * 4);
    pt_ext* K16 = nullptr;
    if (use16) {
      K16 = s.alloc<pt_ext>(1);
      launch_centre_constant(t->M16, ncols, K16, s.st);
    }
    launch_msm_rows_direct_u32(t->M, t->npts, use16 ? t->M16 : nullptr, K16, ds, ncols, nrows, ncols, nw, col_mul, col_add, part,
                               dout, nullptr, nullptr, s.st);
    s.sync();
    s.down(out, dout, (size_t)nrows * 4);
    s.sync();
  });
}

}  // extern "C"
