// Test harness for the Fr forms of the lookup-value kernels (tables of arbitrary field elements), built by Makefile.fr
// as libkernel_harness_fr.so: one extern "C" wrapper per launcher, with the conventions of harness.cu (host inputs
// copied in, ONE launcher on a stream of its own, outputs copied back).  Field elements are 4 x u64 Montgomery limbs.
#include "harness_common.cuh"

using namespace lb;
using kh::guarded;
using kh::KhTables;  // created by kh_tables_create (harness.cu, libkernel_harness.so)
using kh::Scope;

extern "C" {

// nrows x ncols Montgomery scalars (row stride ncols) over the 8-bit multiples table, local column c <-> generator
// c * col_mul + col_add.  out: nrows x 16 u64 (x, y, t, z) arkworks limbs.
int kh_msm_rows_direct_fr(const KhTables* t, const uint64_t* scalars, int nrows, int ncols, int nw, int col_mul, int col_add,
                          uint64_t* out) {
  if (!t || (size_t)(ncols - 1) * col_mul + col_add >= t->npts) return -4;
  return guarded([&] {
    Scope s;
    const fr_t* ds = s.up<fr_t>(scalars, (size_t)nrows * ncols);
    pt_ext* part = s.alloc<pt_ext>(nrows);
    fq_t* dout = s.alloc<fq_t>((size_t)nrows * 4);
    launch_msm_rows_direct_fr(t->M, t->npts, ds, ncols, nrows, ncols, nw, col_mul, col_add, part, dout, nullptr, nullptr,
                              s.st);
    s.sync();
    s.down(out, dout, (size_t)nrows * 4);
    s.sync();
  });
}

int kh_bound_fr(const uint64_t* Z, const uint64_t* L, size_t L_size, size_t R_size, uint64_t* out) {
  return guarded([&] {
    Scope s;
    const fr_t* dZ = s.up<fr_t>(Z, L_size * R_size);
    const fr_t* dL = s.up<fr_t>(L, L_size);
    fr_t* partial = s.alloc<fr_t>((size_t)bound_max_chunks() * R_size);
    fr_t* dout = s.alloc<fr_t>(R_size);
    launch_bound_fr(dZ, dL, L_size, R_size, partial, dout, s.st);
    s.sync();
    s.down(out, dout, R_size);
    s.sync();
  });
}

// base: npolys x stride elements (the first n of each row are used)
int kh_multi_dot_fr(const uint64_t* base, size_t stride, int npolys, const uint64_t* eq, size_t n, uint64_t* out) {
  return guarded([&] {
    Scope s;
    const fr_t* dz = s.up<fr_t>(base, (size_t)npolys * stride);
    const fr_t* deq = s.up<fr_t>(eq, n);
    fr_t* partial = s.alloc<fr_t>((size_t)sumcheck_max_blocks() * npolys);
    fr_t* dout = s.alloc<fr_t>(npolys);
    launch_multi_dot_fr(dz, stride, npolys, deq, n, partial, dout, s.st);
    s.sync();
    s.down(out, dout, npolys);
    s.sync();
  });
}

}  // extern "C"
