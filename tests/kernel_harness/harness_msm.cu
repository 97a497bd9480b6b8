// Test harness for the row-MSM family of msm_kernels.cu (tests/test_gpu_msm_rows.py): the bucket row-MSM with its
// finish, the cross-GPU gather-then-add, the canonicalisation that sizes the variable-base windows, and the out_raw
// branch of the bucket-free row launchers.  Conventions of harness.cu: host inputs copied in, ONE launcher on a stream
// of its own, every output copied back.  Any output pointer may be null; the launcher then gets null for it too.
// Points: out_ext nrows x 16 u64 (x, y, x y, 1) arkworks Montgomery limbs; out_comp nrows x 32 B compressed;
// out_raw nrows x 32 u32 un-normalised internal (X, Y, Z, T).
#include <cstring>

#include "harness_common.cuh"

using namespace lb;
using kh::guarded;
using kh::KhTables;
using kh::Scope;

namespace {

// what the gap between two rows holds when row_stride > ncols: read as a scalar it would change the row's point
constexpr uint32_t kPoison = 0xa5a5a5a5u;

struct Outs {
  fq_t* ext = nullptr;
  uint32_t* comp = nullptr;
  uint32_t* raw = nullptr;
  Outs(Scope& s, int nrows, const void* ext_h, const void* comp_h, const void* raw_h) {
    if (ext_h) ext = s.alloc<fq_t>((size_t)nrows * 4);
    if (comp_h) comp = s.alloc<uint32_t>((size_t)nrows * 8);
    if (raw_h) raw = s.alloc<uint32_t>((size_t)nrows * 32);
  }
  void down(Scope& s, int nrows, void* ext_h, void* comp_h, void* raw_h) const {
    if (ext) s.down(ext_h, ext, (size_t)nrows * 4);
    if (comp) s.down(comp_h, comp, (size_t)nrows * 8);
    if (raw) s.down(raw_h, raw, (size_t)nrows * 32);
  }
};

bool columns_fit(const KhTables* t, int ncols, int col_mul, int col_add) {
  return t && ncols >= 1 && col_mul >= 1 && col_add >= 0 && (size_t)(ncols - 1) * col_mul + col_add < t->npts;
}

}  // namespace

extern "C" {

// launch_msm_rows over the tables' window table T (stride npts; shifted == 0 reads window 0 only, the table
// msm_variable_base builds).  scalars: nrows x ncols x limbs u32, compact (limbs 1: u32 integers, 8: canonical 256-bit);
// on the device row r starts at r * row_stride scalars and the rest of its stride is kPoison.
int kh_msm_rows(const KhTables* t, int shifted, const uint32_t* scalars, int limbs, size_t row_stride, int nrows, int ncols,
                int nw, int col_mul, int col_add, uint64_t* out_ext, uint8_t* out_comp, uint32_t* out_raw) {
  if (!columns_fit(t, ncols, col_mul, col_add) || nrows < 1 || (limbs != 1 && limbs != 8) || row_stride < (size_t)ncols ||
      nw < 1 || nw > (limbs == 1 ? 5 : kMsmFullWindows))
    return -4;
  return guarded([&] {
    Scope s;
    std::vector<uint32_t> h((size_t)nrows * row_stride * limbs, kPoison);
    for (int r = 0; r < nrows; r++)
      memcpy(h.data() + (size_t)r * row_stride * limbs, scalars + (size_t)r * ncols * limbs, (size_t)ncols * limbs * 4);
    const uint32_t* ds = s.up<uint32_t>(h.data(), h.size());
    pt_ext* part = s.alloc<pt_ext>(msm_partials_count(nrows, ncols, nw));
    const Outs o(s, nrows, out_ext, out_comp, out_raw);
    launch_msm_rows(t->T, t->npts, shifted, ds, limbs, row_stride, nrows, ncols, nw, col_mul, col_add, part, o.ext, o.comp,
                    o.raw, s.st);
    s.sync();
    o.down(s, nrows, out_ext, out_comp, out_raw);
    s.sync();
  });
}

// raw: nsrc x nrows x 32 u32, source k of row r at (k * nrows + r) * 32 (the all-gathered partial points)
int kh_sum_raw_points(const uint32_t* raw, int nsrc, int nrows, uint32_t* out_raw, uint8_t* out_comp, uint64_t* out_ext) {
  if (nsrc < 1 || nrows < 1) return -4;
  return guarded([&] {
    Scope s;
    const uint32_t* dr = s.up<uint32_t>(raw, (size_t)nsrc * nrows * 32);
    const Outs o(s, nrows, out_ext, out_comp, out_raw);
    launch_sum_raw_points(dr, nsrc, nrows, o.raw, o.comp, o.ext, s.st);
    s.sync();
    o.down(s, nrows, out_ext, out_comp, out_raw);
    s.sync();
  });
}

// in: n Montgomery elements -> out: n canonical integers (4 x u64); *max_bits: the device counter, preset to
// max_bits_preset before the launch, as the launch left it
int kh_canonicalize(const uint64_t* in, size_t n, unsigned max_bits_preset, uint64_t* out, unsigned* max_bits) {
  return guarded([&] {
    Scope s;
    const fr_t* din = s.up<fr_t>(in, n);
    fr_t* dout = s.alloc<fr_t>(n);
    unsigned* dmb = s.up<unsigned>(&max_bits_preset, 1);
    launch_canonicalize(din, dout, n, dmb, s.st);
    s.sync();
    s.down(out, dout, n);
    s.down(max_bits, dmb, 1);
    s.sync();
  });
}

// the out_raw branch (msm_finish_kernel) of launch_msm_rows_direct_u32 (form 0: nrows x ncols u32 scalars; use16: with
// the tables' M16, built for exactly this ncols and column map, and K16 from launch_centre_constant) or of
// launch_msm_rows_direct_fr (form 1: nrows x ncols Montgomery elements).  Row stride ncols.
int kh_msm_rows_direct_raw(const KhTables* t, int form, const void* scalars, int nrows, int ncols, int nw, int col_mul,
                           int col_add, int use16, uint32_t* out_raw, uint8_t* out_comp) {
  if (!columns_fit(t, ncols, col_mul, col_add) || nrows < 1 || !out_raw || (form != 0 && form != 1) || (form == 1 && use16) ||
      (use16 && (!t->M16 || t->ncols16 != (size_t)ncols)))
    return -4;
  return guarded([&] {
    Scope s;
    pt_ext* part = s.alloc<pt_ext>(nrows);
    const Outs o(s, nrows, nullptr, out_comp, out_raw);
    if (form == 0) {
      const uint32_t* ds = s.up<uint32_t>(scalars, (size_t)nrows * ncols);
      pt_ext* K16 = nullptr;
      if (use16) {
        K16 = s.alloc<pt_ext>(1);
        launch_centre_constant(t->M16, ncols, K16, s.st);
      }
      launch_msm_rows_direct_u32(t->M, t->npts, use16 ? t->M16 : nullptr, K16, ds, ncols, nrows, ncols, nw, col_mul, col_add,
                                 part, nullptr, o.comp, o.raw, s.st);
    } else {
      const fr_t* ds = s.up<fr_t>(scalars, (size_t)nrows * ncols);
      launch_msm_rows_direct_fr(t->M, t->npts, ds, ncols, nrows, ncols, nw, col_mul, col_add, part, nullptr, o.comp, o.raw,
                                s.st);
    }
    s.sync();
    o.down(s, nrows, nullptr, out_comp, out_raw);
    s.sync();
  });
}

}  // extern "C"
