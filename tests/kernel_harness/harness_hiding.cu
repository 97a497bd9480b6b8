// Test harness for the blind term of hiding row commitments (launch_row_blinds, msm_kernels.cu), built by
// Makefile.hiding as libkernel_harness_hiding.so (tests/test_gpu_hiding.py), with the conventions of harness.cu: host
// inputs copied in, ONE launcher on a stream of its own, the output copied back.  The window and multiples tables come
// from kh_tables_create (harness.cu, libkernel_harness.so).
#include "harness_common.cuh"

using namespace lb;
using kh::guarded;
using kh::KhTables;
using kh::Scope;

extern "C" {

// out_comp = raw_i + blinds[i] * G_hcol: raw nrows x 32 u32 un-normalised points, blinds nrows Montgomery elements,
// out_comp nrows x 32 B compressed.  source 0: the multiples of G_hcol read from column hcol of the tables' M;
// source 1: built for G_hcol alone from the window table (launch_build_multiples, npts = 1), as a hiding commitment
// without the multiples table builds them.
int kh_row_blinds(const KhTables* t, int source, size_t hcol, const uint32_t* raw, const uint64_t* blinds, int nrows,
                  uint8_t* out_comp) {
  if (!t || hcol >= t->npts || nrows < 1 || (source != 0 && source != 1) || !out_comp) return -4;
  return guarded([&] {
    Scope s;
    const uint32_t* dr = s.up<uint32_t>(raw, (size_t)nrows * 32);
    const fr_t* db = s.up<fr_t>(blinds, (size_t)nrows);
    uint32_t* comp = s.alloc<uint32_t>((size_t)nrows * 8);
    if (source == 0) {
      launch_row_blinds(t->M + hcol * 128, t->npts * 128, db, dr, nrows, comp, s.st);
    } else {
      pt_niels* mh = s.alloc<pt_niels>((size_t)kMsmFullWindows * 128);
      launch_build_multiples(t->T + hcol, t->npts, 1, kMsmFullWindows, mh, s.st);
      launch_row_blinds(mh, 128, db, dr, nrows, comp, s.st);
    }
    s.sync();
    s.down(out_comp, comp, (size_t)nrows * 8);
    s.sync();
  });
}

}  // extern "C"
