// Test harness for the two inputs every proof is built from (tests/test_gpu_densify_launch.py, test_gpu_gens_tables.py):
// the densified representation (launch_densify, densify_kernels.cu) and the generator tables (launch_build_table,
// launch_build_multiples, launch_build_multiples16, launch_centre_constant, msm_kernels.cu).  Conventions of harness.cu:
// host inputs copied in, the launcher on a stream of its own, every output copied back.
// Return codes: see harness_common.cuh.
// fq_mul as msm_kernels.cu compiles it, so that the entries are normalised exactly as normalize_rows_kernel does
#define LB_FQ_MUL_ATTR static __host__ __device__ __noinline__
#define LB_FQ_MUL_BYVALUE
#include <cstring>

#include "harness_common.cuh"

using namespace lb;
using kh::ck;
using kh::guarded;
using kh::KhTables;
using kh::Scope;

namespace {

// every table entry as arkworks affine (x, y) plus a third coordinate: t2d of a niels entry, T / Z of an extended one
__global__ void __launch_bounds__(128)
    table_entries_kernel(const pt_niels* niels, const pt_ext* ext, const uint64_t* idx, size_t count, fq_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  pt_ext p;
  fq_t t;
  if (niels) {
    const pt_niels n = niels[idx[i]];
    p = pt_from_niels(n);
    t = n.t2d;
  } else {
    p = ext[idx[i]];
    t = fq_mul(p.T, fq_inv(p.Z));
  }
  fq_t x, y;
  pt_to_affine_canonical(p, x, y);
  out[3 * i + 0] = fq_to_ark(x);
  out[3 * i + 1] = fq_to_ark(y);
  out[3 * i + 2] = fq_to_ark(t);
}

}  // namespace

extern "C" {

// ---------------------------------------------------------------- densify
// idx: the index matrix, entry (k, i) at idx[k * row_stride + i * col_stride], u32 or u64 (elem_bytes).  One
// launch_densify.  dim / read / fin: C * dim_stride (read_stride,
// final_stride) u32 each, uploaded as given (the caller poisons them) and copied back whole, so a write outside a shard
// shows as a changed word.  check != 0: with a DzRangeCheck (pinned flag + event); bad_out = the flag, else 0.
int kh_densify(const void* idx, int elem_bytes, size_t row_stride, size_t col_stride, size_t n, size_t s, int C,
               size_t log_m, int G, int g, int check, uint32_t* dim, size_t dim_stride, uint32_t* read, size_t read_stride,
               uint32_t* fin, size_t final_stride, uint32_t* bad_out) {
  if ((elem_bytes != 4 && elem_bytes != 8) || n < 1 || n > s || C < 1 || C > 16 || G < 1 || g < 0 || g >= G ||
      !densify_gpu_supported(s, log_m))
    return -4;
  return guarded([&] {
    Scope sc;
    const size_t span = (n - 1) * row_stride + (size_t)(C - 1) * col_stride + 1;  // elements the launcher may read
    const void* d_idx = elem_bytes == 8 ? (const void*)sc.up<uint64_t>(idx, span) : (const void*)sc.up<uint32_t>(idx, span);
    // zeroed: a wrong sort that leaves a slot unwritten makes dz_read_kernel read (address 0, access 0) from it, a
    // wrong output rather than an index past the outputs
    uint32_t* scratch = sc.alloc<uint32_t>(densify_scratch_words(s, C, log_m));
    uint32_t* d_dim = sc.up<uint32_t>(dim, (size_t)C * dim_stride);
    uint32_t* d_read = sc.up<uint32_t>(read, (size_t)C * read_stride);
    uint32_t* d_fin = sc.up<uint32_t>(fin, (size_t)C * final_stride);
    unsigned* h_bad = nullptr;
    cudaEvent_t ev = nullptr;
    if (check) {
      ck(cudaHostAlloc((void**)&h_bad, sizeof(unsigned), cudaHostAllocDefault));
      sc.host.push_back(h_bad);
      *h_bad = 0xffffffffu;  // neither verdict: the launch must write it
      ck(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    }
    const DzIndices di{d_idx, elem_bytes, row_stride, col_stride};
    const DzRangeCheck rc{h_bad, ev};
    try {
      launch_densify(di, check ? &rc : nullptr, n, s, C, log_m, G, g, scratch, d_dim, dim_stride, d_read, read_stride, d_fin,
                     final_stride, sc.st);
      if (check) ck(cudaEventSynchronize(ev));
      sc.sync();
    } catch (...) {
      if (ev) cudaEventDestroy(ev);
      throw;
    }
    if (ev) cudaEventDestroy(ev);
    *bad_out = check ? *h_bad : 0u;
    sc.down(dim, d_dim, (size_t)C * dim_stride);
    sc.down(read, d_read, (size_t)C * read_stride);
    sc.down(fin, d_fin, (size_t)C * final_stride);
    sc.sync();
  });
}

// ---------------------------------------------------------------- generator tables as a proof builds them
// gens_build_tables (prover.cu) launch for launch: T over n_points generators (stride n_points), M over the first nd
// with table_stride n_points, M16 over ncols16 local columns (column jl <-> generator jl * col_mul + col_add) with
// npts8 = nd, and K16[k] for every 2^k <= ncols16.  Released by kh_tables_destroy (harness.cu).
int kh_tables_build(const uint64_t* gens_affine, size_t n_points, size_t nd, size_t ncols16, size_t col_mul, size_t col_add,
                    KhTables** out) {
  *out = nullptr;
  if (nd < 1 || nd > n_points || (ncols16 && (col_mul < 1 || (ncols16 - 1) * col_mul + col_add >= nd))) return -4;
  KhTables* t = new KhTables();
  int rc = guarded([&] {
    Scope s;
    t->npts = n_points;
    t->nd = nd;
    t->ncols16 = ncols16;
    ck(cudaMalloc(&t->T, (size_t)kMsmFullWindows * n_points * sizeof(pt_niels)));
    ck(cudaMalloc(&t->M, (size_t)kMsmFullWindows * nd * 128 * sizeof(pt_niels)));
    const fq_t* d_bases = s.up<fq_t>(gens_affine, n_points * 2);
    launch_build_table(d_bases, n_points, t->T, n_points, kMsmFullWindows, s.st);
    launch_build_multiples(t->T, n_points, nd, kMsmFullWindows, t->M, s.st);
    if (ncols16) {
      ck(cudaMalloc(&t->M16, ncols16 * 32768 * sizeof(pt_niels)));
      ck(cudaMalloc(&t->K16, 32 * sizeof(pt_ext)));
      launch_build_multiples16(t->T, t->M, nd, ncols16, col_mul, col_add, t->M16, s.st);
      for (size_t k = 0; ((size_t)1 << k) <= ncols16 && k < 32; k++) {
        launch_centre_constant(t->M16, 1 << k, t->K16 + k, s.st);
        t->nk16 = k + 1;
      }
    }
    s.sync();
  });
  if (rc != 0) {
    cudaFree(t->T);
    cudaFree(t->M);
    cudaFree(t->M16);
    cudaFree(t->K16);
    delete t;
    return rc;
  }
  *out = t;
  return 0;
}

// entries flat_idx[0 .. count) of one table (which: 0 T, 1 M, 2 M16, 3 K16; indices into the table as it is laid out)
// -> out: count x 12 u64, arkworks Montgomery limbs of x, y and t2d (T, M, M16) or T / Z (K16)
int kh_table_entries(const KhTables* t, int which, const uint64_t* flat_idx, size_t count, uint64_t* out) {
  if (!t || which < 0 || which > 3 || count < 1) return -4;
  const size_t size[4] = {(size_t)kMsmFullWindows * t->npts, (size_t)kMsmFullWindows * t->nd * 128, t->ncols16 * 32768,
                          t->nk16};
  for (size_t i = 0; i < count; i++)
    if (flat_idx[i] >= size[which]) return -4;
  return guarded([&] {
    Scope s;
    const uint64_t* d_idx = s.up<uint64_t>(flat_idx, count);
    fq_t* d_out = s.alloc<fq_t>(3 * count);
    const pt_niels* niels = which == 0 ? t->T : which == 1 ? t->M : which == 2 ? t->M16 : nullptr;
    launch(table_entries_kernel, (unsigned)((count + 127) / 128), 128, 0, s.st, niels, which == 3 ? t->K16 : nullptr, d_idx,
           count, d_out);
    s.sync();
    s.down(out, d_out, 3 * count);
    s.sync();
  });
}

}  // extern "C"
