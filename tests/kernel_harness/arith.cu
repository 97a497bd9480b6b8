// Arithmetic harness (tests/test_gpu_arith.py): the primitives of fr.cuh, fq.cuh, ed25519.cuh and quad.cuh applied to
// n elements, one thread (or one quad of lanes) per element, in either compilation of fq_mul the library uses.
// Element layout and the operations: arith_ops.cuh.  Return codes: harness_common.cuh.
#include "arith_ops.cuh"
#include "harness_common.cuh"

void kh_arith_launch_default(int op, size_t n, const uint32_t* a, const uint32_t* b, const uint64_t* k, uint32_t* out,
                             cudaStream_t st);
void kh_arith_launch_msm(int op, size_t n, const uint32_t* a, const uint32_t* b, const uint64_t* k, uint32_t* out,
                         cudaStream_t st);

extern "C" {

// name of operation `op`, nullptr past the last one
const char* kh_arith_op_name(int op) { return arith::op_name(op); }

// variant 0: fq_mul inlined, arguments by reference; 1: out of line, by value (msm_kernels.cu, msm_large.cu).
// a, b, out: n x 16 u64 (out is copied back whole), k: n u64.
int kh_arith(int variant, int op, size_t n, const uint64_t* a, const uint64_t* b, const uint64_t* k, uint64_t* out) {
  if ((variant != 0 && variant != 1) || !arith::op_name(op) || n == 0) return -4;
  return kh::guarded([&] {
    kh::Scope s;
    const uint32_t* da = s.up<uint32_t>(a, 32 * n);
    const uint32_t* db = s.up<uint32_t>(b, 32 * n);
    const uint64_t* dk = s.up<uint64_t>(k, n);
    uint32_t* dout = s.alloc<uint32_t>(32 * n);
    (variant ? kh_arith_launch_msm : kh_arith_launch_default)(op, n, da, db, dk, dout, s.st);
    s.sync();
    s.down(out, dout, 32 * n);
    s.sync();
  });
}

}  // extern "C"
