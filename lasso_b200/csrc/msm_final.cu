// lasso_b200 — last step of the large MSM (msm_large.cu): per window W = A_0 + L_0 (A_1 + L_1 (...)), then the window
// combination sum_w 2^(c w) W_w (src/msm/mod.rs:150-163: c doublings per window) and the normalisation.  ONE warp:
// the ~250 doublings are a dependent chain, so the only lever is the latency of a doubling — quad-lane arithmetic
// (quad.cuh: two multiplication levels per doubling) with the field multiplication INLINED (this translation unit
// keeps fq_mul's default attributes; the big kernels next door call it out of line to stay small).
#include "kernels.cuh"
#include "msm.cuh"
#include "quad.cuh"

namespace lb {

namespace {
__device__ __forceinline__ pt_ext ldp(const pt_ext* p) {
  pt_ext r;
  r.X = ld_fq(&p->X);
  r.Y = ld_fq(&p->Y);
  r.Z = ld_fq(&p->Z);
  r.T = ld_fq(&p->T);
  return r;
}
}  // namespace

struct MsmLgL {
  int v[8];
};
__global__ void __launch_bounds__(32)
    msm_final_kernel(const pt_ext* A, int nlev, MsmLgL lgL, int nw, int c, fq_t* out_ext, uint32_t* out_raw) {
  __shared__ fq_t sw[32 * 4];
  const int lane = threadIdx.x, role = lane & 3;
  if (lane < nw) {
    pt_ext v = ldp(A + (size_t)lane * nlev + (nlev - 1));
    for (int k = nlev - 2; k >= 0; k--) {
      for (int d = 0; d < lgL.v[k]; d++) v = pt_dbl(v);
      v = pt_add(v, ldp(A + (size_t)lane * nlev + k));
    }
    sw[lane * 4 + 0] = v.X;
    sw[lane * 4 + 1] = v.Y;
    sw[lane * 4 + 2] = v.Z;
    sw[lane * 4 + 3] = v.T;
  }
  __syncwarp();
  fq_t mine = sw[(nw - 1) * 4 + role];  // every quad runs the same chain (uniform control flow); quad 0's result is used
  for (int w = nw - 2; w >= 0; w--) {
    for (int d = 0; d < c; d++) mine = quad_dbl(0xffffffffu, lane, mine);
    mine = quad_add(0xffffffffu, lane, mine, sw + w * 4);
  }
  pt_ext acc;
  acc.X = shfl_fq(0xffffffffu, mine, 0);
  acc.Y = shfl_fq(0xffffffffu, mine, 1);
  acc.Z = shfl_fq(0xffffffffu, mine, 2);
  acc.T = shfl_fq(0xffffffffu, mine, 3);
  if (lane == 0) {
    if (out_raw) {
#pragma unroll
      for (int l = 0; l < 8; l++) {
        out_raw[l] = acc.X.v[l];
        out_raw[8 + l] = acc.Y.v[l];
        out_raw[16 + l] = acc.Z.v[l];
        out_raw[24 + l] = acc.T.v[l];
      }
    }
    if (out_ext) {
      fq_t x, y;
      pt_to_affine_canonical(acc, x, y);
      out_ext[0] = fq_to_ark(x);
      out_ext[1] = fq_to_ark(y);
      out_ext[2] = fq_to_ark(fq_mul(x, y));
      out_ext[3] = fq_to_ark(fq_one());
    }
  }
}

void launch_msm_final(const pt_ext* A, int nlev, const int* lgL, int nw, int c, fq_t* out_ext, uint32_t* out_raw, cudaStream_t st) {
  MsmLgL lg;
  for (int k = 0; k < 8; k++) lg.v[k] = lgL[k];
  launch(msm_final_kernel, 1, 32, 0, st, A, nlev, lg, nw, c, out_ext, out_raw);
}

}  // namespace lb
