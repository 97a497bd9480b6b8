// Steady-state (warm, back-to-back) duration of the latency-bound kernels of the prover, timed with CUDA
// events over many launches: the per-round cost the host actually waits for.  Links the product's kernel
// objects (lasso_b200/_build/*.o); not part of the product.
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "../../lasso_b200/csrc/kernels.cuh"
#include "../../lasso_b200/csrc/msm.cuh"
using namespace lb;

__global__ void empty_kernel() {}
__global__ void fill_kernel(uint32_t* p, size_t nwords, uint32_t mask) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nwords; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t x = (uint32_t)i * 2654435761u + 12345u;
    x ^= x >> 13;
    p[i] = x & mask;
  }
}
template <typename F>
static double time_us(F f, int iters, cudaStream_t st) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  for (int i = 0; i < 20; i++) f();
  cudaStreamSynchronize(st);
  cudaEventRecord(e0, st);
  for (int i = 0; i < iters; i++) f();
  cudaEventRecord(e1, st);
  cudaStreamSynchronize(st);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(e));
  return 1e3 * ms / iters;
}
int main(int argc, char** argv) {
  cudaStream_t st;
  cudaStreamCreate(&st);
  const int ncirc = 8;
  const size_t maxlen = (size_t)1 << 19;
  std::vector<fr_t*> hA(ncirc), hB(ncirc);
  for (int k = 0; k < ncirc; k++) {
    cudaMalloc(&hA[k], maxlen * 32);
    cudaMalloc(&hB[k], maxlen * 32);
    fill_kernel<<<256, 256, 0, st>>>((uint32_t*)hA[k], maxlen * 8, 0x0fffffffu);
    fill_kernel<<<256, 256, 0, st>>>((uint32_t*)hB[k], maxlen * 8, 0x0fffffffu);
  }
  fr_t **dA, **dB, *C0, *C1, *partial;
  cudaMalloc(&dA, ncirc * 8);
  cudaMalloc(&dB, ncirc * 8);
  cudaMemcpy(dA, hA.data(), ncirc * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dB, hB.data(), ncirc * 8, cudaMemcpyHostToDevice);
  cudaMalloc(&C0, maxlen * 32);
  cudaMalloc(&C1, maxlen * 32);
  fill_kernel<<<256, 256, 0, st>>>((uint32_t*)C0, maxlen * 8, 0x0fffffffu);
  cudaMalloc(&partial, 1 << 22);
  unsigned* counter;
  cudaMalloc(&counter, 64);
  cudaMemset(counter, 0, 64);
  uint32_t* small32;
  cudaMalloc(&small32, 4096);
  // one publication region in mapped pinned memory, as the prover's (nobody waits for the messages here)
  const size_t pub_bytes = (size_t)kPubElems * kPubSlotWords * 8;
  unsigned long long *h_pub, *d_pub;
  cudaHostAlloc((void**)&h_pub, pub_bytes, cudaHostAllocMapped);
  cudaHostGetDevicePointer((void**)&d_pub, h_pub, 0);
  PubDst pub = {};
  pub.dst[0] = d_pub;
  pub.ndst = 1;
  pub.tag = 1;
  fr_t r;
  for (int l = 0; l < 8; l++) r.v[l] = 0x01234567u * (l + 1) & 0x0fffffffu;
  Finalize fz;
  fz.partial = partial;
  fz.counter = counter;
  fz.pub = pub;
  CubicCoeffs cf;
  for (int k = 0; k < 32; k++) cf.v[k] = r;
  printf("%-52s %8.2f us\n", "empty kernel, back-to-back", time_us([&] { empty_kernel<<<1, 32, 0, st>>>(); }, 2000, st));
  for (size_t h : {2, 8, 32, 128, 512, 2048, 8192, 32768, 262144}) {
    char nm[96];
    snprintf(nm, sizeof nm, "sc_bind_eval_cubic ncirc=8 h=%zu (mapped)", h);
    printf("%-52s %8.2f us\n", nm,
           time_us([&] { launch_sumcheck_bind_eval_cubic_comb(dA, dB, C0, C1, ncirc, h, r, cf, 0, fz, st); }, 500, st));
  }
  for (size_t half : {1, 16, 256, 4096}) {
    char nm[96];
    snprintf(nm, sizeof nm, "sc_eval_cubic ncirc=8 half=%zu (mapped)", half);
    printf("%-52s %8.2f us\n", nm, time_us([&] { launch_sumcheck_eval_cubic_comb(dA, dB, C0, ncirc, half, cf, 1, fz, st); }, 500, st));
  }
  // Bulletproofs round pieces at n = 2048 (the 2^20-lookup openings)
  for (size_t n : {1024, 2048, 4096}) {
    fr_t *a0 = hA[0], *b0 = hB[0], *a1 = hA[1], *b1 = hB[1], *w0 = hA[2], *w1 = hA[3], *sLR = hA[4];
    char nm[96];
    // table for n+2 generators: any niels-shaped data works for timing (field ops are data-independent)
    pt_niels* table;
    cudaMalloc(&table, (size_t)kMsmFullWindows * (n + 2) * sizeof(pt_niels));
    fill_kernel<<<256, 256, 0, st>>>((uint32_t*)table, (size_t)kMsmFullWindows * (n + 2) * 24, 0xffffffffu);
    // canonical scalars: 253-bit, half the columns zero in each row like a real round
    fill_kernel<<<256, 256, 0, st>>>((uint32_t*)sLR, 2 * (n + 2) * 8, 0x0fffffffu);
    pt_ext* part;
    cudaMalloc(&part, msm_partials_count(2, (int)(n + 2), kMsmFullWindows) * sizeof(pt_ext));
    snprintf(nm, sizeof nm, "msm 2 rows x %zu cols x 32 windows (bucket+finish)", n + 2);
    printf("%-52s %8.2f us\n", nm,
           time_us([&] {
             launch_msm_rows(table, n + 2, 1, sLR, 8, n + 2, 2, (int)(n + 2), kMsmFullWindows, 1, 0, part, nullptr, nullptr, small32,
                             st);
           }, 300, st));
    {  // bucket-free MSM over the multiples table
      pt_niels* M;
      const size_t npts = n + 2;
      if (cudaMalloc(&M, (size_t)kMsmFullWindows * npts * 128 * sizeof(pt_niels)) == cudaSuccess) {
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0, st);
        launch_build_multiples(table, n + 2, npts, kMsmFullWindows, M, st);
        cudaEventRecord(e1, st);
        cudaStreamSynchronize(st);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        snprintf(nm, sizeof nm, "build multiples table, %zu generators (%.0f MB)", npts, kMsmFullWindows * npts * 128 * 96 / 1e6);
        printf("%-52s %8.2f ms\n", nm, ms);
        // one whole Bulletproofs round: scalars, both rows, tail terms, publication
        pt_ext* part_f;
        cudaMalloc(&part_f, 2 * (size_t)bullet_fused_chunks((int)n) * sizeof(pt_ext));
        for (size_t m : {n / 2, (size_t)64, (size_t)2}) {
          snprintf(nm, sizeof nm, "bullet_fused n=%zu m=%zu fold=1", n, m);
          printf("%-52s %8.2f us\n", nm,
                 time_us([&] { launch_bullet_fused(M, npts, a0, b0, w0, a1, b1, w1, n, m, 1, r, r, r, r, part_f, partial, counter, pub, st); },
                         500, st));
        }
        cudaFree(part_f);
        snprintf(nm, sizeof nm, "msm_direct 2 rows x %zu terms (direct+finish)", n + 2);
        printf("%-52s %8.2f us\n", nm,
               time_us([&] { launch_msm_direct(M, npts, (const uint32_t*)sLR, (int)(n + 2), part, pub, st); }, 300, st));
        cudaFree(M);
      }
    }
    cudaFree(table);
    cudaFree(part);
  }
  return 0;
}
