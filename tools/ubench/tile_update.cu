// Micro-benchmark of the band workers' 32x32x32 tile update T -= A B^T with both operands in shared memory, in the two
// DMMA shapes the band kernels use (band_tile.cuh):
//   k4   128 x mma.m8n8k4, operands staged with the padded column stride 40 the workers used before (m8n8k4 maps)
//   k16  16 x mma.m16n8k16, operands in swizzled stages (stage16_*), streamed one k-step at a time (stage16_gemm_sub)
// One CTA per SM with W warps (one update stream per warp, own A / B stages), like pool A (W = 4) and pool B (W = 8).
// Prints cycles per update per warp (clock64 of warp 0) and the chip's fp64 rate, after checking both shapes against a
// host product.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I../../dynosam_b200/csrc tile_update.cu -o tile_update
#include <cstdio>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#include "band_tile.cuh"
using namespace dynoba;

constexpr int TS4 = 40;   // padded column stride of the m8n8k4 operand stages
__device__ __forceinline__ void frag8_load_s40(const double* t, double (&f)[TILE], int lane) {
  const double* p = t + (lane & 3)*TS4 + (lane >> 2);
#pragma unroll
  for (int b = 0; b < 4; b++)
#pragma unroll
    for (int kb = 0; kb < 8; kb++) f[b*8 + kb] = p[4*kb*TS4 + 8*b];
}

// in: A, B (column-major 32x32); out[warp-global]: T - iters * A B^T with T = 0 (warp 0 of CTA 0 checked on the host)
template <bool K16>
__global__ void update_kernel(const double* __restrict__ A, const double* __restrict__ B, double* out, int iters, long long* cyc) {
  extern __shared__ __align__(16) double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = K16 ? 2*TILE2 : 2*TILE*TS4;
  double* sa = sm + (size_t)warp*per;
  double* sb = sa + per/2;
  for (int e = lane; e < TILE2; e += 32) {
    const int r = e & 31, c = e >> 5;
    if (K16) { sa[stage16_index(r, c)] = A[e]; sb[stage16_index(r, c)] = B[e]; }
    else { sa[c*TS4 + r] = A[e]; sb[c*TS4 + r] = B[e]; }
  }
  __syncwarp();
  double acc[TILE];
#pragma unroll
  for (int e = 0; e < TILE; e++) acc[e] = 0.0;
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    asm volatile("" ::: "memory");    // the operands are re-read from shared memory every update, as in the workers
    if (K16) stage16_gemm_sub(acc, sa, sb, lane);
    else {
      double fa[TILE], fb[TILE];
      frag8_load_s40(sa, fa, lane); frag8_load_s40(sb, fb, lane);
      frag8_gemm_sub(acc, fa, fb);
    }
  }
  const long long t1 = clock64();
  double* o = out + ((size_t)blockIdx.x*(blockDim.x >> 5) + warp)*TILE2;
  if (K16) cfrag16_store(o, acc, lane); else cfrag8_store(o, acc, lane);
  if (blockIdx.x == 0 && threadIdx.x == 0) *cyc = t1 - t0;
}

int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs\n", prop.name, sms);
  std::vector<double> hA(TILE2), hB(TILE2), ref(TILE2, 0.0);
  for (int e = 0; e < TILE2; e++) { hA[e] = std::sin(0.37*e); hB[e] = std::cos(0.11*e + 0.5); }
  const int iters = 2000, check_iters = 3;
  for (int r = 0; r < TILE; r++)
    for (int c = 0; c < TILE; c++) {
      double s = 0; for (int k = 0; k < TILE; k++) s += hA[k*TILE + r]*hB[k*TILE + c];
      ref[c*TILE + r] = -check_iters*s;
    }
  double *dA, *dB, *dO; long long* dc;
  cudaMalloc(&dA, TILE2*8); cudaMalloc(&dB, TILE2*8); cudaMalloc(&dO, (size_t)sms*8*TILE2*8); cudaMalloc(&dc, 8);
  cudaMemcpy(dA, hA.data(), TILE2*8, cudaMemcpyHostToDevice); cudaMemcpy(dB, hB.data(), TILE2*8, cudaMemcpyHostToDevice);
  for (int k16 = 0; k16 < 2; k16++) {
    auto kern = k16 ? update_kernel<true> : update_kernel<false>;
    for (int W : {4, 8}) {
      const size_t smem = (size_t)W*(k16 ? 2*TILE2 : 2*TILE*TS4)*8;
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      kern<<<sms, W*32, smem>>>(dA, dB, dO, check_iters, dc);
      std::vector<double> got(TILE2);
      cudaMemcpy(got.data(), dO, TILE2*8, cudaMemcpyDeviceToHost);
      double err = 0; for (int e = 0; e < TILE2; e++) err = std::fmax(err, std::fabs(got[e] - ref[e]));
      cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
      kern<<<sms, W*32, smem>>>(dA, dB, dO, iters, dc);
      cudaEventRecord(e0); kern<<<sms, W*32, smem>>>(dA, dB, dO, iters, dc); cudaEventRecord(e1);
      cudaDeviceSynchronize();
      float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
      long long cyc = 0; cudaMemcpy(&cyc, dc, 8, cudaMemcpyDeviceToHost);
      const double flops = 2.0*32*32*32*(double)iters*W*sms;
      printf("tile update %-4s %d warps/SM: %7.1f cycles per update per warp, chip %5.2f TFLOP/s, max error %.1e  %s\n",
             k16 ? "k16" : "k4", W, (double)cyc/iters, flops/(ms*1e-3)/1e12, err, cudaGetErrorString(cudaGetLastError()));
    }
  }
  return 0;
}
