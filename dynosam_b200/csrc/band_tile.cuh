// band_tile.cuh -- device functions of the band kernels shared by kernels_band.cu (factorisation, solve) and
// kernels_cov.cu (selected inversion): dataflow flags and fp64 tensor-core (DMMA) products of 32x32 tiles.
#pragma once
#include "internal.cuh"

namespace dynoba {

__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void wait_flag(const int* f, int lane) {
  if (lane == 0) {
    int spins = 0;
    while (ld_acquire(f) == 0) { if (++spins > 8) __nanosleep(64); }
  }
  __syncwarp();
}
__device__ __forceinline__ void wait_flag_ge(const int* f, int v, int lane) {
  if (lane == 0) {
    int spins = 0;
    while (ld_acquire(f) < v) { if (++spins > 8) __nanosleep(64); }
  }
  __syncwarp();
}
__device__ __forceinline__ void set_flag_value(int* f, int v, int lane) {
  // the lanes' tile stores are ordered before lane 0's release by the warp barrier (release is cumulative).  No
  // __threadfence(): that is MEMBAR.SC.GPU + ERRBAR + CCTL.IVALL, microseconds per flag on the two-die part.
  __syncwarp();
  if (lane == 0) st_release(f, v);
}
__device__ __forceinline__ void set_flag(int* f, int lane) { set_flag_value(f, 1, lane); }

// ---- fp64 tensor-core tile update for the workers: T(32x32) -= LI LK^T as 128 x mma.m8n8k4 (DMMA).  The FMA version
// reads its B operand from shared memory (one LDS.128 per two FMAs) and saturates the SM's shared-memory pipe with four
// warps at about half the fp64 rate; the MMA fragments live in registers, so the inner loop has no memory operation.
// Fragment maps (g = lane >> 2, q = lane & 3):  A/B operand block b, k-step kb: L[8b + g][4kb + q];
// accumulator block (rb, cb): T[8rb + g][8cb + 2q + {0, 1}].  Tiles are column-major (element (r, c) at c*32 + r).
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void frag_load(const double* t, double (&f)[TILE], int lane) {
  const double* p = t + (lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int b = 0; b < 4; b++)
#pragma unroll
    for (int kb = 0; kb < 8; kb++) f[b*8 + kb] = __ldcg(p + 4*kb*TILE + 8*b);
}
__device__ __forceinline__ void cfrag_load(const double* t, double (&c)[TILE], int lane) {
  const double* p = t + 2*(lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 4; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++) { c[(rb*4 + cb)*2] = __ldcg(p + 8*cb*TILE + 8*rb); c[(rb*4 + cb)*2 + 1] = __ldcg(p + (8*cb + 1)*TILE + 8*rb); }
}
__device__ __forceinline__ void cfrag_store(double* t, const double (&c)[TILE], int lane) {
  double* p = t + 2*(lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 4; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++) { p[8*cb*TILE + 8*rb] = c[(rb*4 + cb)*2]; p[(8*cb + 1)*TILE + 8*rb] = c[(rb*4 + cb)*2 + 1]; }
}
// c -= A B^T with A, B given as operand fragments
__device__ __forceinline__ void frag_gemm_sub(double (&c)[TILE], const double (&a)[TILE], const double (&b)[TILE]) {
#pragma unroll
  for (int kb = 0; kb < 8; kb++)
#pragma unroll
    for (int rb = 0; rb < 4; rb++) {
      const double na = -a[rb*8 + kb];
#pragma unroll
      for (int cb = 0; cb < 4; cb++) dmma(c[(rb*4 + cb)*2], c[(rb*4 + cb)*2 + 1], na, b[cb*8 + kb]);
    }
}

}  // namespace dynoba
