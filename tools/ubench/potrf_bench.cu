// Micro-benchmark of the spine's 32x32 potrf variants in isolation (one warp), optionally with spinning sibling warps.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xcompiler -fopenmp -I../../dynosam_b200/csrc potrf_bench.cu -o potrf_bench
#include <cstdio>
#include "../../dynosam_b200/csrc/kernels_band.cu"
using namespace dynoba;

template <int V>
__device__ __noinline__ void big_body(double* sX, double* o, int lane) {
  double r[TILE];
#pragma unroll
  for (int c = 0; c < TILE; c++) r[c] = lane + c + V;
#pragma unroll
  for (int rep = 0; rep < 6; rep++) { double fa[TILE], fb[TILE];
#pragma unroll
    for (int k = 0; k < TILE; k++) { fa[k] = sX[(k*37 + lane + rep + V) % TSZ]; fb[k] = sX[(k*11 + lane + rep) % TSZ]; }
    frag_gemm_sub(r, fa, fb); }   // unrolled: a distinct ~1k-instruction body per copy
  double s2 = 0;
#pragma unroll
  for (int c = 0; c < TILE; c++) s2 += r[c];
  if (s2 == 12345.678 + V) o[lane] = s2;
}
template <int V> struct BigRun { static __device__ void run(double* sX, double* o, int lane, int which) { if (which == V) big_body<V>(sX, o, lane); else BigRun<V - 1>::run(sX, o, lane, which); } };
template <> struct BigRun<-1> { static __device__ void run(double*, double*, int, int) {} };

// sibling modes: 0 exit, 1 poll (ev_wait-style), 2 rank-32 updates (LDS.128 + DFMA) on warps with (warp & mask) != 0
__global__ void potrf_bench(double* out, long long* cyc, int mode, int iters, int sib_mode, int sib_mask) {
  __shared__ double sPan[4*PANSZ];
  __shared__ double sIv[TILE];
  __shared__ double sP[256];
  __shared__ double sX[2*TSZ];
  __shared__ volatile int ev[EV_N];
  __shared__ volatile int stop;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < EV_N) ev[threadIdx.x] = 0;
  if (threadIdx.x == 0) stop = 0;
  for (int i = threadIdx.x; i < 2*TSZ; i += blockDim.x) sX[i] = 1e-3*(i % 37);
  __syncthreads();
  if (warp != 0) {
    const bool heavy = sib_mode >= 2 && (warp & sib_mask) != 0;
    if (sib_mode == 0) return;
    if (!heavy) {
      if (lane == 0) { int spins = 0; while (stop == 0) { if (++spins > 16) __nanosleep(20); } }
      __syncwarp();
      return;
    }
    double r[TILE];
#pragma unroll
    for (int c = 0; c < TILE; c++) r[c] = lane + c;
    if (sib_mode == 2) { while (stop == 0) spine_rank32(r, sX, sX + TSZ, false, ev, -1, 0, lane); }
    else { int w = warp; while (stop == 0) { BigRun<15>::run(sX, out + 64, lane, w & 15); w += 3; if (lane == 0) __nanosleep(sib_mode == 3 ? 2000 : 200); __syncwarp(); } }
    double s2 = 0;
#pragma unroll
    for (int c = 0; c < TILE; c++) s2 += r[c];
    if (s2 == 12345.678) out[40 + warp] = s2;
    return;
  }
  double row0[TILE], row[TILE];
#pragma unroll
  for (int c = 0; c < TILE; c++) { const int d = lane > c ? lane - c : c - lane; row0[c] = (d == 0 ? 8.0 : 0.0) + 1.0/(1.0 + d); }
  long long total = 0, prof[3] = {0, 0, 0}; bool ok = true;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int c = 0; c < TILE; c++) row[c] = row0[c];
    __syncwarp();
    const long long t0 = clock64();
    if (mode == 0) ok &= spine_potrf(row, lane, sPan, sIv, ev, it + 1, prof);
    else if (mode == 1) { spine_rank32(row, sX, sX + TSZ, false, ev, -1, 0, lane); }
    else { spine_trsm(row, lane, sPan, sIv, ev, 0, sX, -1); }
    total += clock64() - t0;
  }
  double s = 0.0;
#pragma unroll
  for (int c = 0; c < TILE; c++) if (c <= lane) s += row[c];
  out[lane] = s + (ok ? 0.0 : 1e300);
  if (lane == 0) { cyc[0] = total/iters; for (int k = 0; k < 3; k++) cyc[1 + k] = prof[k]/iters; stop = 1; }
}

int main() {
  double* out; long long* cyc; cudaMalloc(&out, 128*8); cudaMalloc(&cyc, 32);
  const char* names[3] = {"spine_potrf", "spine_rank32", "spine_trsm"};
  struct Cfg { int nw, sib, mask; const char* what; } cfgs[] = {
    {1, 0, 0, "alone"}, {8, 1, 0, "7 polling siblings"}, {8, 2, 4, "heavy on warps 4-7 (same scheduler as warp 0: warp 4)"},
    {8, 2, 3, "heavy on warps 1,2,3,5,6,7 (other schedulers), warp 4 polls"}, {8, 2, 7, "heavy on all 7 siblings"},
    {8, 3, 3, "big code (16 x 1.6k-instr bodies), low duty, other schedulers"}, {8, 4, 3, "big code, medium duty, other schedulers"}, {8, 4, 7, "big code, medium duty, all siblings"} };
  for (auto& c : cfgs) for (int mode = 0; mode < 3; mode++) {
    potrf_bench<<<1, 32*c.nw>>>(out, cyc, mode, 200, c.sib, c.mask);
    cudaDeviceSynchronize();
    long long h[4]; cudaMemcpy(h, cyc, 32, cudaMemcpyDeviceToHost);
    printf("%-14s %8lld cycles  [load %lld, factor %lld, trailing %lld]   %s  (%s)\n", names[mode], h[0], h[1], h[2], h[3], c.what, cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}
