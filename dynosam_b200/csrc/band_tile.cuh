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

// ---- fp64 tensor-core (DMMA) products of 32x32 tiles, in two shapes.  Tiles are column-major (element (r, c) at c*32 + r);
// g = lane >> 2, q = lane & 3.
//
// m8n8k4 set (dmma8, frag8_*, cfrag8_*): T(32x32) -= LI LK^T as 128 x mma.m8n8k4.  Used by the band spine (rank-8 steps
// as its TRSM panels appear) and by the selected inversion (kernels_cov.cu), whose transposed loaders share these maps:
// operand block b, k-step kb: L[8b + g][4kb + q];  accumulator block (rb, cb): T[8rb + g][8cb + 2q + {0, 1}].
__device__ __forceinline__ void dmma8(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void frag8_load(const double* t, double (&f)[TILE], int lane) {
  const double* p = t + (lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int b = 0; b < 4; b++)
#pragma unroll
    for (int kb = 0; kb < 8; kb++) f[b*8 + kb] = __ldcg(p + 4*kb*TILE + 8*b);
}
__device__ __forceinline__ void cfrag8_load(const double* t, double (&c)[TILE], int lane) {
  const double* p = t + 2*(lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 4; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++) { c[(rb*4 + cb)*2] = __ldcg(p + 8*cb*TILE + 8*rb); c[(rb*4 + cb)*2 + 1] = __ldcg(p + (8*cb + 1)*TILE + 8*rb); }
}
__device__ __forceinline__ void cfrag8_store(double* t, const double (&c)[TILE], int lane) {
  double* p = t + 2*(lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 4; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++) { p[8*cb*TILE + 8*rb] = c[(rb*4 + cb)*2]; p[(8*cb + 1)*TILE + 8*rb] = c[(rb*4 + cb)*2 + 1]; }
}
// c -= A B^T with A, B given as operand fragments
__device__ __forceinline__ void frag8_gemm_sub(double (&c)[TILE], const double (&a)[TILE], const double (&b)[TILE]) {
#pragma unroll
  for (int kb = 0; kb < 8; kb++)
#pragma unroll
    for (int rb = 0; rb < 4; rb++) {
      const double na = -a[rb*8 + kb];
#pragma unroll
      for (int cb = 0; cb < 4; cb++) dmma8(c[(rb*4 + cb)*2], c[(rb*4 + cb)*2 + 1], na, b[cb*8 + kb]);
    }
}

// m16n8k16 set (dmma16, frag16_*, cfrag16_*, stage16_*): the same product as 16 x mma.m16n8k16, which issues the
// 32x32x32 update in half the tensor-pipe cycles of the m8n8k4 form (tools/ubench/tile_update.cu).  Used by the band
// factorisation's worker pools.  PTX fragment maps:  A (16x16) a[i]: row g + 8(i&1), col q + 4(i>>1);
// B (16x8) b[i]: k = q + 4i, n = g;  C (16x8) c[i]: row g + 8(i>>1), col 2q + (i&1).
// Operand fragment of a tile L for k-step kb (columns 16kb .. 16kb+15), 16 per lane:  f[cb*4 + j] = L[8cb + g][16kb + q + 4j]
// (cb: 8-row block).  f[cb*4 .. cb*4+3] is the B fragment of row block cb, and the A fragment of 16-row block rb is the
// same registers: a[i] = f[(2rb + (i&1))*4 + (i>>1)].  So one fragment serves both sides, and L L^T loads L once.  An
// update runs k-step by k-step: 16 + 16 operand registers live instead of 64.
// Accumulator (32 per lane):  c[(rb*4 + cb)*4 + i] = T[16rb + g + 8(i>>1)][8cb + 2q + (i&1)].
constexpr int KF16 = 16;   // operand fragment registers per k-step
// c[c0 .. c0+3] += A B^T, A: one A fragment (8 values), B: fragment b[b0 .. b0+3]
__device__ __forceinline__ void dmma16(double (&c)[TILE], int c0, const double (&a)[8], const double (&b)[KF16], int b0) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, {%12, %13, %14, %15}, {%0, %1, %2, %3};"
               : "+d"(c[c0]), "+d"(c[c0 + 1]), "+d"(c[c0 + 2]), "+d"(c[c0 + 3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[b0]), "d"(b[b0 + 1]), "d"(b[b0 + 2]), "d"(b[b0 + 3]));
}
// operand fragment of k-step kb from a tile in global memory (L2: the tiles are written by other SMs)
__device__ __forceinline__ void frag16_load(const double* t, double (&f)[KF16], int kb, int lane) {
  const double* p = t + (16*kb + (lane & 3))*TILE + (lane >> 2);
#pragma unroll
  for (int cb = 0; cb < 4; cb++)
#pragma unroll
    for (int j = 0; j < 4; j++) f[cb*4 + j] = __ldcg(p + 4*j*TILE + 8*cb);
}
// the same of the tile's TRANSPOSE: f[cb*4 + j] = L[16kb + q + 4j][8cb + g] (the joint covariance's backward sweep)
__device__ __forceinline__ void frag16_load_t(const double* t, double (&f)[KF16], int kb, int lane) {
  const double* p = t + (lane >> 2)*TILE + 16*kb + (lane & 3);
#pragma unroll
  for (int cb = 0; cb < 4; cb++)
#pragma unroll
    for (int j = 0; j < 4; j++) f[cb*4 + j] = __ldcg(p + 8*cb*TILE + 4*j);
}
// Shared-memory stage of a tile: 32 columns of 32 doubles (stride 32, 8 KB, no padding), rows XOR-swizzled per column:
// element (r, c) at c*32 + (r ^ 4(c & 3)).  The swizzle flips row bits 2-3 only, so every 16-byte pair of rows (2p, 2p+1)
// stays together and cp.async fills a stage with 16-byte copies (stage16_prefetch).
// Why each LDS.64 of frag16_load_s is conflict-free: one load instruction reads, per lane, column c = 16kb + 4j + q (so
// c & 3 = q) and row r = 8cb + g.  A 64-bit shared load is served per half-warp, 16 lanes x 8 bytes = the 32 banks once,
// so it is conflict-free when the 16 lanes of a half-warp hit 16 distinct 8-byte bank pairs, i.e. distinct addresses mod
// 16 doubles.  c*32 is 0 mod 16; (8cb + g) ^ 4q mod 16 has bits 0-1 = g & 3 and bits 2-3 = (2(cb & 1) + (g >> 2)) ^ q.  In a
// half-warp g >> 2 is fixed and (g & 3, q) runs over all 16 pairs, so the 16 addresses are distinct.  (Unswizzled stride
// 32 would put the four q of a half-warp on one bank pair: 4-way.)
__device__ __forceinline__ int stage16_index(int r, int c) { return c*TILE + (r ^ ((c & 3) << 2)); }
__device__ __forceinline__ void frag16_load_s(const double* s, double (&f)[KF16], int kb, int lane) {
  const int g = lane >> 2, q = lane & 3;
  const double* p = s + (16*kb + q)*TILE;
#pragma unroll
  for (int cb = 0; cb < 4; cb++)
#pragma unroll
    for (int j = 0; j < 4; j++) f[cb*4 + j] = p[4*j*TILE + ((8*cb + g) ^ (q << 2))];
}
// asynchronous copy (cp.async, 16 bytes per request) of a column-major 32x32 tile into a swizzled stage by NTHR threads
// (32: one warp; 256: a CTA), `tid` = this thread's index among them; the caller commits the group
template <int NTHR>
__device__ __forceinline__ void stage16_prefetch(double* s, const double* t, int tid) {
#pragma unroll
  for (int i = 0; i < 512/NTHR; i++) {
    const int ch = tid + NTHR*i, c = ch >> 4, r = 2*(ch & 15);
    const unsigned dst = (unsigned)__cvta_generic_to_shared(s + stage16_index(r, c));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(t + c*TILE + r) : "memory");
  }
}
__device__ __forceinline__ void cfrag16_load(const double* t, double (&c)[TILE], int lane) {
  const double* p = t + 2*(lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 2; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++)
#pragma unroll
      for (int i = 0; i < 4; i++) c[(rb*4 + cb)*4 + i] = __ldcg(p + (8*cb + (i & 1))*TILE + 16*rb + 8*(i >> 1));
}
// to a column-major tile in global or shared memory
__device__ __forceinline__ void cfrag16_store(double* t, const double (&c)[TILE], int lane) {
  double* p = t + 2*(lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 2; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++)
#pragma unroll
      for (int i = 0; i < 4; i++) p[(8*cb + (i & 1))*TILE + 16*rb + 8*(i >> 1)] = c[(rb*4 + cb)*4 + i];
}
// c -= A B^T over one k-step, A and B given as operand fragments of that k-step (a == b allowed).  A is negated one A
// fragment at a time, so only 8 more registers are live.
__device__ __forceinline__ void frag16_gemm_sub(double (&c)[TILE], const double (&a)[KF16], const double (&b)[KF16]) {
#pragma unroll
  for (int rb = 0; rb < 2; rb++) {
    double na[8];
#pragma unroll
    for (int i = 0; i < 8; i++) na[i] = -a[(2*rb + (i & 1))*4 + (i >> 1)];
#pragma unroll
    for (int cb = 0; cb < 4; cb++) dmma16(c, (rb*4 + cb)*4, na, b, cb*4);
  }
}
// c -= A B^T for two tiles in swizzled stages (sa == sb: c -= A A^T, A loaded once)
__device__ __forceinline__ void stage16_gemm_sub(double (&c)[TILE], const double* sa, const double* sb, int lane) {
#pragma unroll
  for (int kb = 0; kb < 2; kb++) {
    double fb[KF16];
    frag16_load_s(sb, fb, kb, lane);
    if (sa == sb) frag16_gemm_sub(c, fb, fb);
    else {
      double fa[KF16];
      frag16_load_s(sa, fa, kb, lane);
      frag16_gemm_sub(c, fa, fb);
    }
  }
}

}  // namespace dynoba
