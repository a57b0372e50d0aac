// kernels_cov.cu -- marginal covariances: gtsam::Marginals(graph, values, CHOLESKY).marginalCovariance(key) for every
// variable kind, from the plain band factor S = L L^T of the undamped reduced system (dynoba_marginal_covariance).
//
// Selected inversion.  Sigma = S^-1 restricted to the tile band of L is computed in place over L's tiles, backward over
// the tile columns K = NT-1 ... 0 with B = K+1 .. min(K+WB, NT-1) (tests/selinv_reference.py is the executable
// statement):
//     Sigma(B,K) = -Sigma(B,B) L(B,K) L_KK^-1            (X tiles)
//     Sigma(K,K) = L_KK^-T (L_KK^-1 - L(B,K)^T Sigma(B,K))
// Every Sigma(I,J) it reads lies inside the band; for I < J it is the transpose of the stored tile (J, I).  L_KK^-1 are
// the factorisation's diagonal-tile inverses (diag_inverse_kernel; nothing overwrites them afterwards).
// One persistent dataflow kernel, one warp per tile task, tasks in a fixed global order that every warp walks in
// order (all warps co-resident: cooperative launch), so a task only ever waits for tasks of a smaller index.  Per column
// K, in order:
//   X(K, dd)   dd = 1..WB:  X = -(sum_J Sigma(K+dd, J) L(J,K)) L_KK^-1 and its share P = L(K+dd,K)^T X of the diagonal
//              tile, both into a staging ring (column K's L tiles are still read by its other X tasks)
//   D(K)       Sigma(K,K) = L_KK^-T (L_KK^-1 - sum_dd P_dd), written symmetric over the diagonal tile
//   C(K, dd)   copies X(K, dd) over L(K+dd, K) once D(K) has seen every X of the column (so every read of L(., K) is done)
// The terms of X(K, dd) are summed from J = K+WB down, so the ones that need column K+1 come last: a column's X tasks
// start while the columns after it are still in flight (the skewed wavefront of the factorisation).
#include <algorithm>
#include <cooperative_groups.h>
#include "band_tile.cuh"
#include "landmark.cuh"

namespace dynoba {

constexpr int SEL_WARPS = 4;
constexpr int COV_WARPS = 4;

// m8n8k4 operand fragments (band_tile.cuh, frag8 maps) of a column-major tile's TRANSPOSE, from global memory; of a tile / of its
// transpose staged in shared memory
__device__ __forceinline__ void frag8_load_t(const double* t, double (&f)[TILE], int lane) {
  const double* p = t + (lane >> 2)*TILE + (lane & 3);
#pragma unroll
  for (int b = 0; b < 4; b++)
#pragma unroll
    for (int kb = 0; kb < 8; kb++) f[b*8 + kb] = __ldcg(p + 8*b*TILE + 4*kb);
}
__device__ __forceinline__ void frag8_load_s(const double* t, double (&f)[TILE], int lane) {
  const double* p = t + (lane & 3)*TILE + (lane >> 2);
#pragma unroll
  for (int b = 0; b < 4; b++)
#pragma unroll
    for (int kb = 0; kb < 8; kb++) f[b*8 + kb] = p[4*kb*TILE + 8*b];
}
__device__ __forceinline__ void frag8_load_ts(const double* t, double (&f)[TILE], int lane) {
  const double* p = t + (lane >> 2)*TILE + (lane & 3);
#pragma unroll
  for (int b = 0; b < 4; b++)
#pragma unroll
    for (int kb = 0; kb < 8; kb++) f[b*8 + kb] = p[8*b*TILE + 4*kb];
}

struct SelJob {
  double* tiles; const double* linv; int* flags;    // plain chain: tiles [NT][WB+1][TILE2], linv [NT][TILE2]
  double* stage;                                      // [R][WB][2][TILE2]: X and P of column K in ring slot K % R
  int NT, WB, R;
};
__device__ __forceinline__ int* sel_done(const SelJob& j, int K, int t) { return j.flags + (size_t)K*(j.WB + 1) + t; }   // Sigma tile (K, t) in place
__device__ __forceinline__ int* sel_x(const SelJob& j, int K, int dd) { return j.flags + (size_t)j.NT*(j.WB + 1) + (size_t)K*(j.WB + 1) + dd; }
__device__ __forceinline__ double* sel_tile(const SelJob& j, int K, int t) { return j.tiles + ((size_t)K*(j.WB + 1) + t)*TILE2; }
__device__ __forceinline__ double* sel_stage(const SelJob& j, int K, int dd, int which) {
  return j.stage + (((size_t)(K % j.R)*j.WB + (dd - 1))*2 + which)*TILE2;
}

__device__ __forceinline__ void selinv_x(const SelJob& j, int K, int dd, double* sm, int lane) {
  const int I = K + dd, Jhi = min(K + j.WB, j.NT - 1);
  double acc[TILE];
#pragma unroll
  for (int e = 0; e < TILE; e++) acc[e] = 0.0;
  for (int J = Jhi; J > K; J--) {        // acc -= Sigma(I, J) L(J, K)
    double a[TILE], b[TILE];
    if (I >= J) { wait_flag(sel_done(j, J, I - J), lane); frag8_load(sel_tile(j, J, I - J), a, lane); }
    else { wait_flag(sel_done(j, I, J - I), lane); frag8_load_t(sel_tile(j, I, J - I), a, lane); }
    frag8_load_t(sel_tile(j, K, J - K), b, lane);
    frag8_gemm_sub(acc, a, b);
  }
  const double* linv = j.linv + (size_t)K*TILE2;
  double a[TILE], b[TILE], c[TILE];
  __syncwarp(); cfrag8_store(sm, acc, lane); __syncwarp();
  frag8_load_s(sm, a, lane); frag8_load_t(linv, b, lane);
#pragma unroll
  for (int e = 0; e < TILE; e++) c[e] = 0.0;
  frag8_gemm_sub(c, a, b);                 // c = -acc L_KK^-1 = -X
  __syncwarp(); cfrag8_store(sm, c, lane); __syncwarp();
  frag8_load_ts(sm, b, lane); frag8_load_t(sel_tile(j, K, dd), a, lane);
#pragma unroll
  for (int e = 0; e < TILE; e++) acc[e] = 0.0;
  frag8_gemm_sub(acc, a, b);               // acc = L(I,K)^T X = P
#pragma unroll
  for (int e = 0; e < TILE; e++) c[e] = -c[e];
  // the ring slot's previous column (K + R) must have been copied out
  if (K + j.R < j.NT && dd <= min(j.WB, j.NT - 1 - (K + j.R))) wait_flag(sel_done(j, K + j.R, dd), lane);
  cfrag8_store(sel_stage(j, K, dd, 0), c, lane);
  cfrag8_store(sel_stage(j, K, dd, 1), acc, lane);
  set_flag(sel_x(j, K, dd), lane);
}

__device__ __forceinline__ void selinv_d(const SelJob& j, int K, double* sm, int lane) {
  const int m = min(j.WB, j.NT - 1 - K);
  const double* linv = j.linv + (size_t)K*TILE2;
  double acc[TILE];
  cfrag8_load(linv, acc, lane);
  for (int dd = 1; dd <= m; dd++) {      // M = L_KK^-1 - sum_dd P_dd
    wait_flag(sel_x(j, K, dd), lane);
    double p[TILE];
    cfrag8_load(sel_stage(j, K, dd, 1), p, lane);
#pragma unroll
    for (int e = 0; e < TILE; e++) acc[e] -= p[e];
  }
  double a[TILE], b[TILE];
  __syncwarp(); cfrag8_store(sm, acc, lane); __syncwarp();
  frag8_load_ts(sm, b, lane); frag8_load_t(linv, a, lane);
#pragma unroll
  for (int e = 0; e < TILE; e++) acc[e] = 0.0;
  frag8_gemm_sub(acc, a, b);               // acc = -L_KK^-T M = -Sigma(K,K)
  __syncwarp(); cfrag8_store(sm, acc, lane); __syncwarp();
  double* t = sel_tile(j, K, 0);
#pragma unroll
  for (int c = 0; c < TILE; c++) t[c*TILE + lane] = -(lane >= c ? sm[c*TILE + lane] : sm[lane*TILE + c]);   // the lower triangle, mirrored
  set_flag(sel_done(j, K, 0), lane);
}

__device__ __forceinline__ void selinv_c(const SelJob& j, int K, int dd, int lane) {
  wait_flag(sel_done(j, K, 0), lane);
  const double* s = sel_stage(j, K, dd, 0);
  double* t = sel_tile(j, K, dd);
#pragma unroll 8
  for (int c = 0; c < TILE; c++) t[c*TILE + lane] = __ldcg(s + c*TILE + lane);
  set_flag(sel_done(j, K, dd), lane);
}

__global__ void __launch_bounds__(SEL_WARPS*32) band_selinv_kernel(SelJob j) {
  extern __shared__ double sel_sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* sm = sel_sm + (size_t)warp*TILE2;
  const long long per = 2LL*j.WB + 1, ntasks = per*j.NT, nworkers = (long long)gridDim.x*SEL_WARPS;
  for (long long t = (long long)blockIdx.x*SEL_WARPS + warp; t < ntasks; t += nworkers) {
    const int K = j.NT - 1 - (int)(t/per), u = (int)(t%per), m = min(j.WB, j.NT - 1 - K);
    if (u < j.WB) { if (u + 1 <= m) selinv_x(j, K, u + 1, sm, lane); }
    else if (u == j.WB) selinv_d(j, K, sm, lane);
    else if (u - j.WB <= m) selinv_c(j, K, u - j.WB, lane);
  }
}

size_t selinv_stage_count(int WB) { return (size_t)(WB + 2)*std::max(WB, 1)*2*TILE2; }

int launch_band_selinv(const BandProb& P, int WB, double* stage, cudaStream_t s) {
  static int per_sm = -1, sms = 1;
  const size_t smem = (size_t)SEL_WARPS*TILE2*sizeof(double);
  if (per_sm < 0) {
    cudaFuncSetAttribute(band_selinv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, band_selinv_kernel, SEL_WARPS*32, smem);
    sms = device_sm_count();
    if (per_sm < 1) per_sm = 1;
  }
  SelJob j{ P.tiles, P.linv, P.flags, stage, P.NT, WB, WB + 2 };
  cudaMemsetAsync(P.flags, 0, (size_t)2*P.NT*(WB + 1)*sizeof(int), s);
  const long long ntasks = (2LL*WB + 1)*P.NT;
  const int grid = (int)std::max(1LL, std::min((long long)per_sm*sms, (ntasks + SEL_WARPS - 1)/SEL_WARPS));
  void* args[] = { (void*)&j };
  cudaLaunchCooperativeKernel((void*)band_selinv_kernel, dim3(grid), dim3(SEL_WARPS*32), args, smem, s);
  return 2;
}

// ---- joint marginal covariances (dynoba_joint_marginal_covariance): X = S^-1 E_C over the plain band factor L, E_C the
// unit columns of the requested scalars C.  L^-1 E_C is zero above the first requested scalar, so both sweeps run over the
// tile columns [J0, NT) only, J0 the tile of min(C):
//     forward   Y_J = L_JJ^-1 (E_J - sum_{t=1..WB} L(J, J-t) Y_{J-t})          J = J0 .. NT-1
//     backward  X_J = L_JJ^-T (Y_J - sum_{t=1..WB} L(J+t, J)^T X_{J+t})      J = NT-1 .. J0
// (tests/joint_reference.py is the executable statement).  The panel of right-hand sides is cut into chunks of
// SWEEP_COLS columns, one CTA each; a chunk's panel tiles are square and hold the TRANSPOSE (tile (J, k) element (r, c) =
// X[32J + c][32k + r]), so every product is T -= A B^T of two 32x32 tiles on the m16n8k16 loaders of band_tile.cuh:
//     forward   Y^T_J -= Y^T_{J-t} L(J, J-t)^T        backward  X^T_J -= X^T_{J+t} L(J+t, J)
// The WB products of a tile column are dealt over the CTA's warps, their partial sums added in shared memory, and one
// warp multiplies by the factorisation's diagonal-tile inverse.  Work and memory: (NT - J0) WB |C| / 32 tile products and
// (NT - J0) |C| / 32 panel tiles.
constexpr int SWEEP_COLS = 32;    // right-hand sides per chunk (a multiple of 8: one n8 block per 8 columns)
constexpr int SWEEP_WARPS = 8;    // warps sharing a tile column's WB products
static_assert(SWEEP_COLS == TILE, "the panel's tiles are square");

struct SweepJob {
  const double* tiles; const double* linv; int TPC, NT, WB, J0;
  const int* cs; int nc;          // [nc] band scalar of each right-hand side's unit entry
  double* panel; int nchunk;      // [NT - J0][nchunk][TILE2]
};
// operand fragment (frag16_load's map) of a tile this CTA wrote: plain loads, global or shared memory
__device__ __forceinline__ void frag16_load_p(const double* t, double (&f)[KF16], int kb, int lane) {
  const double* p = t + (16*kb + (lane & 3))*TILE + (lane >> 2);
#pragma unroll
  for (int cb = 0; cb < 4; cb++)
#pragma unroll
    for (int j = 0; j < 4; j++) f[cb*4 + j] = p[4*j*TILE + 8*cb];
}

template <bool FWD>
__device__ __forceinline__ void sweep_column(const SweepJob& j, int J, const int* cs, double* sm, int warp, int lane) {
  const int k = blockIdx.x;
  double* part = sm + (size_t)warp*TILE2;
  double* z = sm + (size_t)SWEEP_WARPS*TILE2;
  double* pj = j.panel + ((size_t)(J - j.J0)*j.nchunk + k)*TILE2;
  double acc[TILE];
#pragma unroll
  for (int e = 0; e < TILE; e++) acc[e] = 0.0;
  const int m = FWD ? min(j.WB, J - j.J0) : min(j.WB, j.NT - 1 - J);
  for (int t = 1 + warp; t <= m; t += SWEEP_WARPS) {
    const int I = FWD ? J - t : J + t;
    const double* Lt = FWD ? j.tiles + ((size_t)I*j.TPC + t)*TILE2 : j.tiles + ((size_t)J*j.TPC + t)*TILE2;
    const double* Pt = j.panel + ((size_t)(I - j.J0)*j.nchunk + k)*TILE2;
    double fa[2][KF16], fb[2][KF16];
#pragma unroll
    for (int kb = 0; kb < 2; kb++) {
      if (FWD) frag16_load(Lt, fb[kb], kb, lane); else frag16_load_t(Lt, fb[kb], kb, lane);
      frag16_load_p(Pt, fa[kb], kb, lane);
    }
#pragma unroll
    for (int kb = 0; kb < 2; kb++) frag16_gemm_sub(acc, fa[kb], fb[kb]);
  }
  cfrag16_store(part, acc, lane);
  __syncthreads();
  for (int e = threadIdx.x; e < TILE2; e += SWEEP_WARPS*32) {   // Z^T = E^T_J (forward) / Y^T_J (backward) + partial sums
    double s = FWD ? (cs[e & 31] == J*TILE + (e >> 5) ? 1.0 : 0.0) : pj[e];
#pragma unroll
    for (int w = 0; w < SWEEP_WARPS; w++) s += sm[(size_t)w*TILE2 + e];
    z[e] = s;
  }
  __syncthreads();
  if (warp == 0) {            // Y^T_J = Z^T L_JJ^-T,  X^T_J = Z^T L_JJ^-1
    const double* li = j.linv + (size_t)J*TILE2;
#pragma unroll
    for (int e = 0; e < TILE; e++) acc[e] = 0.0;
#pragma unroll
    for (int kb = 0; kb < 2; kb++) {
      double fa[KF16], fb[KF16];
      frag16_load_p(z, fa, kb, lane);
      if (FWD) frag16_load(li, fb, kb, lane); else frag16_load_t(li, fb, kb, lane);
      frag16_gemm_sub(acc, fa, fb);
    }
#pragma unroll
    for (int e = 0; e < TILE; e++) acc[e] = -acc[e];
    cfrag16_store(pj, acc, lane);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(SWEEP_WARPS*32) band_sweep_kernel(SweepJob j) {
  extern __shared__ double sw_sm[];     // [SWEEP_WARPS] partial sums | Z
  __shared__ int cs[SWEEP_COLS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < SWEEP_COLS) { const int c = blockIdx.x*SWEEP_COLS + threadIdx.x; cs[threadIdx.x] = c < j.nc ? j.cs[c] : -1; }
  __syncthreads();
  for (int J = j.J0; J < j.NT; J++) sweep_column<true>(j, J, cs, sw_sm, warp, lane);
  for (int J = j.NT - 1; J >= j.J0; J--) sweep_column<false>(j, J, cs, sw_sm, warp, lane);
}

size_t joint_panel_count(int NT, int J0, int nc) { return (size_t)(NT - J0)*((nc + SWEEP_COLS - 1)/SWEEP_COLS)*TILE2; }

int launch_band_sweeps(const BandProb& P, int WB, const int* cs, int nc, int J0, double* panel, cudaStream_t s) {
  const size_t smem = (size_t)(SWEEP_WARPS + 1)*TILE2*sizeof(double);
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(band_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
  const int nchunk = (nc + SWEEP_COLS - 1)/SWEEP_COLS;
  SweepJob j{ P.tiles, P.linv, P.TPC, P.NT, WB, J0, cs, nc, panel, nchunk };
  band_sweep_kernel<<<nchunk, SWEEP_WARPS*32, smem, s>>>(j);
  return 1;
}
// X[C, C] row-major from the panel: out[a*nc + b] = X[cs[a]][b]
__global__ void joint_gather_kernel(const double* __restrict__ panel, int nchunk, int J0, const int* __restrict__ cs, int nc,
                                    double* __restrict__ out) {
  const long long e = (long long)blockIdx.x*blockDim.x + threadIdx.x;
  if (e >= (long long)nc*nc) return;
  const int a = (int)(e/nc), b = (int)(e%nc), s = cs[a];
  out[e] = panel[((size_t)((s >> 5) - J0)*nchunk + b/SWEEP_COLS)*TILE2 + (size_t)(s & 31)*TILE + (b % SWEEP_COLS)];
}
int launch_joint_gather(const double* panel, int J0, const int* cs, int nc, double* out, cudaStream_t s) {
  const long long ne = (long long)nc*nc;
  joint_gather_kernel<<<(unsigned)((ne + 255)/256), 256, 0, s>>>(panel, (nc + SWEEP_COLS - 1)/SWEEP_COLS, J0, cs, nc, out);
  return 1;
}

// ---- pose-like blocks: cov[i] = Sigma(s_i .. s_i + d, s_i .. s_i + d), s_i = 6 * solver position of the i-th variable
__global__ void cov_pose_gather_kernel(const double* __restrict__ tiles, int TPC, const int* __restrict__ spos, int n, int d,
                                       double* __restrict__ out) {
  const long long e = (long long)blockIdx.x*blockDim.x + threadIdx.x;
  if (e >= (long long)n*d*d) return;
  const int i = (int)(e/(d*d)), r = (int)(e%(d*d))/d, c = (int)(e%d);
  out[e] = band_sym(tiles, TPC, spos[i] + r, spos[i] + c);
}
int launch_cov_pose_gather(const double* tiles, int TPC, const int* spos, int n, int d, double* out, cudaStream_t s) {
  if (n == 0) return 0;
  const long long ne = (long long)n*d*d;
  cov_pose_gather_kernel<<<(unsigned)((ne + 255)/256), 256, 0, s>>>(tiles, TPC, spos, n, d, out);
  return 1;
}
// ---- landmarks: rows of a per-landmark table (w doubles each) in caller order
__global__ void cov_rows_gather_kernel(const double* __restrict__ src, const int* __restrict__ rows, int n, int w, double* __restrict__ out) {
  const long long e = (long long)blockIdx.x*blockDim.x + threadIdx.x;
  if (e >= (long long)n*w) return;
  out[e] = src[(size_t)rows[e/w]*w + e%w];
}
int launch_cov_rows_gather(const double* src, const int* rows, int n, int w, double* out, cudaStream_t s) {
  if (n == 0) return 0;
  const long long ne = (long long)n*w;
  cov_rows_gather_kernel<<<(unsigned)((ne + 255)/256), 256, 0, s>>>(src, rows, n, w, out);
  return 1;
}

// One-landmark groups (window and per-landmark routes, flows), one warp per group as backsub_simple_kernel:
//   Sigma_l = V^-1 + V^-1 (sum_{a,b} U_a Sigma(p_a, p_b) U_b^T) V^-1,   U_a = B_f^T A_{f,s}  (DL x 6)
// over the terms a = (factor f, pose slot s) of the group; W = A^T B, so sum_{a,b} U_a Sigma_ab U_b^T = W^T Sigma_cc W.
// Lanes own the terms a; the term b of the inner loop is the same on every lane (its Jacobian reads are broadcasts).
template <int DL, int D, int JC, int PCOL0, int LCOL>
__device__ __forceinline__ void cov_term(const DevBlock& blk, int f, int sl, double (&U)[DL*6]) {
#pragma unroll
  for (int e = 0; e < DL*6; e++) U[e] = 0.0;
#pragma unroll
  for (int r = 0; r < D; r++) {
    double bm[DL], am[6];
#pragma unroll
    for (int k = 0; k < DL; k++) bm[k] = blk.J[(size_t)(r*JC + LCOL + k)*blk.stride + f];
#pragma unroll
    for (int c = 0; c < 6; c++) am[c] = blk.J[(size_t)(r*JC + PCOL0 + 6*sl + c)*blk.stride + f];
#pragma unroll
    for (int k = 0; k < DL; k++)
#pragma unroll
      for (int c = 0; c < 6; c++) U[k*6 + c] += bm[k]*am[c];
  }
}
template <int NP, int DL, int D, int PCOL0, int LCOL, int PSLOT0>
__global__ void __launch_bounds__(COV_WARPS*32)
cov_simple_kernel(DevBlock blk, const double* __restrict__ sig, int TPC, double* __restrict__ out, int* __restrict__ fail) {
  constexpr int JC = NP*6 + DL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*COV_WARPS + warp;
  if (g >= blk.n_groups || blk.grp_lmk[g] < 0) return;
  const int f0 = blk.grp_ptr[g], T = blk.grp_ptr[g+1] - f0;
  double V[DL*DL];
#pragma unroll
  for (int k = 0; k < DL*DL; k++) V[k] = 0.0;
  for (int i = lane; i < T; i += 32) {
    double Bm[D*DL];
#pragma unroll
    for (int r = 0; r < D; r++)
#pragma unroll
      for (int c = 0; c < DL; c++) Bm[r*DL + c] = blk.J[(size_t)(r*JC + LCOL + c)*blk.stride + f0 + i];
#pragma unroll
    for (int c1 = 0; c1 < DL; c1++)
#pragma unroll
      for (int c2 = 0; c2 <= c1; c2++)
#pragma unroll
        for (int r = 0; r < D; r++) V[c1*DL + c2] += Bm[r*DL + c1]*Bm[r*DL + c2];
  }
#pragma unroll
  for (int c1 = 0; c1 < DL; c1++)
#pragma unroll
    for (int c2 = 0; c2 <= c1; c2++) { V[c1*DL + c2] = warp_sum(V[c1*DL + c2]); V[c2*DL + c1] = V[c1*DL + c2]; }
  double Vi[DL*DL];
  if (!spd_inverse<DL>(V, Vi)) { if (lane == 0) atomicOr(fail, 1); return; }
  double Q[DL*DL];
#pragma unroll
  for (int k = 0; k < DL*DL; k++) Q[k] = 0.0;
  const int N = T*NP;
  for (int a = lane; a < N; a += 32) {
    const int fa = f0 + a/NP, sa = a%NP;
    const int pa = 6*blk.idx[(size_t)(PSLOT0 + sa)*blk.stride + fa];
    double Ua[DL*6];
    cov_term<DL, D, JC, PCOL0, LCOL>(blk, fa, sa, Ua);
    for (int b = 0; b < N; b++) {
      const int fb = f0 + b/NP, sb = b%NP;
      const int pb = 6*blk.idx[(size_t)(PSLOT0 + sb)*blk.stride + fb];
      double Ub[DL*6], G[DL*6];
      cov_term<DL, D, JC, PCOL0, LCOL>(blk, fb, sb, Ub);
#pragma unroll
      for (int e = 0; e < DL*6; e++) G[e] = 0.0;
#pragma unroll
      for (int c = 0; c < 6; c++)
#pragma unroll
        for (int c2 = 0; c2 < 6; c2++) {
          const double s = band_sym(sig, TPC, pa + c, pb + c2);
#pragma unroll
          for (int k = 0; k < DL; k++) G[k*6 + c2] += Ua[k*6 + c]*s;
        }
#pragma unroll
      for (int k1 = 0; k1 < DL; k1++)
#pragma unroll
        for (int k2 = 0; k2 < DL; k2++)
#pragma unroll
          for (int c = 0; c < 6; c++) Q[k1*DL + k2] += G[k1*6 + c]*Ub[k2*6 + c];
    }
  }
#pragma unroll
  for (int k = 0; k < DL*DL; k++) Q[k] = warp_sum(Q[k]);
  if (lane != 0) return;
  double VQ[DL*DL];
#pragma unroll
  for (int r = 0; r < DL; r++)
#pragma unroll
    for (int c = 0; c < DL; c++) { double s = 0; for (int k = 0; k < DL; k++) s += Vi[r*DL + k]*Q[k*DL + c]; VQ[r*DL + c] = s; }
  double* o = out + (size_t)blk.grp_lmk[g]*DL*DL;
#pragma unroll
  for (int r = 0; r < DL; r++)
#pragma unroll
    for (int c = 0; c <= r; c++) {
      double s = Vi[r*DL + c];
      for (int k = 0; k < DL; k++) s += VQ[r*DL + k]*Vi[k*DL + c];
      o[r*DL + c] = s; o[c*DL + r] = s;
    }
}
int launch_cov_simple(const DevBlock& blk, const double* sig, int TPC, double* out_point, double* out_flow, int* fail, cudaStream_t s) {
  if (blk.n_groups == 0) return 0;
  const int grid = (blk.n_groups + COV_WARPS - 1)/COV_WARPS;
  switch (blk.type) {
    case F_POSE2POINT3: case F_STEREO3: case F_LINEAR_PP3:
      cov_simple_kernel<1, 3, 3, 0, 6, 0><<<grid, COV_WARPS*32, 0, s>>>(blk, sig, TPC, out_point, fail); return 1;
    case F_HYBRID3: case F_HYBRID_STEREO3: case F_LINEAR_PPP3:
      cov_simple_kernel<2, 3, 3, 0, 12, 0><<<grid, COV_WARPS*32, 0, s>>>(blk, sig, TPC, out_point, fail); return 1;
    case F_FLOWPROJ2:
      cov_simple_kernel<1, 2, 2, 2, 0, 1><<<grid, COV_WARPS*32, 0, s>>>(blk, sig, TPC, out_flow, fail); return 1;
    default: return 0;
  }
}

}  // namespace dynoba
