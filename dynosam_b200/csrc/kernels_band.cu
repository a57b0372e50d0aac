// kernels_band.cu -- K5: Cholesky factorisation and solve of the reduced camera/object-motion system.
//
// Replaces GTSAM's multifrontal Cholesky on the COLAMD ordering (SURVEY.md 8a row a11, [GTSAM-ext]) for the
// reduced system that is left after the landmarks are eliminated.  With pose-like variables ordered by frame
// the system is banded (half-width = the co-visibility window, <= max track age), stored as 32x32 tiles.
// Hopper's wgmma has no fp64 shape: tile updates run on mma.sync (DMMA; m16n8k16 in the worker pools, m8n8k4 in the
// spine), triangular work on fp64 FMAs.
//
// A band Cholesky is one long dependency chain (potrf(K,K) -> trsm -> update -> potrf(K+1,K+1)), so the time axis is
// cut into CELLS (nested dissection in time; internal.cuh, tools/cell_proto.py): every cell is two chains that are
// eliminated towards a middle separator, chains next to a boundary separator carry their fill ("spike") with them,
// and the separators are solved last.  All chains of all cells of this GPU run in ONE persistent dataflow kernel
// (no grid-wide barriers), band_cholesky_dataflow_kernel_v3:
//   * one spine CTA per chain owns the sequential chain and the two tiles below it, in shared memory / registers;
//   * worker warps own one tile task at a time: every left-looking update T_IK -= L_IJ L_KJ^T as soon as the per-tile
//     "done" flags of the operand tiles are released, then the TRSM against L_KK; the spike tiles Z and the separator
//     block FF -= Z Z^T are more tasks of the same kind; one task per column folds the forward substitution in.
// The same kernel then factors the cell separator systems [M | Qa | Qb] (dense, M eliminated) and the boundary system.
// Solve = explicit inverses of the diagonal tiles (one warp each, fully parallel), backward sweep on a cluster of 8 CTAs
// per chain.
#include <algorithm>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <climits>
#include <chrono>
#include <vector>
#include <cooperative_groups.h>
#include "band_tile.cuh"

namespace cg = cooperative_groups;

namespace dynoba {

constexpr int TS = 40, TSZ = TILE*TS;      // column stride of the spine's shared-memory tiles that feed m8n8k4 operand fragments
constexpr int FF_CH = 16;                  // columns per FF accumulation task
constexpr int MAX_PROBS = 2*MAX_CELLS;

// x(row = lane) <- x * L^-T with L staged as sL[k*32 + c] = L[c][k]; sinv[c] = 1 / L[c][c].  Blocked by 8 columns: the
// serial chain is 8 x (mul, fma) per panel, the rank-8 update of the columns behind a panel has 24/16/8 independent chains.
__device__ __forceinline__ void tile_trsm(double (&x)[TILE], const double* sL, const double* sinv) {
#pragma unroll
  for (int p = 0; p < 4; p++) {
#pragma unroll
    for (int kk = 0; kk < 8; kk++) {
      const int k = 8*p + kk;
      const double l = x[k]*sinv[k];
      x[k] = l;
#pragma unroll
      for (int c = k + 1; c < 8*p + 8; c++) x[c] -= l*sL[k*TILE + c];
    }
    if (p < 3) {
#pragma unroll
      for (int c = 8*p + 8; c < TILE; c += 2) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const double2 b = *reinterpret_cast<const double2*>(sL + (8*p + j)*TILE + c);
          x[c] -= x[8*p + j]*b.x; x[c + 1] -= x[8*p + j]*b.y;
        }
      }
    }
  }
}
__device__ __forceinline__ void tile_load(const double* t, double (&r)[TILE], int lane) {
#pragma unroll
  for (int c = 0; c < TILE; c++) r[c] = __ldcg(t + c*TILE + lane);
}
__device__ __forceinline__ void tile_store(double* t, const double (&r)[TILE], int lane) {
#pragma unroll
  for (int c = 0; c < TILE; c++) t[c*TILE + lane] = r[c];
}
// stage a tile held one row per lane into shared memory (s[c*32 + row]) + reciprocals of its diagonal
__device__ __forceinline__ void tile_stage(double* s, const double (&r)[TILE], int lane) {
  __syncwarp();
#pragma unroll
  for (int c = 0; c < TILE; c++) s[c*TILE + lane] = r[c];
  __syncwarp();
}

// both flags set?  (non-blocking, acquire)
__device__ __forceinline__ bool flags_ready(const int* fa, const int* fb, int lane) {
  int ok = 0;
  if (lane == 0) ok = ld_acquire(fa) != 0 && ld_acquire(fb) != 0;
  return __shfl_sync(0xffffffffu, ok, 0) != 0;
}

// optional stage profile (dynoba_set_tuning "band_profile"): finish times of the spines and of the two worker pools
__device__ unsigned long long g_prof[40];
__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

// One launch of the factorisation kernel: np band problems of the same tile bandwidth WB.
struct CholJob { const BandProb* p; int np, WB, skew, any_spiked, ncols, band_ctas, profile; };   // band_ctas: worker CTAs of pool A
__device__ __forceinline__ int* flag_done(const BandProb& P) { return P.flags; }
__device__ __forceinline__ int* flag_pre(const BandProb& P) { return P.flags + (size_t)P.NT*P.TPC; }
__device__ __forceinline__ int* flag_ydone(const BandProb& P) { return P.flags + (size_t)2*P.NT*P.TPC; }
__device__ __forceinline__ int* flag_ffcnt(const BandProb& P) { return P.flags + (size_t)2*P.NT*P.TPC + P.NT; }

// acc -= sum_{J = Jlo..Jhi} A_J B_J^T  with A_J = tile (J, A0 - A1*J), B_J = tile (J, B0 - B1*J) of problem P (same: A == B);
// waits for the operand tiles' done flags.  stage: per-warp [2][2][TILE2] swizzled shared-memory operand stages (band_tile.cuh)
// -- while update J runs on the tensor pipe, the operand tiles of J+1 (when their flags are already up) stream into the
// other stage with cp.async, so the L2 latency leaves the critical path.  Updates are m16n8k16 (frag16_gemm_sub).
__device__ __forceinline__ void accumulate_updates(const BandProb& P, double (&acc)[TILE], int Jlo, int Jhi, int A0, int A1, int B0, int B1,
                                                   bool same, double* stage, int lane) {
  const int* done = flag_done(P);
  const int TPC = P.TPC;
  int st = 0; bool have = false;
  for (int J = Jlo; J <= Jhi; J++) {
    const size_t oA = (size_t)J*TPC + (A0 - A1*J), oB = (size_t)J*TPC + (B0 - B1*J);
    if (!have) {
      wait_flag(done + oB, lane);
      if (!same) wait_flag(done + oA, lane);
      stage16_prefetch<32>(stage + (size_t)(st*2 + 1)*TILE2, P.tiles + oB*TILE2, lane);
      if (!same) stage16_prefetch<32>(stage + (size_t)(st*2)*TILE2, P.tiles + oA*TILE2, lane);
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    bool next = false;
    if (J + 1 <= Jhi) {
      const size_t nA = (size_t)(J + 1)*TPC + (A0 - A1*(J + 1)), nB = (size_t)(J + 1)*TPC + (B0 - B1*(J + 1));
      next = flags_ready(done + nB, done + (same ? nB : nA), lane);
      if (next) {
        stage16_prefetch<32>(stage + (size_t)((st ^ 1)*2 + 1)*TILE2, P.tiles + nB*TILE2, lane);
        if (!same) stage16_prefetch<32>(stage + (size_t)((st ^ 1)*2)*TILE2, P.tiles + nA*TILE2, lane);
        asm volatile("cp.async.commit_group;" ::: "memory");
      }
    }
    if (next) asm volatile("cp.async.wait_group 1;" ::: "memory"); else asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    const double* sb = stage + (size_t)(st*2 + 1)*TILE2;
    stage16_gemm_sub(acc, same ? sb : stage + (size_t)(st*2)*TILE2, sb, lane);
    __syncwarp();            // the stage is free for the prefetch after next
    st ^= 1; have = next;
  }
}

// Band worker warp `wid` of `nworkers` (pool A).  Tasks of column K of a problem (slot dd):
//   dd <= WB        band tile (K + dd, K).  dd == 0, 1: workers apply the updates from columns J <= K-3 / K-2 ("pre"), the
//                   spine applies the rest and finishes; dd == 2: workers apply J <= K-1 ("pre"), the spine does the TRSM;
//                   dd >= 3: workers apply J <= K-1 and do the TRSM once done(K,K) is released
//   dd == WB + 1    rhs task: folds the forward substitution y_K = L_KK^-1 (g_K - sum_J L_KJ y_J) in
// Task order: skewed wavefronts s = skew*K + dd instead of column-major.  A worker processes its tasks in order and
// blocks on operands, so a task's lead over the spine has to cover its own serial work; the (WB - dd) updates of a tile
// near the diagonal need more lead than the short tasks far from it.  Every operand of a task has a strictly smaller s,
// so in-order blocking cannot deadlock (all CTAs are co-resident: cooperative launch).
__device__ __forceinline__ void tile_finish_trsm(const BandProb& P, double (&acc)[TILE], int K, double* tp, int* doneflag, double* sb, double* sinv, int lane) {
  // accumulator fragments (m16n8k16 C map) -> one row per lane, through the warp's shared-memory tile
  __syncwarp();
  cfrag16_store(sb, acc, lane);
  __syncwarp();
#pragma unroll
  for (int cc = 0; cc < TILE; cc++) acc[cc] = sb[cc*TILE + lane];
  const size_t oD = (size_t)K*P.TPC;
  wait_flag(flag_done(P) + oD, lane);
  __syncwarp();
#pragma unroll
  for (int cc = 0; cc < TILE; cc++) sb[cc*TILE + lane] = __ldcg(P.tiles + oD*TILE2 + cc*TILE + lane);
  __syncwarp();
  sinv[lane] = 1.0/sb[lane*TILE + lane];
  __syncwarp();
  tile_trsm(acc, sb, sinv);
  tile_store(tp, acc, lane);
  set_flag(doneflag, lane);
}

__device__ __forceinline__ void band_worker(const CholJob& job, int wid, int nworkers, double* sb, double* sinv, double* stage, int lane) {
  const int WB = job.WB, W1 = WB + 1, R = W1 + 1;          // task slots per column
  const int ncols = job.ncols;
  const int skew = job.skew, nj = (R + skew - 1)/skew;
  const long long per_s = (long long)job.np*nj;
  const long long ntasks = ((long long)skew*ncols + R)*per_s;
  for (long long t = wid; t < ntasks; t += nworkers) {
    const int sidx = (int)(t/per_s); const int u = (int)(t - (long long)sidx*per_s);
    const int q = u/nj, j = u - q*nj;
    const int dd = sidx%skew + skew*j, K = sidx/skew - j;
    if (dd >= R || K < 0 || K >= ncols) continue;
    const BandProb P = job.p[q];
    const int NT = P.NT, TPC = P.TPC;
    if (K >= NT) continue;
    int* done = flag_done(P); int* pre = flag_pre(P);
    if (dd == W1) {
      // ---- rhs task; rows >= Kend only collect the factored columns' part
      int* ydone = flag_ydone(P);
      double v = P.rhs[(size_t)K*TILE + lane];
      const int Jend = min(K, P.Kend);
      for (int J = max(0, K - WB); J < Jend; J++) {
        const size_t oK = (size_t)J*TPC + (K - J);
        wait_flag(done + oK, lane);
        double a[TILE];
        tile_load(P.tiles + oK*TILE2, a, lane);
        wait_flag(ydone + J, lane);
        const double yj = __ldcg(P.rhs + (size_t)J*TILE + lane);
#pragma unroll
        for (int k = 0; k < TILE; k++) v -= a[k]*__shfl_sync(0xffffffffu, yj, k);
      }
      if (K >= P.Kend) { P.rhs[(size_t)K*TILE + lane] = v; continue; }
      wait_flag(done + (size_t)K*TPC, lane);
      double l[TILE];
      tile_load(P.tiles + (size_t)K*TPC*TILE2, l, lane);
      double y = 0.0, mydiag = 1.0;
#pragma unroll
      for (int cc = 0; cc < TILE; cc++) if (lane == cc) mydiag = l[cc];
      const double rinv = 1.0/mydiag;
#pragma unroll
      for (int cc = 0; cc < TILE; cc++) {
        const double yc = __shfl_sync(0xffffffffu, v, cc)*__shfl_sync(0xffffffffu, rinv, cc);
        if (lane == cc) y = yc;
        if (lane > cc) v -= l[cc]*yc;
      }
      P.rhs[(size_t)K*TILE + lane] = y;
      set_flag(ydone + K, lane);
      continue;
    }
    const int I = K + dd;
    if (I >= NT) continue;
    double acc[TILE];                       // accumulator fragments while the updates run, one row per lane afterwards
    const size_t o = (size_t)K*TPC + dd;
    double* tp = P.tiles + o*TILE2;
    cfrag16_load(tp, acc, lane);
    // the spine finishes the tiles of columns <= Kend itself: it owns the last two updates of a diagonal tile and the last
    // update of a first sub-diagonal tile
    const int Jhi = min(dd == 0 ? (K <= P.Kend ? K - 3 : K - 1) : (dd == 1 ? K - 2 : K - 1), P.Kend - 1);
    accumulate_updates(P, acc, max(0, I - WB), Jhi, I, 1, K, 1, dd == 0, stage, lane);
    if (dd <= 2 || K >= P.Kend) {
      cfrag16_store(tp, acc, lane);
      set_flag(pre + o, lane);
    } else tile_finish_trsm(P, acc, K, tp, done + o, sb, sinv, lane);
  }
}

// Spike pool (pool B; only launched when a chain of the job is spiked): the spike tiles Z and the separator block FF.
// Its tasks never feed the spine, so they live in their own pool -- a 30-update spike task in front of a band task in
// the same in-order queue would stall the chain -- and it is organised for THROUGHPUT: a whole CTA (8 warps, two per
// scheduler, so one warp's shared-memory / barrier phases hide behind the other's DMMAs) takes a group task of up to 8
// output tiles that share their B operand, which is staged ONCE per step for all of them (9 tiles of L2 traffic per 8
// tile updates instead of 16):
//   spike group (K, g)       Z_r(K) = (Z_r(K) - sum_J Z_r(J) L(K,J)^T) L_KK^-T  for the rows r = 8g .. 8g+7   (B = L(K,J))
//   FF group (chunk, r2, g)  FF(r, r2) -= sum_{J in chunk} Z_r(J) Z_r2(J)^T      for 8 rows r >= r2              (B = Z_r2(J))
// Column-major task order.  Flags are checked per PHASE, not per step: done(L(K,Jhi)) implies every L(K,J), J < Jhi, and
// done(Z_r(J)) implies the earlier tiles of row r, so the bulk of a task (all steps but the last) runs as soon as the
// operands of the step before the last exist, and the row chain Z_r(K-1) -> Z_r(K) only carries one update + the TRSM.
// Operands come from pool A / the spine (which never wait on pool B) or from earlier tasks of this order: no deadlock.
// Steps are m16n8k16 updates (frag16_gemm_sub) out of a three-stage ring of swizzled stages (band_tile.cuh): the loads
// of step J+2 go into the stage step J-1 read, so the one barrier per step that publishes step J's stage also frees it.
constexpr int SPK_ROWS = 8;
constexpr int SPK_STAGES = 3;
__device__ __forceinline__ void spike_cta_worker(const CholJob& job, int cw, int ncw, double* smem) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int WB = job.WB, W1 = WB + 1;
  const int G = (WB + SPK_ROWS - 1)/SPK_ROWS;
  int NGF = 0; for (int r2 = 0; r2 < WB; r2++) NGF += (WB - r2 + SPK_ROWS - 1)/SPK_ROWS;
  const int R = G + NGF;
  double* sB = smem;                                                  // [3][TILE2] shared B operand (also L_KK for the TRSM)
  double* sA = smem + (size_t)(1 + warp)*SPK_STAGES*TILE2;            // [3][TILE2] this warp's A operand (also its layout-conversion scratch)
  double* sinv = smem + (size_t)(1 + SPK_ROWS)*SPK_STAGES*TILE2;      // [32]
  const long long per_col = (long long)job.np*R;
  const long long ntasks = (long long)job.ncols*per_col;
  for (long long t = cw; t < ntasks; t += ncw) {
    const int K = (int)(t/per_col); const int u = (int)(t - (long long)K*per_col);
    const int q = u/R; int slot = u - q*R;
    const BandProb P = job.p[q];
    if (!P.spiked || K >= P.NT) continue;
    const int TPC = P.TPC;
    const int* done = flag_done(P);
    int r, Bslot0, Bslot1, Jlo, Jhi, r2 = -1, chunk = 0;       // this warp's row; B tile of column J = slot Bslot0 - Bslot1*J
    const bool ff = slot >= G;
    if (!ff) {
      r = slot*SPK_ROWS + warp;
      Bslot0 = K; Bslot1 = 1; Jlo = max(0, K - WB); Jhi = min(K - 1, P.Kend - 1);
    } else {
      if (K >= P.Kend || !(((K + 1) % FF_CH) == 0 || K == P.Kend - 1)) continue;
      slot -= G;
      r2 = 0;
      for (;;) { const int ng = (WB - r2 + SPK_ROWS - 1)/SPK_ROWS; if (slot < ng) break; slot -= ng; r2++; }
      r = r2 + slot*SPK_ROWS + warp;
      chunk = K/FF_CH;
      Bslot0 = W1 + r2; Bslot1 = 0; Jlo = chunk*FF_CH; Jhi = K;
    }
    const bool mine = r < WB;                        // warps without a row still stage B and keep the barriers
    double* tp = !mine ? nullptr : (ff ? P.ff + ((size_t)r*WB + r2)*TILE2 : P.tiles + ((size_t)K*TPC + W1 + r)*TILE2);
    double acc[TILE];
    if (mine) {
      if (ff) wait_flag_ge(flag_ffcnt(P) + r*WB + r2, chunk, lane);
      cfrag16_load(tp, acc, lane);
    }
    if (Jhi >= Jlo) {
      // ---- operand flags.  FF: everything exists once the chunk's last column does.  Spike: the flags form monotone
      // frontiers (done(Z_r(J)) implies the row's earlier tiles, done(L(K,J)) every L(K, J' < J)), so a warp probes a few
      // columns from the far end once and only blocks, step by step, on what lies beyond the frontier it found
      int frontA = Jlo - 1, frontB = Jlo - 1;          // last column whose A (own row) / B operand is known to exist (every warp
                                                       // checks what it loads itself: no barrier between the check and the loads)
      if (ff) { wait_flag(done + (size_t)K*TPC + W1 + r2, lane); if (mine) wait_flag(done + (size_t)K*TPC + W1 + r, lane); frontA = frontB = Jhi; }
      else {
        if (lane == 0) {
          for (int back = 0; back <= Jhi - Jlo; back = back ? 2*back : 1) {
            const int J = Jhi - back;
            if (mine && frontA < Jlo && ld_acquire(done + (size_t)J*TPC + W1 + r) != 0) frontA = J;
            if (frontB < Jlo && ld_acquire(done + (size_t)J*TPC + (K - J)) != 0) frontB = J;
            if ((!mine || frontA >= Jlo) && frontB >= Jlo) break;
          }
        }
        frontA = __shfl_sync(0xffffffffu, frontA, 0); frontB = __shfl_sync(0xffffffffu, frontB, 0);
      }
      auto need = [&](int J) {                          // block until the operands of step J exist
        if (mine && J > frontA) { wait_flag(done + (size_t)J*TPC + W1 + r, lane); frontA = J; }
        if (J > frontB) { wait_flag(done + (size_t)J*TPC + (K - J), lane); frontB = J; }
      };
      auto stage_loads = [&](int J, int st) {
        need(J);
        stage16_prefetch<256>(sB + (size_t)st*TILE2, P.tiles + ((size_t)J*TPC + (Bslot0 - Bslot1*J))*TILE2, threadIdx.x);
        if (mine) stage16_prefetch<32>(sA + (size_t)st*TILE2, P.tiles + ((size_t)J*TPC + W1 + r)*TILE2, lane);
        asm volatile("cp.async.commit_group;" ::: "memory");
      };
      stage_loads(Jlo, 0);
      if (Jlo + 1 <= Jhi) stage_loads(Jlo + 1, 1);
      for (int J = Jlo, st = 0; J <= Jhi; J++, st = st == SPK_STAGES - 1 ? 0 : st + 1) {
        if (J + 1 <= Jhi) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                               // stage st is complete for every warp, and every warp is done with step J-1
        if (J + 2 <= Jhi) stage_loads(J + 2, st == 0 ? SPK_STAGES - 1 : st - 1);   // ... so step J-1's stage takes step J+2
        if (mine) {
          const double* sb = sB + (size_t)st*TILE2;
          stage16_gemm_sub(acc, ff && r == r2 ? sb : sA + (size_t)st*TILE2, sb, lane);
        }
      }
      __syncthreads();                                 // the ring is free for the next task
    }
    if (ff) {
      if (mine) { cfrag16_store(tp, acc, lane); set_flag_value(flag_ffcnt(P) + r*WB + r2, chunk + 1, lane); }
      continue;
    }
    if (K >= P.Kend) {                                 // spike tile of a separator column: its Schur complement, final
      if (mine) { cfrag16_store(tp, acc, lane); set_flag(flag_done(P) + (size_t)K*TPC + W1 + r, lane); }
      continue;
    }
    // ---- TRSM against L_KK (staged once for the CTA, column-major with stride TILE in the B buffer)
    if (warp == 0) wait_flag(done + (size_t)K*TPC, lane);
    __syncthreads();
    for (int e = threadIdx.x; e < TILE2; e += 256) sB[e] = __ldcg(P.tiles + (size_t)K*TPC*TILE2 + e);
    __syncthreads();
    if (threadIdx.x < TILE) sinv[threadIdx.x] = 1.0/sB[threadIdx.x*TILE + threadIdx.x];
    __syncthreads();
    if (mine) {
      __syncwarp();
      cfrag16_store(sA, acc, lane);                    // accumulator fragments -> one row per lane
      __syncwarp();
#pragma unroll
      for (int cc = 0; cc < TILE; cc++) acc[cc] = sA[cc*TILE + lane];
      tile_trsm(acc, sB, sinv);
      tile_store(tp, acc, lane);
      set_flag(flag_done(P) + (size_t)K*TPC + W1 + r, lane);
    }
    __syncthreads();                                   // sB / sinv are reused by the next task
  }
}

// =====================================================================================================================
// Spine.  One CTA of 8 warps per band problem; the compute warps work out of shared memory / registers only and
// never touch global memory, fences or flags -- three I/O warps do that one column ahead / behind:
// (warp w issues on scheduler w % 4: each A warp shares its scheduler with a mostly sleeping I/O warp)
//   A pair (warps 0, 1)  alternate per column between  potrf(K,K)  and  accumulating the next diagonal tile
//                        D(K+1) = T(K+1,K+1) - X2(K-1) X2(K-1)^T - X1(K) X1(K)^T  (rank-8 updates as X1 panels appear)
//   B pair (warps 2, 3)  alternate between the TRSM of X1(K) = L(K+1,K), one panel behind the potrf, and accumulating
//                        Xn = T(K+2,K+1) - X2(K) X1(K)^T
//   C      (warp 6)      TRSM of X2(K) = L(K+2,K) and its store; runs on its own clock (its input arrives late from the workers)
//   IO0    (warp 7)      L(K,K), X1(K) -> global, done flags
//   IO1    (warp 5)      T(K+1,K+1), T(K+2,K+1) (worker-updated) -> shared memory, one column ahead
// Hand-offs are monotone event counters in shared memory (value c+1 = "done for column c").
constexpr int SP_WARPS = 8;
constexpr int PSTR = 10, PANSZ = TILE*PSTR;     // potrf panel [row][8], row stride 10 doubles: conflict-free LDS.128 per row
enum { EV_PAN = 0, EV_X1P = 4, EV_X2 = 8, EV_DIN = 9, EV_XNIN = 10, EV_ST_L = 11, EV_ST_X1 = 12, EV_ST_X2 = 13, EV_TK_D = 14, EV_TK_XN = 15, EV_N = 16 };

__device__ __forceinline__ void ev_signal(volatile int* ev, int i, int v, int lane) {
  __syncwarp();
  if (lane == 0) asm volatile("st.release.cta.shared.s32 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared((const void*)(ev + i))), "r"(v) : "memory");
}
__device__ __forceinline__ void ev_wait(volatile int* ev, int i, int v, int lane) {
  if (lane == 0) {
    const unsigned a = (unsigned)__cvta_generic_to_shared((const void*)(ev + i));
    int cur, spins = 0;
    for (;;) {
      asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(cur) : "r"(a) : "memory");
      if (cur >= v) break;
      if (++spins > 16) __nanosleep(20);
    }
  }
  __syncwarp();
}

// The spine's code must stay small: a warp that runs thousands of straight-line instructions once per column is bound by
// instruction fetch, not by the arithmetic (tools/ubench/potrf_bench.cu: 5.8k cycles per tile alone, 14-17k inside a
// 25k-instruction kernel).  So the panel loops below are ROLLED; the register tile keeps static indices through
// block-of-8 switches on the (warp-uniform) panel number.
#define SPINE_BLOCK_SWITCH(p, BODY) \
  do { if ((p) == 0) { constexpr int B8 = 0; BODY } else if ((p) == 1) { constexpr int B8 = 8; BODY } \
       else if ((p) == 2) { constexpr int B8 = 16; BODY } else { constexpr int B8 = 24; BODY } } while (0)

// Cholesky of a 32x32 tile held one row per lane, in 4 panels of 8 columns.  The 8x8 diagonal block of a panel is read
// back from shared memory by EVERY lane and factored redundantly in registers, each lane solving its own row against it
// on the way (no shuffles); the serial chain per column is rsqrt -> scale -> one FMA.  Finished panels are published:
// sPan[p][row*PSTR + j] = L[row][8p + j], sIv[k] = 1 / L[k][k], event EV_PAN + p.
__device__ __forceinline__ bool spine_potrf(double (&row)[TILE], int lane, double* sPan, double* sIv, volatile int* ev, int cval) {
  bool ok = true;
#pragma unroll 1
  for (int p = 0; p < 4; p++) {
    double* sP = sPan + p*PANSZ;
    double x[8];
    SPINE_BLOCK_SWITCH(p, {
#pragma unroll
      for (int j = 0; j < 8; j++) x[j] = row[B8 + j];
    });
#pragma unroll
    for (int j = 0; j < 8; j += 2) *reinterpret_cast<double2*>(sP + lane*PSTR + j) = make_double2(x[j], x[j + 1]);
    __syncwarp();
    double G[36];                                   // packed lower triangle, G[i(i+1)/2 + j] = block[i][j]
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j <= i; j++) G[i*(i + 1)/2 + j] = sP[(8*p + i)*PSTR + j];
    __syncwarp();
    double myinv = 0.0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const double d = G[k*(k + 1)/2 + k];
      if (!(d > 0.0)) ok = false;
      const double inv = rsqrt(d);
      if ((lane & 7) == k) myinv = inv;      // published after the loop: a store inside it makes ptxas clone the rsqrt
      x[k] *= inv;
#pragma unroll
      for (int i = k + 1; i < 8; i++) G[i*(i + 1)/2 + k] *= inv;
#pragma unroll
      for (int j = k + 1; j < 8; j++) {
        const double ljk = G[j*(j + 1)/2 + k];
        x[j] -= x[k]*ljk;
#pragma unroll
        for (int i = j; i < 8; i++) G[i*(i + 1)/2 + j] -= G[i*(i + 1)/2 + k]*ljk;
      }
    }
    if (lane < 8) sIv[8*p + lane] = myinv;
#pragma unroll
    for (int j = 0; j < 8; j += 2) *reinterpret_cast<double2*>(sP + lane*PSTR + j) = make_double2(x[j], x[j + 1]);
    ev_signal(ev, EV_PAN + p, cval, lane);
    // rank-8 update of the columns behind the panel (blocks of 8 columns, static register indices)
#pragma unroll
    for (int blk = 1; blk < 4; blk++) {
      if (blk > p) {
#pragma unroll
        for (int cc = 0; cc < 8; cc++) {
          const int c = 8*blk + cc;
          double acc = row[c];
#pragma unroll
          for (int j = 0; j < 8; j += 2) {
            const double2 b = *reinterpret_cast<const double2*>(sP + c*PSTR + j);
            acc -= x[j]*b.x; acc -= x[j + 1]*b.y;
          }
          row[c] = acc;
        }
      }
    }
  }
  return ok;
}
// x(row = lane) <- x * L^-T from the published panels; every finished panel of x is staged k-major (sX[k*TS + row]) and
// announced on ev_out + p (ev_out < 0: no per-panel events)
__device__ __forceinline__ void spine_trsm(double (&x)[TILE], int lane, const double* sPan, const double* sIv, volatile int* ev, int cval,
                                           double* sX, int ev_out) {
#pragma unroll 1
  for (int p = 0; p < 4; p++) {
    const double* sP = sPan + p*PANSZ;
    ev_wait(ev, EV_PAN + p, cval, lane);
    double xs[8];
    SPINE_BLOCK_SWITCH(p, {
#pragma unroll
      for (int j = 0; j < 8; j++) xs[j] = x[B8 + j];
    });
#pragma unroll
    for (int kk = 0; kk < 8; kk++) {
      const double l = xs[kk]*sIv[8*p + kk];
      xs[kk] = l;
#pragma unroll
      for (int j = kk + 1; j < 8; j++) xs[j] -= l*sP[(8*p + j)*PSTR + kk];
    }
#pragma unroll
    for (int j = 0; j < 8; j++) sX[(8*p + j)*TS + lane] = xs[j];
    if (ev_out >= 0) ev_signal(ev, ev_out + p, cval, lane);
#pragma unroll
    for (int blk = 1; blk < 4; blk++) {
      if (blk > p) {
#pragma unroll
        for (int cc = 0; cc < 8; cc++) {
          const int c = 8*blk + cc;
          double acc = x[c];
#pragma unroll
          for (int j = 0; j < 8; j += 2) {
            const double2 b = *reinterpret_cast<const double2*>(sP + c*PSTR + j);
            acc -= xs[j]*b.x; acc -= xs[j + 1]*b.y;
          }
          x[c] = acc;
        }
      }
    }
  }
}
// Rank-32 update of an accumulator tile held as MMA fragments (see frag8_gemm_sub): c -= XA XB^T, XA / XB k-major tiles in
// shared memory with column stride TS, applied in four rank-8 steps (two k-steps of the m8n8k4 MMA each) as the panels
// of XB appear (ev_base >= 0: wait for event ev_base + p first).  16 LDS.64 + 32 DMMA per step: next to nothing on the
// shared-memory pipe, which the FMA formulation (one LDS.128 per two FMAs) saturates when several spine warps run it.
// This stays on m8n8k4 while the worker pools use m16n8k16: a k = 16 step needs two TRSM panels of XB, so it would wait
// for the second one, and the step after the last panel -- the one on the chain's critical path -- would be twice as long.
__device__ __forceinline__ void spine_rank32(double (&c)[TILE], const double* xa, const double* xb, bool same,
                                             volatile int* ev, int ev_base, int cval, int lane) {
  const int off = (lane & 3)*TS + (lane >> 2);
#pragma unroll 1
  for (int p = 0; p < 4; p++) {
    if (ev_base >= 0) ev_wait(ev, ev_base + p, cval, lane);
#pragma unroll
    for (int kk = 0; kk < 2; kk++) {
      const int kb = 2*p + kk;
      double fa[4], fb[4];
#pragma unroll
      for (int b = 0; b < 4; b++) fb[b] = xb[off + 4*kb*TS + 8*b];
#pragma unroll
      for (int b = 0; b < 4; b++) fa[b] = same ? -fb[b] : -xa[off + 4*kb*TS + 8*b];
#pragma unroll
      for (int rb = 0; rb < 4; rb++)
#pragma unroll
        for (int cb = 0; cb < 4; cb++) dmma8(c[(rb*4 + cb)*2], c[(rb*4 + cb)*2 + 1], fa[rb], fb[cb]);
    }
  }
}
// m8n8k4 accumulator fragments <-> shared-memory tile with column stride S
template <int S>
__device__ __forceinline__ void cfrag8_load_s(const double* t, double (&c)[TILE], int lane) {
  const double* p = t + 2*(lane & 3)*S + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 4; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++) { c[(rb*4 + cb)*2] = p[8*cb*S + 8*rb]; c[(rb*4 + cb)*2 + 1] = p[(8*cb + 1)*S + 8*rb]; }
}
template <int S>
__device__ __forceinline__ void cfrag8_store_s(double* t, const double (&c)[TILE], int lane) {
  double* p = t + 2*(lane & 3)*S + (lane >> 2);
#pragma unroll
  for (int rb = 0; rb < 4; rb++)
#pragma unroll
    for (int cb = 0; cb < 4; cb++) { p[8*cb*S + 8*rb] = c[(rb*4 + cb)*2]; p[(8*cb + 1)*S + 8*rb] = c[(rb*4 + cb)*2 + 1]; }
}
// accumulator fragments -> one row per lane through a private shared-memory tile
__device__ __forceinline__ void cfrag_to_rows(double (&r)[TILE], double* scr, int lane) {
  __syncwarp();
  cfrag8_store_s<TILE>(scr, r, lane);
  __syncwarp();
#pragma unroll
  for (int col = 0; col < TILE; col++) r[col] = scr[col*TILE + lane];
  __syncwarp();
}

__global__ void __launch_bounds__(SP_WARPS*32)
band_cholesky_dataflow_kernel_v3(CholJob job, int* __restrict__ fail) {
  extern __shared__ __align__(16) double chol_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if ((int)blockIdx.x >= job.np) {
    const int w = (int)blockIdx.x - job.np;
    if (job.profile && threadIdx.x == 0) atomicMin(&g_prof[34], gtimer());
    if (w >= job.band_ctas) {
      spike_cta_worker(job, w - job.band_ctas, (int)gridDim.x - job.np - job.band_ctas, chol_smem);
      if (job.profile && threadIdx.x == 0) atomicMax(&g_prof[33], gtimer());
      return;
    }
    if (warp >= 4) return;       // four band worker warps per CTA (one per scheduler): [warp][2 stages][2 tiles][TILE2] | [TILE2] | [TILE]
    double* base = chol_smem + (size_t)warp*(5*TILE2 + TILE);
    band_worker(job, w*4 + warp, job.band_ctas*4, base + 4*TILE2, base + 5*TILE2, base, lane);
    if (job.profile && lane == 0) atomicMax(&g_prof[32], gtimer());
    return;
  }
  const BandProb P = job.p[blockIdx.x];
  const int WB = job.WB, TPC = P.TPC, NT = P.NT, Kend = P.Kend;
  if (Kend <= 0) return;
  double* sPan = chol_smem;                   // [2][4][PANSZ]
  double* sIv = sPan + 2*4*PANSZ;             // [2][32]
  double* sX1 = sIv + 2*TILE;                 // [2][TSZ]  k-major, column stride TS
  double* sX2 = sX1 + 2*TSZ;                  // [2][TSZ]
  double* sDin = sX2 + 2*TSZ;                 // [2][TSZ]  column-major, column stride TS
  double* sXnin = sDin + 2*TSZ;               // [2][TSZ]
  double* sScr = sXnin + 2*TSZ;               // [4][TILE2] layout-conversion scratch of the A / B warps
  volatile int* ev = reinterpret_cast<volatile int*>(sScr + 4*TILE2);
  if (threadIdx.x < EV_N) ev[threadIdx.x] = 0;
  __syncthreads();
  int* done = flag_done(P); int* pre = flag_pre(P);
  const bool x2 = WB >= 2;
  double r[TILE];
  if (warp == 0 || warp == 1) {
    // ---------------------------------------------------------------- A pair: potrf / next diagonal tile
    const int i = warp;
    for (int c = -1; c < Kend; c++) {
      if (c >= 0 && (c & 1) == i) {
        ev_wait(ev, EV_ST_L, c - 1, lane);
        if (!spine_potrf(r, lane, sPan + (c & 1)*4*PANSZ, sIv + (c & 1)*TILE, ev, c + 1) && lane == 0) atomicOr(fail, 2);
      } else if (((c + 1) & 1) == i && c + 1 < NT) {
        ev_wait(ev, EV_DIN, c + 2, lane);
        cfrag8_load_s<TS>(sDin + ((c + 1) & 1)*TSZ, r, lane);      // r: accumulator fragments until cfrag_to_rows
        ev_signal(ev, EV_TK_D, c + 2, lane);
        // term 0: X2(c-1) = L(c+1, c-1), staged two columns ago and still in its buffer; term 1: X1(c), panel by panel
#pragma unroll 1
        for (int t = 0; t < 2; t++) {
          if (t == 0 ? !(x2 && c - 1 >= 0) : !(c >= 0)) continue;
          if (t == 0) ev_wait(ev, EV_X2, c, lane);
          const double* xa = t == 0 ? sX2 + ((c - 1) & 1)*TSZ : sX1 + (c & 1)*TSZ;
          spine_rank32(r, xa, xa, true, ev, t == 0 ? -1 : EV_X1P, c + 1, lane);
        }
        cfrag_to_rows(r, sScr + i*TILE2, lane);
        if (c + 1 == Kend) tile_store(P.tiles + (size_t)Kend*TPC*TILE2, r, lane);   // not factored here: hand it back
      }
    }
  } else if (warp == 2 || warp == 3) {
    // ---------------------------------------------------------------- B pair: X1 TRSM / next X1 input
    const int i = warp - 2;
    for (int c = -1; c < Kend; c++) {
      if (c >= 0 && (c & 1) == i) {
        if (c + 1 < NT) {
          ev_wait(ev, EV_ST_X1, c - 1, lane);
          spine_trsm(r, lane, sPan + (c & 1)*4*PANSZ, sIv + (c & 1)*TILE, ev, c + 1, sX1 + (c & 1)*TSZ, EV_X1P);
        }
      } else if (((c + 1) & 1) == i && c + 2 < NT) {
        ev_wait(ev, EV_XNIN, c + 2, lane);
        cfrag8_load_s<TS>(sXnin + ((c + 1) & 1)*TSZ, r, lane);
        ev_signal(ev, EV_TK_XN, c + 2, lane);
        if (x2 && c >= 0) {
          ev_wait(ev, EV_X2, c + 1, lane);
          spine_rank32(r, sX2 + (c & 1)*TSZ, sX1 + (c & 1)*TSZ, false, ev, EV_X1P, c + 1, lane);
        }
        cfrag_to_rows(r, sScr + (2 + i)*TILE2, lane);
        if (c + 1 == Kend) tile_store(P.tiles + ((size_t)Kend*TPC + 1)*TILE2, r, lane);
      }
    }
  } else if (warp == 6) {
    // ---------------------------------------------------------------- C: X2 TRSM
    if (x2) for (int c = 0; c < Kend; c++) if (c + 2 < NT) {
      wait_flag(pre + (size_t)c*TPC + 2, lane);
      tile_load(P.tiles + ((size_t)c*TPC + 2)*TILE2, r, lane);
      spine_trsm(r, lane, sPan + (c & 1)*4*PANSZ, sIv + (c & 1)*TILE, ev, c + 1, sX2 + (c & 1)*TSZ, -1);
      ev_signal(ev, EV_X2, c + 1, lane);
      // publish X2(c) from its staged copy (this warp runs on its own clock: the store is off the spine's critical path)
      {
        const double* sx = sX2 + (c & 1)*TSZ;
        double* t = P.tiles + ((size_t)c*TPC + 2)*TILE2;
#pragma unroll
        for (int col = 0; col < TILE; col++) t[col*TILE + lane] = sx[col*TS + lane];
      }
      set_flag(done + (size_t)c*TPC + 2, lane);
    }
  } else if (warp == 7) {
    // ---------------------------------------------------------------- IO0: L(c,c), X1(c) -> global
    for (int c = 0; c < Kend; c++) {
      ev_wait(ev, EV_PAN + 3, c + 1, lane);
      const double* pan = sPan + (c & 1)*4*PANSZ;
      double* t = P.tiles + (size_t)c*TPC*TILE2;
#pragma unroll
      for (int p = 0; p < 4; p++)
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          const double2 v = *reinterpret_cast<const double2*>(pan + p*PANSZ + lane*PSTR + j);
          t[(8*p + j)*TILE + lane] = v.x; t[(8*p + j + 1)*TILE + lane] = v.y;
        }
      set_flag(done + (size_t)c*TPC, lane);
      ev_signal(ev, EV_ST_L, c + 1, lane);
      if (c + 1 < NT) {
        ev_wait(ev, EV_X1P + 3, c + 1, lane);
        const double* sx = sX1 + (c & 1)*TSZ;
#pragma unroll
        for (int col = 0; col < TILE; col++) t[TILE2 + col*TILE + lane] = sx[col*TS + lane];
        set_flag(done + (size_t)c*TPC + 1, lane);
        ev_signal(ev, EV_ST_X1, c + 1, lane);
      }
    }
    if (job.profile && lane == 0 && blockIdx.x < 32) g_prof[blockIdx.x] = gtimer();
  } else if (warp == 5) {
    // ---------------------------------------------------------------- IO1: inputs of column c+1 -> shared memory
    for (int c = -1; c < Kend; c++) if (c + 1 < NT) {
      const double* t = P.tiles + (size_t)(c + 1)*TPC*TILE2;
      ev_wait(ev, EV_TK_D, c, lane);
      wait_flag(pre + (size_t)(c + 1)*TPC, lane);
      tile_load(t, r, lane);
      double* sd = sDin + ((c + 1) & 1)*TSZ;
#pragma unroll
      for (int col = 0; col < TILE; col++) sd[col*TS + lane] = r[col];
      ev_signal(ev, EV_DIN, c + 2, lane);
      if (c + 2 < NT) {
        ev_wait(ev, EV_TK_XN, c, lane);
        wait_flag(pre + (size_t)(c + 1)*TPC + 1, lane);
        tile_load(t + TILE2, r, lane);
        double* sx = sXnin + ((c + 1) & 1)*TSZ;
#pragma unroll
        for (int col = 0; col < TILE; col++) sx[col*TS + lane] = r[col];
        ev_signal(ev, EV_XNIN, c + 2, lane);
      }
    }
  }
  // warp 4 has no role: it leaves scheduler 0 to the A warp that issues there
}

// explicit inverse of every diagonal tile: Linv[K] = L_KK^-1 (lower triangular), one warp per tile
__global__ void __launch_bounds__(128) diag_inverse_kernel(const BandProb* __restrict__ probs) {
  __shared__ double sL[4][TILE2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const BandProb P = probs[blockIdx.y];
  const int K = blockIdx.x*4 + warp;
  if (K >= P.Kend) return;
  const double* t = P.tiles + (size_t)K*P.TPC*TILE2;
  double* linv = P.linv;
  double* s = sL[warp];
#pragma unroll
  for (int c = 0; c < TILE; c++) s[c*TILE + lane] = t[c*TILE + lane];
  __syncwarp();
  // lane j solves L x = e_j  -> column j of L^-1
  double x[TILE];
#pragma unroll
  for (int r = 0; r < TILE; r++) {
    double v = (r == lane) ? 1.0 : 0.0;
#pragma unroll
    for (int k = 0; k < r; k++) v -= s[k*TILE + r]*x[k];      // L[r][k]
    x[r] = v/s[r*TILE + r];
  }
  double* o = linv + (size_t)K*TILE2;
#pragma unroll
  for (int r = 0; r < TILE; r++) o[lane*TILE + r] = (r >= lane) ? x[r] : 0.0;   // element (r, j=lane) at j*32 + r
}

// backward sweep  x_J = Linv_JJ^T (y_J - sum_{I>J} L_IJ^T x_I) for J = Jtop-1 ... Jbot; rhs overwritten.
// One thread-block CLUSTER of 8 CTAs (8 SMs) per band problem: the off-diagonal tiles of a column are spread over
// 8 x 4 warps so the 240 KB a column reads come through eight SMs' load paths; per-CTA partial sums are all-gathered
// through distributed shared memory and every CTA finishes x_J itself (one cluster barrier per column).
// Columns >= Jtop are already solved (the middle separator of the two-directional scheme): their x primes the ring.
struct BackProb { const double* tiles; double* rhs; const double* linv; int NT, Jtop, Jbot; };
struct BackJob { const BandProb* p; int WB; };
constexpr int BW_CL = 8, BW_TW = 4;      // cluster size, tile warps per CTA
constexpr int BW_PS = 34;                // padded column stride of warp 0's shared-memory tiles (conflict-free LDS.128 per column)
// dot product of 32 register values with a 32-vector in shared memory (broadcast reads)
__device__ __forceinline__ double dot32(const double (&a)[TILE], const double* x) {
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
  for (int r = 0; r < TILE; r += 4) {
    const double2 u = *reinterpret_cast<const double2*>(x + r), w = *reinterpret_cast<const double2*>(x + r + 2);
    s0 += a[r]*u.x; s1 += a[r + 1]*u.y; s2 += a[r + 2]*w.x; s3 += a[r + 3]*w.y;
  }
  return (s0 + s1) + (s2 + s3);
}
// Backward sweep x_J = L_JJ^-T (y_J - sum_{I>J} L_IJ^T x_I), TWO columns per cluster barrier: the off-diagonal terms of
// columns J and J-1 that involve x_I, I > J, are independent of each other (and use the same x_I: tile (I,J) and tile
// (I,J-1) go to the same warp), only L(J,J-1)^T x_J has to wait for x_J and is done by warp 0 between the two solves.
// Every tile GEMV^T is COLUMN-per-lane: lane c holds column c of the tile (32 contiguous doubles) and reads x as
// broadcast LDS.128 -- 32 FMAs and no shuffles (the row-per-lane form needs a 31-shuffle transpose-sum per tile).
__global__ void __cluster_dims__(BW_CL, 1, 1) __launch_bounds__((BW_TW + 1)*32)
band_backward_cluster_kernel(BackJob job) {
  extern __shared__ __align__(16) double sm[];
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const BandProb Q = job.p[blockIdx.x/BW_CL];
  const BackProb P = { Q.tiles, Q.rhs, Q.linv, Q.NT, Q.Kend, 0 };     // columns >= Kend are solved already: their x primes the ring
  const int NT = P.NT, WB = job.WB, W1 = Q.TPC /* column stride in tiles */, ring = WB + 2;
  double* xs = sm;                                   // [ring][32] solved blocks (replicated in every CTA)
  double* lpart = sm + (size_t)ring*TILE;            // [2][BW_TW][32] partial sums of this CTA's tile warps, per column
  double* cpart = lpart + 2*BW_TW*TILE;              // [2][2][BW_CL][32] all-gathered per-CTA partials (pair parity, column)
  double* sv = cpart + 4*BW_CL*TILE;                 // [32] warp 0: right-hand side to broadcast
  double* sW0 = sv + TILE;                           // [2 stages][3][32*BW_PS] warp 0: Linv(J), Linv(J-1), L(J,J-1) of a pair, fetched with
                                                     // cp.async one pair ahead
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int I = P.Jtop + warp; I < min(NT, P.Jtop + WB); I += BW_TW + 1) xs[(size_t)(I % ring)*TILE + lane] = P.rhs[(size_t)I*TILE + lane];
  __syncthreads();
  const int myq = rank*BW_TW + (warp - 1);           // this warp's tile of column J; of column J-1 it takes tile myq + 1
  double tA[TILE], tB[TILE];                          // column `lane` of the prefetched tiles (warp 0: tA = Linv(J))
  auto load_col = [&](const double* tile, double (&t)[TILE]) {
    const double2* p = reinterpret_cast<const double2*>(tile + lane*TILE);
#pragma unroll
    for (int r = 0; r < TILE/2; r++) { const double2 u = p[r]; t[2*r] = u.x; t[2*r + 1] = u.y; }
  };
  // software prefetch: the tiles of the next pair are loaded while this pair is processed
  auto prefetchA = [&](int J) { if (J >= P.Jbot && myq < min(WB, NT - 1 - J)) load_col(P.tiles + (size_t)J*W1*TILE2 + (size_t)(myq + 1)*TILE2, tA); };
  auto prefetchB = [&](int J) { if (J - 1 >= P.Jbot && myq + 1 < min(WB, NT - J)) load_col(P.tiles + (size_t)(J - 1)*W1*TILE2 + (size_t)(myq + 2)*TILE2, tB); };
  auto fetch_w0 = [&](int J, int stage) {              // warp 0: the three tiles of pair (J, J-1) -> shared memory stage
    if (J >= P.Jbot) {
      double* dst = sW0 + (size_t)stage*3*TILE*BW_PS;
      const double* l0 = P.linv + (size_t)J*TILE2;
      const double* l1 = P.linv + (size_t)(J - 1)*TILE2;
      const double* tp = P.tiles + (size_t)(J - 1)*W1*TILE2 + TILE2;
      const bool two = J - 1 >= P.Jbot;
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const int ch = lane + 32*i, c = ch >> 4, part = ch & 15;
        const unsigned d = (unsigned)__cvta_generic_to_shared(dst + c*BW_PS + 2*part);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(d), "l"(l0 + 2*ch) : "memory");
        if (two) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(d + (unsigned)(TILE*BW_PS*8)), "l"(l1 + 2*ch) : "memory");
        if (two && WB >= 1) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(d + (unsigned)(2*TILE*BW_PS*8)), "l"(tp + 2*ch) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");   // always: keeps the group count in step with the pair count
  };
  // the factor is far larger than L2 and was written long ago: pull the tiles of the pair after next into L2 early, so
  // that the register / cp.async prefetches above see L2 latency instead of HBM latency
  auto l2_line = [&](const double* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); };
  auto warm = [&](int J) {
    if (J < P.Jbot) return;
    if (warp >= 1) {
      if (myq < min(WB, NT - 1 - J)) { const double* t = P.tiles + (size_t)J*W1*TILE2 + (size_t)(myq + 1)*TILE2; l2_line(t + lane*16); l2_line(t + 512 + lane*16); }
      if (J - 1 >= P.Jbot && myq + 1 < min(WB, NT - J)) { const double* t = P.tiles + (size_t)(J - 1)*W1*TILE2 + (size_t)(myq + 2)*TILE2; l2_line(t + lane*16); l2_line(t + 512 + lane*16); }
    } else {
      const double* t = P.linv + (size_t)J*TILE2; l2_line(t + lane*16); l2_line(t + 512 + lane*16);
      if (J - 1 >= P.Jbot) {
        const double* u = P.linv + (size_t)(J - 1)*TILE2; l2_line(u + lane*16); l2_line(u + 512 + lane*16);
        const double* w = P.tiles + (size_t)(J - 1)*W1*TILE2 + TILE2; l2_line(w + lane*16); l2_line(w + 512 + lane*16);
      }
    }
  };
  if (warp >= 1) { prefetchA(P.Jtop - 1); prefetchB(P.Jtop - 1); } else fetch_w0(P.Jtop - 1, 0);
  warm(P.Jtop - 3); warm(P.Jtop - 5); warm(P.Jtop - 7);
  int par = 0;
  for (int J = P.Jtop - 1; J >= P.Jbot; J -= 2, par ^= 1) {
    const bool hasB = J - 1 >= P.Jbot;
    const int nbA = min(WB, NT - 1 - J), nbB = min(WB, NT - J);       // tiles below the diagonal in columns J, J-1
    warm(J - 8);
    if (warp >= 1) {
      double sA = 0.0, sB = 0.0;
      if (myq < nbA) {
        const double* xv = xs + (size_t)((J + 1 + myq) % ring)*TILE;
        sA += dot32(tA, xv);                                          // lane c: sum_r L[r][c] x[r]
        if (hasB && myq + 1 < nbB) sB += dot32(tB, xv);
      }
      for (int q = myq + BW_CL*BW_TW; q < nbA; q += BW_CL*BW_TW) {    // only when WB > 32 (tA / tB double as scratch)
        const double* xv = xs + (size_t)((J + 1 + q) % ring)*TILE;
        load_col(P.tiles + (size_t)J*W1*TILE2 + (size_t)(q + 1)*TILE2, tA);
        sA += dot32(tA, xv);
        if (hasB && q + 1 < nbB) { load_col(P.tiles + (size_t)(J - 1)*W1*TILE2 + (size_t)(q + 2)*TILE2, tB); sB += dot32(tB, xv); }
      }
      prefetchA(J - 2);                                                // in flight across the cluster barrier
      prefetchB(J - 2);
      lpart[(warp - 1)*TILE + lane] = sA;
      lpart[(BW_TW + warp - 1)*TILE + lane] = sB;
    }
    __syncthreads();
    if (warp == 0) {
      double sA = 0.0, sB = 0.0;
#pragma unroll
      for (int w = 0; w < BW_TW; w++) { sA += lpart[w*TILE + lane]; sB += lpart[(BW_TW + w)*TILE + lane]; }
#pragma unroll
      for (int r = 0; r < BW_CL; r++) {
        double* cp = cl.map_shared_rank(cpart, r) + (size_t)par*2*BW_CL*TILE;
        cp[rank*TILE + lane] = sA; cp[(BW_CL + rank)*TILE + lane] = sB;
      }
      fetch_w0(J - 2, par ^ 1);                                        // next pair's tiles
      tA[0] = P.rhs[(size_t)J*TILE + lane];                            // this pair's right-hand sides: latency under the barrier
      tA[1] = hasB ? P.rhs[(size_t)(J - 1)*TILE + lane] : 0.0;
    }
    cl.sync();
    if (warp == 0) {
      const double* cp = cpart + (size_t)par*2*BW_CL*TILE;
      const double* st = sW0 + (size_t)par*3*TILE*BW_PS;
      double v = tA[0], v2 = tA[1];
#pragma unroll
      for (int r = 0; r < BW_CL; r++) { v -= cp[r*TILE + lane]; v2 -= cp[(BW_CL + r)*TILE + lane]; }
      asm volatile("cp.async.wait_group 1;" ::: "memory");           // everything but the group issued above has landed
      sv[lane] = v;
      __syncwarp();
      auto col = [&](const double* tile) {
        const double2* lc = reinterpret_cast<const double2*>(tile + lane*BW_PS);
#pragma unroll
        for (int r = 0; r < TILE/2; r++) { const double2 u = lc[r]; tB[2*r] = u.x; tB[2*r + 1] = u.y; }
      };
      col(st);
      const double x = dot32(tB, sv);                                 // lane c: sum_r Linv[r][c] v[r]
      double* xj = xs + (size_t)(J % ring)*TILE;
      xj[lane] = x;
      if (rank == 0) P.rhs[(size_t)J*TILE + lane] = x;
      if (hasB) {
        __syncwarp();
        if (WB >= 1) { col(st + 2*TILE*BW_PS); v2 -= dot32(tB, xj); }   // (L(J,J-1)^T x_J)[lane]
        __syncwarp();
        sv[lane] = v2;
        __syncwarp();
        col(st + TILE*BW_PS);
        const double x2 = dot32(tB, sv);
        xs[(size_t)((J - 1) % ring)*TILE + lane] = x2;
        if (rank == 0) P.rhs[(size_t)(J - 1)*TILE + lane] = x2;
      }
    }
    __syncthreads();
  }
}

// =====================================================================================================================
// Separator plumbing (element-wise kernels; tools/cell_proto.py stages 2-4)

// g_Q -= sum_{J < Kend} Z(J) y_J of every spiked chain: partial sums per chunk of SF_CH columns, then a fixed-order sum
constexpr int SF_CH = 8;
__global__ void __launch_bounds__(256) spike_forward_partial_kernel(const BandProb* __restrict__ probs, int WB, double* __restrict__ scratch, int maxchunks) {
  const BandProb P = probs[blockIdx.y];
  const int J0 = blockIdx.x*SF_CH;
  if (!P.spiked || J0 >= P.Kend) return;
  __shared__ double sy[SF_CH][TILE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nJ = min(SF_CH, P.Kend - J0);
  if (warp < nJ) sy[warp][lane] = P.rhs[(size_t)(J0 + warp)*TILE + lane];
  __syncthreads();
  for (int r = warp; r < WB; r += 8) {
    double s = 0.0;
    for (int jj = 0; jj < nJ; jj++) {
      const double* z = P.tiles + ((size_t)(J0 + jj)*P.TPC + WB + 1 + r)*TILE2;
#pragma unroll 8
      for (int c = 0; c < TILE; c++) s += z[c*TILE + lane]*sy[jj][c];
    }
    scratch[(((size_t)blockIdx.y*maxchunks + blockIdx.x)*WB + r)*TILE + lane] = s;
  }
}
__global__ void spike_forward_reduce_kernel(const BandProb* __restrict__ probs, int WB, const double* __restrict__ scratch, int maxchunks) {
  const BandProb P = probs[blockIdx.y];
  if (!P.spiked) return;
  const int e = blockIdx.x*blockDim.x + threadIdx.x;       // element of gf: r*32 + lane
  if (e >= WB*TILE) return;
  const int nchunk = (P.Kend + SF_CH - 1)/SF_CH;
  double s = 0.0;
  for (int k = 0; k < nchunk; k++) s += scratch[((size_t)blockIdx.y*maxchunks + k)*WB*TILE + e];
  P.gf[e] -= s;
}
// y_J -= sum_r Z_r(J)^T x_Q[r] for every factored column J of every spiked chain (x_Q in the chain's order in P.gf)
__global__ void __launch_bounds__(256) spike_backward_kernel(const BandProb* __restrict__ probs, int WB) {
  extern __shared__ double sx[];        // [WB][32]
  const BandProb P = probs[blockIdx.y];
  if (!P.spiked || (int)blockIdx.x*8 >= P.Kend) return;
  for (int i = threadIdx.x; i < WB*TILE; i += blockDim.x) sx[i] = P.gf[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int J = blockIdx.x*8 + warp;
  if (J >= P.Kend) return;
  double s0 = 0.0, s1 = 0.0;
  for (int r = 0; r < WB; r++) {
    const double2* z = reinterpret_cast<const double2*>(P.tiles + ((size_t)J*P.TPC + WB + 1 + r)*TILE2 + lane*TILE);   // column `lane`
    const double* x = sx + r*TILE;
#pragma unroll
    for (int k = 0; k < TILE/2; k++) { const double2 u = z[k]; s0 += u.x*x[2*k]; s1 += u.y*x[2*k + 1]; }
  }
  P.rhs[(size_t)J*TILE + lane] -= s0 + s1;
}

struct CellRefs { const BandProb* chains; const BandProb* cs; const BandProb* gq; const CellGeom* cells; const int* local_cells; int WB; };

// entry (i >= j) of the cell separator system [M | Qa | Qb] of cell c from the chains' storage after their factorisation
__device__ __forceinline__ double cs_value(const BandProb& A, const BandProb& Bc, int WB, bool has_qa, int i, int j) {
  const int w = WB*TILE, zi = i/w, zj = j/w, ii = i - zi*w, jj = j - zj*w;
  const bool iQa = has_qa && zi == 1, jQa = has_qa && zj == 1;
  if (zj == 0) {
    if (zi == 0) {
      const int li = w - 1 - jj, lj = w - 1 - ii;
      return A.tiles[tile_elem(A.TPC, A.Kend + (jj >> 5), (ii >> 5) - (jj >> 5), ii & 31, jj & 31)] +
             Bc.tiles[tile_elem(Bc.TPC, Bc.Kend + (lj >> 5), (li >> 5) - (lj >> 5), li & 31, lj & 31)];
    }
    if (iQa) return A.tiles[tile_elem(A.TPC, A.Kend + (jj >> 5), WB + 1 + (ii >> 5), ii & 31, jj & 31)];
    const int s = w - 1 - ii, lc = w - 1 - jj;
    return Bc.tiles[tile_elem(Bc.TPC, Bc.Kend + (lc >> 5), WB + 1 + (s >> 5), s & 31, lc & 31)];
  }
  if (jQa) return iQa ? A.ff[((size_t)(ii >> 5)*WB + (jj >> 5))*TILE2 + (size_t)(jj & 31)*TILE + (ii & 31)] : 0.0;
  const int si = w - 1 - ii, sj = w - 1 - jj;      // sj >= si
  return Bc.ff[((size_t)(sj >> 5)*WB + (si >> 5))*TILE2 + (size_t)(si & 31)*TILE + (sj & 31)];
}
// grid (tiles of the cell system, local cells): one CTA of 256 threads per tile (K, dd)
__global__ void __launch_bounds__(256) cs_assemble_kernel(CellRefs R, int TPCcs) {
  const int c = R.local_cells[blockIdx.y];
  const BandProb S = R.cs[c], A = R.chains[2*c], Bc = R.chains[2*c + 1];
  const bool has_qa = R.cells[c].has_qa != 0;
  const int K = blockIdx.x/TPCcs, dd = blockIdx.x%TPCcs;
  if (K + dd >= S.NT) return;
  double* t = S.tiles + ((size_t)K*S.TPC + dd)*TILE2;
  for (int e = threadIdx.x; e < TILE2; e += 256) {
    const int cj = e >> 5, ri = e & 31, i = (K + dd)*TILE + ri, j = K*TILE + cj;
    t[e] = i >= j ? cs_value(A, Bc, R.WB, has_qa, i, j) : 0.0;
  }
  if (dd == 0 && threadIdx.x < TILE) {
    const int w = R.WB*TILE, p = K*TILE + threadIdx.x, z = p/w, pp = p - z*w;
    double v;
    if (z == 0) v = A.rhs[(size_t)A.Kend*TILE + pp] + Bc.rhs[(size_t)Bc.Kend*TILE + (w - 1 - pp)];
    else if (has_qa && z == 1) v = A.gf[pp];
    else v = Bc.gf[w - 1 - pp];
    S.rhs[p] = v;
  }
}
// adds the Schur complement cell c leaves on its boundary separators into the boundary system (one launch per cell, in
// cell order: two neighbouring cells add into the same diagonal block)
__global__ void gq_add_cell_kernel(CellRefs R, int c, int TPCgq) {
  const BandProb S = R.cs[c], G = R.gq[0];
  const CellGeom g = R.cells[c];
  const int w = R.WB*TILE, nz = g.has_qa + g.has_qb;             // trailing zones of the cell system
  const long long total = (long long)nz*w*nz*w;
  for (long long e = (long long)blockIdx.x*blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x*blockDim.x) {
    const int ti = (int)(e/(nz*w)), tj = (int)(e%(nz*w));
    if (tj > ti) continue;
    const int i = w + ti, j = w + tj;                            // cell-system coordinates
    const int zi = ti/w, zj = tj/w;
    const int qi = (g.has_qa ? c - 1 + zi : c), qj = (g.has_qa ? c - 1 + zj : c);
    const int gi = qi*w + (ti - zi*w), gj = qj*w + (tj - zj*w);
    const double v = S.tiles[tile_elem(S.TPC, j >> 5, (i >> 5) - (j >> 5), i & 31, j & 31)];
    G.tiles[tile_elem(TPCgq, gj >> 5, (gi >> 5) - (gj >> 5), gi & 31, gj & 31)] += v;
  }
  for (int p = blockIdx.x*blockDim.x + threadIdx.x; p < nz*w; p += gridDim.x*blockDim.x) {
    const int z = p/w, q = (g.has_qa ? c - 1 + z : c);
    G.rhs[q*w + (p - z*w)] += S.rhs[w + p];
  }
}
// x_Q -> the cell systems' trailing rows and the chains' spike vectors (chain order)
__global__ void gq_scatter_kernel(CellRefs R) {
  const int c = R.local_cells[blockIdx.y];
  const BandProb S = R.cs[c], A = R.chains[2*c], Bc = R.chains[2*c + 1], G = R.gq[0];
  const CellGeom g = R.cells[c];
  const int w = R.WB*TILE;
  for (int p = blockIdx.x*blockDim.x + threadIdx.x; p < w; p += gridDim.x*blockDim.x) {
    if (g.has_qa) { const double x = G.rhs[(c - 1)*w + p]; S.rhs[w + p] = x; A.gf[p] = x; }
    if (g.has_qb) { const double x = G.rhs[c*w + p]; S.rhs[(1 + g.has_qa)*w + p] = x; Bc.gf[w - 1 - p] = x; }
  }
}
// x_M -> the near-separator rows of both chains (B reversed)
__global__ void cs_to_chain_kernel(CellRefs R) {
  const int c = R.local_cells[blockIdx.y];
  const BandProb S = R.cs[c], A = R.chains[2*c], Bc = R.chains[2*c + 1];
  const int w = R.WB*TILE;
  for (int p = blockIdx.x*blockDim.x + threadIdx.x; p < w; p += gridDim.x*blockDim.x) {
    const double x = S.rhs[p];
    A.rhs[(size_t)A.Kend*TILE + p] = x; Bc.rhs[(size_t)Bc.Kend*TILE + (w - 1 - p)] = x;
  }
}
__global__ void gather_dp_kernel(CellRefs R, double* __restrict__ dp) {
  const int c = R.local_cells[blockIdx.y];
  const BandProb S = R.cs[c], A = R.chains[2*c], Bc = R.chains[2*c + 1];
  const CellGeom g = R.cells[c];
  const int w = R.WB*TILE, hi = g.b1 + (g.has_qb ? w : 0);
  for (int p = g.a0 + blockIdx.x*blockDim.x + threadIdx.x; p < hi; p += gridDim.x*blockDim.x) {
    double x;
    if (p < g.m0) x = A.rhs[p - g.a0];
    else if (p < g.m0 + w) x = S.rhs[p - g.m0];
    else if (p < g.b1) x = Bc.rhs[g.b1 - 1 - p];
    else x = R.gq[0].rhs[c*w + (p - g.b1)];
    dp[p] = x;
  }
}

// =====================================================================================================================
// Host side

static int g_max_blocks = 0;
static int g_band_ctas_per_chain = 0;       // 0: split the worker CTAs by the work of the two pools
static int g_band_profile = 0;
void band_set_tuning(int band_ctas_per_chain) { if (band_ctas_per_chain >= 0) g_band_ctas_per_chain = band_ctas_per_chain; else g_band_profile = -band_ctas_per_chain; }
// stage timer of the optional profile (dynoba_set_tuning "band_profile"): synchronises the stream, so never on in timed runs
struct StageTimer { cudaStream_t s; std::chrono::steady_clock::time_point t; bool on;
  StageTimer(cudaStream_t s_) : s(s_), on(g_band_profile != 0) { if (on) { cudaStreamSynchronize(s); t = std::chrono::steady_clock::now(); } }
  void lap(const char* what) { if (!on) return; cudaStreamSynchronize(s); auto n = std::chrono::steady_clock::now();
    fprintf(stderr, "[band] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(n - t).count()); t = n; } };
static size_t g_chol_smem = 0;

static void chol_init() {
  if (g_max_blocks) return;
  int dev = 0, sms = 0, per = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // one CTA per SM: every spine CTA is alone on its SM
  const size_t need = std::max((size_t)(2*4*PANSZ + 2*TILE + 8*TSZ + 4*TILE2 + 64), std::max((size_t)4*(5*TILE2 + TILE), (size_t)(1 + SPK_ROWS)*SPK_STAGES*TILE2 + TILE))*sizeof(double);   // spine | band workers with prefetch stages | spike CTA
  g_chol_smem = std::max(need, (size_t)(220*1024) - 2048);
  cudaFuncSetAttribute(band_cholesky_dataflow_kernel_v3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g_chol_smem);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, band_cholesky_dataflow_kernel_v3, SP_WARPS*32, g_chol_smem);
  g_max_blocks = sms*(per > 0 ? per : 1);
  cudaFuncSetAttribute(band_backward_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200*1024);
}
// factorisation of np problems (device descriptors dprobs, host mirrors hprobs), flags cleared first
static int chol_launch(const BandProb* dprobs, const BandProb* hprobs, int np, int WB, int* fail, cudaStream_t s) {
  if (np <= 0) return 0;
  chol_init();
  CholJob job; job.p = dprobs; job.np = np; job.WB = WB; job.skew = 2; job.any_spiked = 0; job.ncols = 0;
  long long ntile = 0;
  for (int q = 0; q < np; q++) {
    const BandProb& P = hprobs[q];
    job.any_spiked |= P.spiked; job.ncols = std::max(job.ncols, P.NT);
    ntile += (long long)P.NT*(P.TPC + 1);
    const size_t nfl = (size_t)2*P.NT*P.TPC + P.NT + (size_t)WB*WB;
    cudaMemsetAsync(P.flags, 0, nfl*sizeof(int), s);
  }
  int grid = g_max_blocks;
  const long long want = (ntile + 3)/4 + np;
  if (grid > want) grid = (int)want;
  if (grid < np + 1 + (job.any_spiked ? 1 : 0)) grid = np + 1 + (job.any_spiked ? 1 : 0);
  // worker CTAs: without spikes all of them work on band tiles; else the two pools share them in proportion to their work
  // (relative work per column 330 : 730, band tiles : spike + FF updates), pool A never below what keeps a chain at the
  // spine's pace (~22 CTAs per chain).  Re-timed on H100 80GB HBM3 (700 W) with the m16n8k16 workers, C5 (WB 30, two
  // cells: plain chains of 4568 columns, spiked ones of 1016; 128 worker CTAs), tools/band_bench.py sweeping
  // band_ctas_per_chain -- pool A CTAs: plain spines done / pool B done / ms_factor per damped solve:
  //    84: 43.3 / 32.1 / 58.3 ms    88: 41.5 / 34.4 / 56.3    91 (these weights): 38.2 / 39.1 / 53.9
  //    92: 39.7 / 36.8 / 54.6      100: 36.9 / 46.5 / 61.3   104: 35.9 / 53.8 / 68.6    116: 34.2 / 99.0 / 114.0
  // The weights put the split where the plain chains and pool B finish together, so they stand.  Below ~21 CTAs per chain
  // the plain chains lose the spine's pace (64 CTAs: 19.9 us per column, 91: 8.4).  Splits whose pool-A warp count is a
  // multiple of the tasks per wavefront step (np * ceil((WB + 2) / skew) = 64 here: 80 or 96 CTAs) are much slower
  // (96: plain 61.2 ms): every warp then always draws the same task slot.
  const int workers = grid - np;
  if (!job.any_spiked) job.band_ctas = workers;
  else {
    double wa = 0, wb = 0;
    for (int q = 0; q < np; q++) { wa += 330.0*hprobs[q].Kend; if (hprobs[q].spiked) wb += 730.0*hprobs[q].Kend; }
    int a = g_band_ctas_per_chain > 0 ? g_band_ctas_per_chain*np : std::max((int)(workers*wa/(wa + wb)), std::min(22*np, workers/2));
    job.band_ctas = std::max(1, std::min(workers - 1, a));
  }
  // cooperative launch only for its co-residency guarantee (the flag waits need every warp resident)
  job.profile = g_band_profile;
  if (g_band_profile) { unsigned long long init[40]; for (int i = 0; i < 40; i++) init[i] = 0; init[34] = ~0ull; cudaMemcpyToSymbolAsync(g_prof, init, sizeof(init), 0, cudaMemcpyHostToDevice, s); }
  void* args[] = { (void*)&job, (void*)&fail };
  cudaLaunchCooperativeKernel((void*)band_cholesky_dataflow_kernel_v3, dim3(grid), dim3(SP_WARPS*32), args, g_chol_smem, s);
  if (g_band_profile) {
    unsigned long long t[40]; cudaStreamSynchronize(s); cudaMemcpyFromSymbol(t, g_prof, sizeof(t));
    fprintf(stderr, "[band]   launch: %d problems, WB %d, grid %d = %d spines + %d band CTAs + %d spike CTAs\n", np, WB, grid, np, job.band_ctas, grid - np - job.band_ctas);
    for (int q = 0; q < np && q < 32; q++) fprintf(stderr, "[band]   spine %d (%d columns%s) done at %8.3f ms\n", q, hprobs[q].Kend, hprobs[q].spiked ? ", spiked" : "", (t[q] - t[34])*1e-6);
    fprintf(stderr, "[band]   band pool done at %8.3f ms, spike pool at %8.3f ms\n", (t[32] - t[34])*1e-6, t[33] ? (t[33] - t[34])*1e-6 : 0.0);
  }
  return 1;
}
static int back_launch(const BandProb* dprobs, int np, int WB, cudaStream_t s) {
  if (np <= 0) return 0;
  chol_init();
  const size_t smem = ((size_t)(WB + 2)*TILE + (size_t)(2*BW_TW + 4*BW_CL + 1)*TILE + 6*TILE*BW_PS)*sizeof(double);
  BackJob job; job.p = dprobs; job.WB = WB;
  band_backward_cluster_kernel<<<np*BW_CL, (BW_TW + 1)*32, smem, s>>>(job);
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// Layout.  Cells are cut so that every chain is at least WB tiles long (a boundary separator then only touches the two
// chains next to it).  Chains without a spike (the first and the last of the system) cost a quarter of the flops per
// column of a spiked chain; `outer_weight` > 1 makes them longer.
static size_t align_up(size_t v, size_t a) { return (v + a - 1)/a*a; }

int band_plan_layout(BandPlan& P, int n, int bw, int ncell_request, int rank, int world) {
  DevBand& B = P.band;
  B = DevBand{};
  P.rank = rank; P.world = world; P.WBcs = P.TPCcs = P.WBgq = P.TPCgq = P.NTgq = 0;
  B.n = n; B.bw = std::max(0, std::min(bw, std::max(n - 1, 0)));
  B.NT = std::max((n + TILE - 1)/TILE, 1); B.n_pad = B.NT*TILE;
  B.WB = (B.bw + TILE - 1)/TILE; if (B.NT > 1 && B.WB < 1) B.WB = 1; if (B.WB > B.NT - 1) B.WB = B.NT - 1;
  const int WB = B.WB, NT = B.NT;
  // largest feasible number of cells: NT >= (2C - 1) WB + 2C max(WB, 2)
  const int minlen = std::max(WB, 2);
  int cmax = WB >= 1 ? (NT + WB)/(2*WB + 2*minlen) : 0;
  cmax = std::min(cmax, MAX_CELLS);
  int C;
  if (ncell_request > 0) C = std::min(ncell_request, cmax);
  else if (ncell_request < 0) C = 0;
  else {
    // default: one cell per GPU.  On one GPU a second cell pays for long systems when its two spiked chains (4x the flops
    // per column) are kept SHORT: the plain end chains then set the time, the worker warps absorb the spike work behind
    // them (C5: 73.4 ms per solve with one cell, 66.8 with two cells and end chains 4.5x as long; equal lengths: 86)
    C = world > 1 ? std::min(world, cmax) : (NT >= 4096 && cmax >= 2 ? 2 : 1);
    if (NT < std::max(8, 4*WB + 4)) C = 0;
    C = std::min(C, cmax);
  }
  B.ncell = C;
  P.cells.clear(); P.chains.clear(); P.cs.clear(); P.gq.clear();
  if (C == 0) {
    BandProb p{}; p.NT = NT; p.Kend = NT; p.TPC = WB + 1; p.spiked = 0;
    P.chains.push_back(p);
  } else {
    const long long free_tiles = (long long)NT - (long long)(2*C - 1)*WB;
    // relative chain lengths.  One GPU: plain end chains 4.5x the spiked ones.  Several GPUs (one cell per rank): a rank in
    // the middle runs two spiked chains (weight 0.5 each); an end rank runs its plain chain at the spine's pace (weight
    // 1.24) and, with the worker CTAs that leaves for the spike pool, a shorter spiked chain (0.6).  All of these weights
    // come from per-column timings of C5 on B200 and have not been re-timed on H100 (tuning: outer_weight, band_profile).
    std::vector<double> wgt(2*C, 1.0);
    if (P.outer_weight > 0 || world == 1 || C != world) { wgt[0] = wgt[2*C - 1] = P.outer_weight > 0 ? P.outer_weight : (C >= 2 ? 4.5 : 1.0); }
    else { for (auto& x : wgt) x = 0.5; wgt[0] = wgt[2*C - 1] = 1.24; wgt[1] = wgt[2*C - 2] = 0.6; }
    double wsum = 0; for (double x : wgt) wsum += x;
    std::vector<int> len(2*C);
    long long used = 0;
    for (int k = 0; k < 2*C; k++) { len[k] = std::max(minlen, (int)(free_tiles*wgt[k]/wsum)); used += len[k]; }
    for (int k = 0; used < free_tiles; k = (k + 1)%(2*C)) { len[k]++; used++; }
    for (int k = 0; used > free_tiles; k = (k + 1)%(2*C)) if (len[k] > minlen) { len[k]--; used--; }
    int t = 0;
    for (int c = 0; c < C; c++) {
      CellGeom g{}; g.has_qa = c > 0; g.has_qb = c < C - 1;
      g.q0 = t*TILE; if (c > 0) t += WB;
      g.a0 = t*TILE; t += len[2*c];
      g.m0 = t*TILE; t += WB;
      t += len[2*c + 1];
      g.b1 = t*TILE;
      P.cells.push_back(g);
      BandProb a{}; a.NT = len[2*c] + WB; a.Kend = len[2*c]; a.spiked = g.has_qa; a.TPC = WB + 1 + (a.spiked ? WB : 0);
      BandProb b{}; b.NT = len[2*c + 1] + WB; b.Kend = len[2*c + 1]; b.spiked = g.has_qb; b.TPC = WB + 1 + (b.spiked ? WB : 0);
      P.chains.push_back(a); P.chains.push_back(b);
    }
    if (t != NT) return -1;
    P.WBcs = std::max(1, (C >= 2 ? 3 : 1)*WB - 1); P.TPCcs = P.WBcs + 1;
    for (int c = 0; c < C; c++) {
      BandProb s{}; s.NT = WB*(1 + P.cells[c].has_qa + P.cells[c].has_qb); s.Kend = WB; s.TPC = P.TPCcs; s.spiked = 0;
      P.cs.push_back(s);
    }
    P.NTgq = (C - 1)*WB;
    if (C >= 2) {
      P.WBgq = std::max(1, std::min(2*WB - 1, P.NTgq - 1)); P.TPCgq = P.WBgq + 1;
      BandProb gq{}; gq.NT = P.NTgq; gq.Kend = P.NTgq; gq.TPC = P.TPCgq; gq.spiked = 0;
      P.gq.push_back(gq);
    } else { P.WBgq = 0; P.TPCgq = 1; }
  }
  P.nchain = (int)P.chains.size(); P.ncs = (int)P.cs.size();
  P.local_cells.clear();
  for (int c = 0; c < C; c++) if (c*world/C == rank) P.local_cells.push_back(c);
  // ---- sizes.  doubles: [accumulated: chain tiles | ff | rhs + gf] [cs tiles + rhs] [gq tiles + rhs] [linv] [spike scratch]
  size_t nd = 0, ni = 0;
  auto take = [&](size_t cnt) { const size_t o = nd; nd += align_up(cnt, 32); return o; };
  for (auto& p : P.chains) take((size_t)p.NT*p.TPC*TILE2);
  for (auto& p : P.chains) if (p.spiked) take((size_t)WB*WB*TILE2);
  for (auto& p : P.chains) { take((size_t)p.NT*TILE); if (p.spiked) take((size_t)WB*TILE); }
  P.acc_count = nd;
  for (auto& p : P.cs) { take((size_t)p.NT*p.TPC*TILE2); take((size_t)p.NT*TILE); }
  for (auto& p : P.gq) { take((size_t)p.NT*p.TPC*TILE2 + (size_t)p.NT*TILE); }
  for (auto& p : P.chains) take((size_t)std::max(p.Kend, 1)*TILE2);
  for (auto& p : P.cs) take((size_t)p.Kend*TILE2);
  for (auto& p : P.gq) take((size_t)p.Kend*TILE2);
  int maxk = 1; for (auto& p : P.chains) maxk = std::max(maxk, p.Kend);
  take((size_t)P.nchain*((maxk + SF_CH - 1)/SF_CH)*std::max(WB, 1)*TILE);
  P.n_doubles = nd;
  auto nflags = [&](const BandProb& p, int wb) { return align_up((size_t)2*p.NT*p.TPC + p.NT + (size_t)wb*wb, 32); };
  for (auto& p : P.chains) ni += nflags(p, WB);
  for (auto& p : P.cs) ni += nflags(p, P.WBcs);
  for (auto& p : P.gq) ni += nflags(p, P.WBgq);
  P.n_ints = ni;
  P.n_desc_bytes = align_up(sizeof(BandProb)*(size_t)(2*P.nchain + 2*P.ncs + 1) + sizeof(CellGeom)*(size_t)std::max(C, 1) + sizeof(int)*(size_t)std::max(C, 1), 256) + 1024;
  return 0;
}

// first scalar position of the cells owned by each rank (bounds[world] = n_pad): what the host needs to shard landmarks
// so that a rank's contribution stays inside its own cells
int band_plan_partition(int n, int bw, int world, int* bounds) {
  BandPlan P{}; P.outer_weight = 0;
  if (band_plan_layout(P, n, bw, 0, 0, world)) return -1;
  const int C = P.band.ncell;
  for (int r = 0; r <= world; r++) bounds[r] = P.band.n_pad;
  bounds[0] = 0;
  for (int c = C - 1; c >= 0; c--) { const int owner = c*world/C; bounds[owner] = c == 0 ? 0 : P.cells[c].q0; }
  for (int r = world - 1; r > 0; r--) if (bounds[r] > bounds[r + 1]) bounds[r] = bounds[r + 1];     // ranks without a cell
  return C;
}

void band_plan_bind(BandPlan& P, double* dbase, int* ibase, void* desc_base, double* dp) {
  DevBand& B = P.band;
  const int WB = B.WB, C = B.ncell;
  size_t nd = 0, ni = 0;
  auto take = [&](size_t cnt) { double* p = dbase + nd; nd += align_up(cnt, 32); return p; };
  auto takei = [&](const BandProb& p, int wb) { int* q = ibase + ni; ni += align_up((size_t)2*p.NT*p.TPC + p.NT + (size_t)wb*wb, 32); return q; };
  P.reduce_ranges.clear();
  for (auto& p : P.chains) p.tiles = take((size_t)p.NT*p.TPC*TILE2);
  for (auto& p : P.chains) p.ff = p.spiked ? take((size_t)WB*WB*TILE2) : nullptr;
  P.rhs_region = dbase + nd;
  for (auto& p : P.chains) { p.rhs = take((size_t)p.NT*TILE); p.gf = p.spiked ? take((size_t)WB*TILE) : nullptr; }
  P.rhs_count = (size_t)(dbase + nd - P.rhs_region);
  B.acc = dbase; B.acc_count = nd;
  for (auto& p : P.cs) { p.tiles = take((size_t)p.NT*p.TPC*TILE2); p.rhs = take((size_t)p.NT*TILE); p.ff = nullptr; p.gf = nullptr; }
  P.gq_base = nullptr; P.gq_count = 0;
  for (auto& p : P.gq) { P.gq_count = (size_t)p.NT*p.TPC*TILE2 + (size_t)p.NT*TILE; P.gq_base = take(P.gq_count); p.tiles = P.gq_base; p.rhs = P.gq_base + (size_t)p.NT*p.TPC*TILE2; p.ff = nullptr; p.gf = nullptr; }
  for (auto& p : P.chains) p.linv = take((size_t)std::max(p.Kend, 1)*TILE2);
  for (auto& p : P.cs) p.linv = take((size_t)p.Kend*TILE2);
  for (auto& p : P.gq) p.linv = take((size_t)p.Kend*TILE2);
  int maxk = 1; for (auto& p : P.chains) maxk = std::max(maxk, p.Kend);
  P.spike_scratch = take((size_t)P.nchain*((maxk + SF_CH - 1)/SF_CH)*std::max(WB, 1)*TILE);
  for (auto& p : P.chains) p.flags = takei(p, WB);
  for (auto& p : P.cs) p.flags = takei(p, P.WBcs);
  for (auto& p : P.gq) p.flags = takei(p, P.WBgq);
  P.flags_base = ibase; P.flags_count = ni;
  // multi-GPU: the accumulated tiles / ff of a cell are summed at its owner
  for (int c = 0; c < C; c++) {
    const int owner = c*P.world/C;
    const BandProb &a = P.chains[2*c], &b = P.chains[2*c + 1];
    P.reduce_ranges.push_back({ a.tiles, (size_t)(b.tiles + (size_t)b.NT*b.TPC*TILE2 - a.tiles), owner });
    if (a.spiked) P.reduce_ranges.push_back({ a.ff, (size_t)WB*WB*TILE2, owner });
    if (b.spiked) P.reduce_ranges.push_back({ b.ff, (size_t)WB*WB*TILE2, owner });
  }
  // ---- descriptors -> device
  std::vector<BandProb> lc, lcs;
  for (int c : P.local_cells) { lc.push_back(P.chains[2*c]); lc.push_back(P.chains[2*c + 1]); lcs.push_back(P.cs[c]); }
  if (C == 0) lc.push_back(P.chains[0]);
  P.d_local_chains_host = lc; P.d_local_cs_host = lcs; P.n_local_chains = (int)lc.size(); P.n_local_cs = (int)lcs.size();
  char* d = (char*)desc_base; size_t off = 0;
  auto put = [&](const void* src, size_t bytes) { void* q = d + off; if (bytes) cudaMemcpy(q, src, bytes, cudaMemcpyHostToDevice); off += align_up(std::max<size_t>(bytes, 1), 16); return q; };
  P.d_chains = (BandProb*)put(P.chains.data(), sizeof(BandProb)*P.chains.size());
  P.d_cs = (BandProb*)put(P.cs.data(), sizeof(BandProb)*P.cs.size());
  P.d_gq = (BandProb*)put(P.gq.data(), sizeof(BandProb)*P.gq.size());
  P.d_local_chains = (BandProb*)put(lc.data(), sizeof(BandProb)*lc.size());
  P.d_local_cs = (BandProb*)put(lcs.data(), sizeof(BandProb)*lcs.size());
  const CellGeom* dcells = (const CellGeom*)put(P.cells.data(), sizeof(CellGeom)*P.cells.size());
  P.d_local_cell_ids = (int*)put(P.local_cells.data(), sizeof(int)*P.local_cells.size());
  B.chains = P.d_chains; B.cells = dcells;
  B.dp = C == 0 ? P.chains[0].rhs : dp;
}

// Rebuilds the per-cell reduce list from the position ranges [lo[r], hi[r]] (scalar, inclusive) the factors of every
// rank touch: the tiles of cell c only have to be summed at its owner over the columns a NON-owner contributes to.
// Entries (i >= j) of a rank lie inside its range, in the column of j (band) or of i (spike tiles of an A chain), so the
// touched columns of a chain are the tiles of range & chain; the Q x Q block of an A chain is touched when the range meets Qa
// (the B chain's only receives spike products, which are formed at the owner).
void band_plan_trim(BandPlan& P, const int* lo, const int* hi) {
  const DevBand& B = P.band; const int C = B.ncell, WB = B.WB, w = WB*TILE;
  P.reduce_ranges.clear();
  for (int c = 0; c < C; c++) {
    const int owner = c*P.world/C;
    const CellGeom& g = P.cells[c];
    const BandProb &a = P.chains[2*c], &b = P.chains[2*c + 1];
    int a_lo = INT32_MAX, a_hi = -1, b_lo = INT32_MAX, b_hi = -1; bool ffa = false;
    for (int r = 0; r < P.world; r++) {
      if (r == owner || lo[r] > hi[r]) continue;
      const int p0 = std::max(lo[r], g.a0), p1 = std::min(hi[r], g.m0 + w - 1);           // chain A: natural order from a0
      if (p0 <= p1) { a_lo = std::min(a_lo, (p0 - g.a0)/TILE); a_hi = std::max(a_hi, (p1 - g.a0)/TILE); }
      const int q0 = std::max(lo[r], g.m0), q1 = std::min(hi[r], g.b1 - 1);                // chain B: reversed from b1 - 1
      if (q0 <= q1) { b_lo = std::min(b_lo, (g.b1 - 1 - q1)/TILE); b_hi = std::max(b_hi, (g.b1 - 1 - q0)/TILE); }
      if (g.has_qa && lo[r] < g.a0 && hi[r] >= g.q0) ffa = true;
    }
    if (a_hi >= a_lo) P.reduce_ranges.push_back({ a.tiles + (size_t)a_lo*a.TPC*TILE2, (size_t)(a_hi - a_lo + 1)*a.TPC*TILE2, owner });
    if (b_hi >= b_lo) P.reduce_ranges.push_back({ b.tiles + (size_t)b_lo*b.TPC*TILE2, (size_t)(b_hi - b_lo + 1)*b.TPC*TILE2, owner });
    if (ffa) P.reduce_ranges.push_back({ a.ff, (size_t)WB*WB*TILE2, owner });
  }
}

static CellRefs cell_refs(const BandPlan& P) { return CellRefs{ P.d_chains, P.d_cs, P.d_gq, P.band.cells, P.d_local_cell_ids, P.band.WB }; }

int launch_band_factor(const BandPlan& P, int* fail, cudaStream_t s) {
  const DevBand& B = P.band; const int WB = B.WB, C = B.ncell;
  int launches = 0;
  StageTimer tm(s);
  launches += chol_launch(P.d_local_chains, P.d_local_chains_host.data(), P.n_local_chains, WB, fail, s);
  tm.lap("chains");
  if (P.n_local_chains) { int maxk = 1; for (auto& p : P.d_local_chains_host) maxk = std::max(maxk, p.Kend);
    diag_inverse_kernel<<<dim3((maxk + 3)/4, P.n_local_chains), 128, 0, s>>>(P.d_local_chains); launches++; }
  if (C == 0) return launches;
  const int nloc = (int)P.local_cells.size();
  if (nloc) {
    bool any_spiked = false; int maxk = 1;
    for (auto& p : P.d_local_chains_host) { any_spiked |= p.spiked != 0; maxk = std::max(maxk, p.Kend); }
    if (any_spiked) {
      int allmaxk = 1; for (auto& p : P.chains) allmaxk = std::max(allmaxk, p.Kend);
      const int maxchunks = (allmaxk + SF_CH - 1)/SF_CH;
      spike_forward_partial_kernel<<<dim3((maxk + SF_CH - 1)/SF_CH, P.n_local_chains), 256, 0, s>>>(P.d_local_chains, WB, P.spike_scratch, maxchunks);
      spike_forward_reduce_kernel<<<dim3((WB*TILE + 255)/256, P.n_local_chains), 256, 0, s>>>(P.d_local_chains, WB, P.spike_scratch, maxchunks);
      launches += 2;
    }
    const int ntcs = WB*(C >= 2 ? 3 : 1);
    tm.lap("diag inverse + spike forward");
    cs_assemble_kernel<<<dim3(ntcs*P.TPCcs, nloc), 256, 0, s>>>(cell_refs(P), P.TPCcs); launches++;
    tm.lap("cell systems: assemble");
    launches += chol_launch(P.d_local_cs, P.d_local_cs_host.data(), P.n_local_cs, P.WBcs, fail, s);
    diag_inverse_kernel<<<dim3((WB + 3)/4, P.n_local_cs), 128, 0, s>>>(P.d_local_cs); launches++;
    tm.lap("cell systems: factor");
  }
  if (C >= 2) {
    cudaMemsetAsync(P.gq_base, 0, P.gq_count*sizeof(double), s);
    for (int c : P.local_cells) { gq_add_cell_kernel<<<device_sm_count(), 256, 0, s>>>(cell_refs(P), c, P.TPCgq); launches++; }
    tm.lap("boundary system: assemble");
  }
  return launches;
}

int launch_band_top(const BandPlan& P, int* fail, cudaStream_t s) {
  const DevBand& B = P.band; const int WB = B.WB, C = B.ncell;
  int launches = 0;
  if (C == 0) { launches += back_launch(P.d_local_chains, P.n_local_chains, WB, s); return launches; }
  const int nloc = (int)P.local_cells.size();
  StageTimer tm(s);
  if (C >= 2) {
    launches += chol_launch(P.d_gq, P.gq.data(), 1, P.WBgq, fail, s);                  // boundary system (replicated on every rank)
    diag_inverse_kernel<<<dim3((P.NTgq + 3)/4, 1), 128, 0, s>>>(P.d_gq); launches++;
    launches += back_launch(P.d_gq, 1, P.WBgq, s);
    if (nloc) { gq_scatter_kernel<<<dim3(8, nloc), 256, 0, s>>>(cell_refs(P)); launches++; }
    tm.lap("boundary system: solve");
  }
  if (P.world > 1) cudaMemsetAsync(B.dp, 0, (size_t)B.n_pad*sizeof(double), s);        // the owners' segments are summed by the caller
  if (!nloc) return launches;
  launches += back_launch(P.d_local_cs, P.n_local_cs, P.WBcs, s);                      // x_M
  cs_to_chain_kernel<<<dim3(8, nloc), 256, 0, s>>>(cell_refs(P)); launches++;
  tm.lap("cell systems: back-substitution");
  bool any_spiked = false; int maxk = 1;
  for (auto& p : P.d_local_chains_host) { any_spiked |= p.spiked != 0; maxk = std::max(maxk, p.Kend); }
  if (any_spiked) { spike_backward_kernel<<<dim3((maxk + 7)/8, P.n_local_chains), 256, (size_t)WB*TILE*sizeof(double), s>>>(P.d_local_chains, WB); launches++; }
  launches += back_launch(P.d_local_chains, P.n_local_chains, WB, s);
  gather_dp_kernel<<<dim3(64, nloc), 256, 0, s>>>(cell_refs(P), B.dp); launches++;
  tm.lap("chains: back-substitution");
  return launches;
}

}  // namespace dynoba
