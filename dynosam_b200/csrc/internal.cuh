// internal.cuh -- device data model shared by the kernel translation units (DESIGN.md "Data layout in HBM").
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <mutex>
#include <vector>
#include "factors.cuh"

namespace dynoba {

constexpr int TILE = 32;           // band-Cholesky tile edge
constexpr int TILE2 = TILE*TILE;
// SM count of the current device: grid of the grid-stride clear / accumulate kernels (any value is correct)
inline int device_sm_count() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 1;
}

// Variables, SoA, fp64.  Pose-like variables are stored in *solver order* (ordered by the frame hint),
// landmarks in group order (sorted by the first pose they touch).  strides are padded to 32.
struct DevVars {
  int np, np_stride;   double* pose;   // [12][np_stride]  rows 0-8 R (row-major), 9-11 t
  int nl, nl_stride;   double* point;  // [3][nl_stride]
  int nf, nf_stride;   double* flow;   // [2][nf_stride]
  int naux, naux_stride; const double* aux;  // [12][naux_stride]
  double K[6];
};

// One homogeneous factor block, sorted by landmark group, SoA.
struct DevBlock {
  int type, n, stride;
  const int* idx;       // [arity][stride]   pose slots: solver position; point/flow slots: device index
  const double* meas;   // [meas][stride]
  const double* isig;   // [sigma_dim][stride]  1/sigma
  int sigma_dim;
  const int* aux;       // [stride] or nullptr
  double robust_k;
  double* J;            // [dim*jcols][stride]  whitened, Huber-weighted Jacobian, element e = row*jcols + col
  double* b;            // [dim][stride]        rhs = -sqrt(w) * r_w
  // landmark groups (simple groups: exactly one landmark, all of its factors in this block)
  int n_groups;
  const int* grp_ptr;   // [n_groups+1] into the sorted factor range
  const int* grp_lmk;   // [n_groups]   device landmark index, or -1 when the group is handled by the general path
  double* num_scratch;  // numeric-Jacobian factor types: per-CTA partial sums of the column-parallel linearize kernel
};

// Storage of the reduced (camera + object-motion) system S, lower triangle, TILE x TILE tiles (column-major inside a
// tile: element (r, c) at c*TILE + r), and of its Cholesky factor, which overwrites it.
//
// With pose-like variables in frame order S is banded (half-width bw <= WB tiles).  The time axis is cut into `ncell`
// CELLS  [Qa] A -> M <- B [Qb]  (tools/cell_proto.py is the executable specification):
//   * chain A = positions [a0, m0 + w) in natural order, chain B = positions [m0, b1) REVERSED (w = WB*TILE): two band
//     problems that are eliminated at the same time towards the middle separator M = [m0, m0 + w), which both hold as
//     their trailing columns and in which both leave their Schur complement;
//   * a boundary separator Q between two cells is eliminated last.  The chain that starts next to it (B of the cell
//     before, A of the cell after) carries WB extra dense tile rows per column, its "spike" Z = coupling to Q, which
//     fills in along the chain, and the Q x Q block `ff`.  Original Q x Q entries live in the `ff` of the A chain after it.
// ncell == 0: one plain band problem (chain 0), no separators.
struct BandProb {
  double* tiles;   // [NT][TPC][TILE2]   tile (K, t): t <= WB: band tile (K + t, K);  t = WB + 1 + r: spike tile (Q tile r, K)
  double* rhs;     // [NT][TILE]         g, then y = L^-1 g, then x
  double* ff;      // [WB][WB][TILE2]    Q x Q block (lower block triangle), spiked chains only
  double* gf;      // [WB][TILE]         rhs of Q
  double* linv;    // [Kend][TILE2]      inverses of the diagonal tiles of L
  int* flags;      // done [NT*TPC] | pre [NT*TPC] | ydone [NT] | ffcnt [WB*WB]
  int NT, Kend;    // columns [0, Kend) are factored; columns [Kend, NT) only receive their Schur complement
  int TPC;         // tiles per column: WB + 1, + WB when spiked
  int spiked;
};
struct CellGeom { int q0, a0, m0, b1, has_qa, has_qb; };   // scalar positions: Qa = [q0, a0) (empty when !has_qa), A interior
                                                           // [a0, m0), M [m0, m0 + w), B interior [m0 + w, b1), Qb [b1, b1 + w)
constexpr int MAX_CELLS = 16;
struct DevBand {
  int n, n_pad, NT, WB, bw;
  int ncell;
  const BandProb* chains;   // [max(1, 2*ncell)]  chain 2c = A of cell c, 2c + 1 = B   (device array; host mirror for host reads)
  const CellGeom* cells;    // [ncell]
  double* acc; size_t acc_count;   // every buffer the Schur kernels accumulate into (tiles, ff, rhs, gf), contiguous
  double* dp;               // [n_pad] solution delta_p in solver order
};
// descriptor reads: read-only path on the device (the descriptors are written once by the host), plain loads on the host
__host__ __device__ __forceinline__ int dld(const int& x) {
#if defined(__CUDA_ARCH__)
  return __ldg(&x);
#else
  return x;
#endif
}
__host__ __device__ __forceinline__ double* dld(double* const& x) {
#if defined(__CUDA_ARCH__)
  return reinterpret_cast<double*>(__ldg(reinterpret_cast<const unsigned long long*>(&x)));
#else
  return x;
#endif
}
__host__ __device__ __forceinline__ size_t tile_elem(int TPC, int K, int t, int r, int c) {
  return ((size_t)K*TPC + t)*TILE2 + (size_t)c*TILE + r;
}
__host__ __device__ __forceinline__ int band_cell(const DevBand& B, int p) {    // cell whose [q0, b1) holds position p
  int c = (int)((long long)p*B.ncell/B.n_pad);
  while (c > 0 && p < dld(B.cells[c].q0)) c--;
  while (c + 1 < B.ncell && p >= dld(B.cells[c + 1].q0)) c++;
  return c;
}
// Geometry and storage of one cell, loaded once (a handful of descriptor reads) and then used for many entries: the
// kernels that scatter 6x6 blocks resolve the cell of the block's first column and address the 36 entries with integer
// arithmetic only.
struct BandCellRef {
  int q0, a0, m0, b1;          // j in [q0, b1) belongs to this cell
  double *ta, *tb, *ffa;       // tiles of chain A / B, Q x Q block of chain A
  int tpca, tpcb;
};
__host__ __device__ __forceinline__ BandCellRef band_cell_ref(const DevBand& B, int j) {
  BandCellRef R;
  if (B.ncell == 0) { R.q0 = 0; R.a0 = 0; R.m0 = B.n_pad; R.b1 = B.n_pad; R.ta = dld(B.chains[0].tiles); R.tb = nullptr; R.ffa = nullptr; R.tpca = B.WB + 1; R.tpcb = 0; return R; }
  const int c = band_cell(B, j);
  R.q0 = dld(B.cells[c].q0); R.a0 = dld(B.cells[c].a0); R.m0 = dld(B.cells[c].m0); R.b1 = dld(B.cells[c].b1);
  R.ta = dld(B.chains[2*c].tiles); R.tb = dld(B.chains[2*c + 1].tiles); R.ffa = dld(B.chains[2*c].ff);
  R.tpca = dld(B.chains[2*c].TPC); R.tpcb = dld(B.chains[2*c + 1].TPC);
  return R;
}
// address of entry (i >= j) whose column j lies in the cell of R
__host__ __device__ __forceinline__ double* band_at_in(const DevBand& B, const BandCellRef& R, int i, int j) {
  const int w = B.WB*TILE;
  if (B.ncell == 0 || (j >= R.a0 && i < R.m0 + w)) { const int li = i - R.a0, lj = j - R.a0; return R.ta + tile_elem(R.tpca, lj >> 5, (li >> 5) - (lj >> 5), li & 31, lj & 31); }
  if (j < R.a0) {
    const int sj = j - R.q0;
    if (i < R.a0) { const int si = i - R.q0; return R.ffa + ((size_t)(si >> 5)*B.WB + (sj >> 5))*TILE2 + (size_t)(sj & 31)*TILE + (si & 31); }
    const int li = i - R.a0;
    return R.ta + tile_elem(R.tpca, li >> 5, B.WB + 1 + (sj >> 5), sj & 31, li & 31);
  }
  if (i < R.b1) { const int li = R.b1 - 1 - j, lj = R.b1 - 1 - i; return R.tb + tile_elem(R.tpcb, lj >> 5, (li >> 5) - (lj >> 5), li & 31, lj & 31); }
  const int s = R.b1 + w - 1 - i, lc = R.b1 - 1 - j;
  return R.tb + tile_elem(R.tpcb, lc >> 5, B.WB + 1 + (s >> 5), s & 31, lc & 31);
}
// address of entry (i >= j) / of rhs element p of the reduced system
__host__ __device__ __forceinline__ double* band_at(const DevBand& B, int i, int j) {
  const BandCellRef R = band_cell_ref(B, j);
  return band_at_in(B, R, i, j);
}
// same, reusing R when column j still lies in its cell (the common case for the entries of one 6x6 block)
__host__ __device__ __forceinline__ double* band_at_cached(const DevBand& B, BandCellRef& R, int i, int j) {
  if (B.ncell != 0 && (j < R.q0 || j >= R.b1)) R = band_cell_ref(B, j);
  return band_at_in(B, R, i, j);
}
// 6x6 block scatter: rows i0..i0+5, columns j0..j0+5 (i0 >= j0).  Almost every block lies inside ONE band chain (A or B
// of one cell): its entries are then addressed from a per-block base with a few integer operations each.  Blocks that
// touch a separator or straddle a zone boundary take the general, out-of-line path per entry (keeps the unrolled
// 36-entry flush loops of the callers small).
struct BandBlockRef { double* base; int tpc, oi, oj, rev, fast; };
#if defined(__CUDACC__)
// fire-and-forget fp64 addition into the reduced system: RED on the GLOBAL window.  A plain atomicAdd through a pointer the
// compiler cannot prove global (loaded from a descriptor) becomes a generic, value-returning ATOM with an address-space
// query per call
__device__ __forceinline__ void red_add(double* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" :: "l"(__cvta_generic_to_global(p)), "d"(v) : "memory");
}
static __device__ __noinline__ double* band_at_slow(DevBand B, int i, int j) { return band_at(B, i, j); }   // (by value: a reference would
                                                                 // force the caller's kernel parameter into local memory)
__device__ __forceinline__ BandBlockRef band_block_ref(const DevBand& B, int i0, int j0) {
  BandBlockRef K; K.fast = 1; K.rev = 0;
  if (B.ncell == 0) { K.base = dld(B.chains[0].tiles); K.tpc = B.WB + 1; K.oi = 0; K.oj = 0; return K; }
  const BandCellRef R = band_cell_ref(B, j0);
  const int w = B.WB*TILE;
  if (j0 >= R.a0 && i0 + 5 < R.m0 + w) { K.base = R.ta; K.tpc = R.tpca; K.oi = R.a0; K.oj = R.a0; return K; }                  // chain A
  if (j0 >= R.m0 && j0 + 5 < R.b1 && i0 >= R.m0 + w && i0 + 5 < R.b1) { K.base = R.tb; K.tpc = R.tpcb; K.oi = R.b1 - 1; K.rev = 1; return K; }   // chain B
  K.fast = 0; K.base = nullptr; K.tpc = 0; K.oi = K.oj = 0;
  return K;
}
__device__ __forceinline__ double* band_block_at(const DevBand& B, const BandBlockRef& K, int i, int j) {
  if (!K.fast) return band_at_slow(B, i, j);
  const int li = K.rev ? K.oi - j : i - K.oi, lj = K.rev ? K.oi - i : j - K.oj;
  return K.base + tile_elem(K.tpc, lj >> 5, (li >> 5) - (lj >> 5), li & 31, lj & 31);
}
#endif
__host__ __device__ __forceinline__ double* rhs_at(const DevBand& B, int p) {
  if (B.ncell == 0) return dld(B.chains[0].rhs) + p;
  const int c = band_cell(B, p), w = B.WB*TILE;
  const int a0 = dld(B.cells[c].a0);
  if (p < a0) return dld(B.chains[2*c].gf) + (p - dld(B.cells[c].q0));
  if (p < dld(B.cells[c].m0) + w) return dld(B.chains[2*c].rhs) + (p - a0);
  return dld(B.chains[2*c + 1].rhs) + (dld(B.cells[c].b1) - 1 - p);
}

// Landmark groups the per-landmark kernels do not cover (chains of points, landmarks spanning factor blocks):
// factor references (block, sorted index) per group, points of a group contiguous from gl0 (gnl of them).
struct GeneralGroups {
  int n_groups;
  const DevBlock* blocks;   // device copy of every factor block descriptor
  const int* gptr;          // [n_groups+1] into refs
  const void* refs;         // [gptr[n_groups]] (int blk, int idx)
  const int* gl0;           // [n_groups] first device point index
  const int* gnl;           // [n_groups] number of points (<= 21)
};

// Window decomposition of a factor block for kernels_window.cu (built by the host in finalize)
constexpr int WIN_NLOC_MAX = 48;          // largest window (local pose-like variables of a chunk)
constexpr int WIN_TMAX = 24;              // factors per landmark on the window path (larger ones: kernels_schur.cu)
constexpr int WIN_SLOT_DOUBLES = 42;      // one staged clique variable of one factor: Wt[3][6] | A[3][6] | rb[3] | meta | pad[2]
constexpr int WIN_BATCH_SLOTS = 256;      // slots per shared-memory buffer of the accumulate kernel
constexpr int WIN_BATCH_LMK = 32;         // landmarks per batch
// The accumulate kernel tiles the window's lower triangle of 6x6 blocks into 8x4 block tiles, one tile per warp (a
// landmark's clique is a contiguous range of local variables, so whole tiles are active or idle together).
__host__ __device__ __forceinline__ int win_ntiles(int nloc) {
  int n = 0;
  for (int tr = 0; tr*8 < nloc; tr++) { const int rmax = (8*tr + 7 < nloc - 1) ? 8*tr + 7 : nloc - 1; n += rmax/4 + 1; }
  return n;
}
constexpr int WIN_ACC_WARPS = 16;         // tiles per CTA (stripe) of the accumulate kernel
struct DevWindows {
  int n_jobs;
  const int4* jobs;              // (chunk, stripe of the window's lower-triangular blocks, first batch, end batch)
  const int4* batches;           // (first group, end group, first factor, end factor): runs of window-path landmarks,
                                 // at most WIN_BATCH_LMK landmarks / WIN_BATCH_SLOTS slots, never crossing a chunk
  const int* chunk_nloc;         // [n_chunks]
  const int* cvars;              // [n_chunks][WIN_NLOC_MAX] solver positions, ascending
  const unsigned char* lvar;     // [npose_slots][stride] local variable of each factor's pose slot
  const unsigned char* grp_win;  // [n_groups] 0: general path, 1: window path, 2: per-landmark atomics path
  double* slots;                 // [n*npose_slots][WIN_SLOT_DOUBLES] staged slots in factor order (HBM scratch)
};

// Dense quadratic prior over n pose-like variables (kernels_prior.cu): gtsam::LinearContainerFactor(HessianFactor)
struct DevPrior {
  int n; const int* pos;          // solver positions of the variables
  const double* lin;              // [n][12] linearisation point
  const double* G; const double* g; double f;   // [6n][6n] row-major information, [6n] linear term, constant
  double* delta; double* gcur;    // [6n] local coordinates / g - G delta at the current linearisation
};
int launch_prior_eval(const DevPrior& P, const DevVars& v, double* partial, int store, cudaStream_t s);
int launch_prior_accum(const DevPrior& P, const DevBand& B, cudaStream_t s);
int launch_prior_model(const DevPrior& P, const DevBand& B, double* partial, cudaStream_t s);

// ---- launchers (each returns the number of kernels it launched)
int launch_linearize(const DevBlock& blk, const DevVars& v, double* partials, cudaStream_t s);
int launch_error(const DevBlock& blk, const DevVars& v, double* partials, double* per_factor, cudaStream_t s);
int launch_sum(const double* partials, int n, double* out, cudaStream_t s);
int linearize_grid(int n);          // number of partial sums a linearize/error launch of n factors writes
int numeric_grid(int type, int n);  // CTAs of the column-parallel linearize kernel (0 for analytic factor types)

int launch_band_clear(const DevBand& B, double lambda, int rank, int world, cudaStream_t s);   // world == 1: rank 0 writes the whole diagonal
int launch_schur_simple(const DevBlock& blk, const unsigned char* grp_win, const DevBand& B, double lambda, int* fail, cudaStream_t s);
int launch_schur_window(const DevBlock& blk, const DevWindows& Wn, const DevBand& B, double lambda, int* fail, cudaStream_t s);
int launch_schur_general(const GeneralGroups& G, const DevBand& B, double lambda, int* fail, cudaStream_t s);
int launch_backsub_general(const GeneralGroups& G, const DevBand& B, double lambda, double* dl_point, int nl_stride,
                           double* partials, cudaStream_t s);
int general_grid(int n_groups);
int launch_pose_factors(const DevBlock& blk, const DevBand& B, cudaStream_t s);
// ---- reduced solve (kernels_band.cu).  band_plan_layout decides the cell decomposition and the sizes of the three
// device allocations; band_plan_bind places every buffer and uploads the problem descriptors.  The solve runs in three
// stages so that the multi-GPU host can put its collectives between them (see api.cu: solve_step).
struct BandPlan {
  DevBand band;                       // device view (chains / cells point to device arrays)
  int rank, world;                    // cells are dealt to ranks in contiguous runs; owner(c) = c*world/ncell
  double outer_weight;                // relative length of the two unspiked end chains (0 = default)
  int nchain, ncs, WBcs, TPCcs, WBgq, TPCgq, NTgq;
  size_t n_doubles, n_ints, n_desc_bytes;        // sizes of the allocations band_plan_bind wants
  size_t acc_count;                   // leading part of the double allocation that band_clear zeroes every trial
  std::vector<BandProb> chains, cs, gq;          // host mirrors (device pointers inside)
  std::vector<CellGeom> cells;
  BandProb *d_chains, *d_cs, *d_gq;   // device descriptor arrays
  std::vector<BandProb> d_local_chains_host; BandProb* d_local_chains; int n_local_chains;   // chains of this rank's cells
  std::vector<BandProb> d_local_cs_host; BandProb* d_local_cs; int n_local_cs;
  std::vector<int> local_cells; int* d_local_cell_ids;
  double *gq_base; size_t gq_count;   // [tiles | rhs] of the boundary-separator system (all-reduced over ranks)
  double *spike_scratch; int* flags_base; size_t flags_count;
  // reduce ranges (multi-GPU): per cell, the accumulated tiles / ff of its two chains, owned by owner(c)
  struct Range { double* p; size_t n; int owner; };
  std::vector<Range> reduce_ranges; double* rhs_region; size_t rhs_count;
};
int band_plan_layout(BandPlan& P, int n, int bw, int ncell_request, int rank, int world);   // 0 = ok
int band_plan_partition(int n, int bw, int world, int* bounds);   // returns the number of cells
void band_plan_bind(BandPlan& P, double* dbase, int* ibase, void* desc_base, double* dp);
void band_plan_trim(BandPlan& P, const int* lo, const int* hi);   // [world] scalar position ranges the ranks' factors touch -> reduce_ranges
void band_set_tuning(int band_ctas_per_chain);
int launch_band_factor(const BandPlan& P, int* fail, cudaStream_t s);       // chains, cell separator systems, local part of the boundary system
int launch_band_top(const BandPlan& P, int* fail, cudaStream_t s);          // boundary system factor + solve, back-substitution, dp of the local cells
int launch_backsub_simple(const DevBlock& blk, const DevBand& B, double lambda, double* dl_point, int nl_stride,
                          double* dl_flow, int nf_stride, double* partials, cudaStream_t s);
int backsub_grid(int n_groups);
int launch_pose_model(const DevBlock& blk, const DevBand& B, double* partials, cudaStream_t s);
int launch_pose_delta_norm(const DevBand& B, double lambda, double* partials, cudaStream_t s);
int pose_norm_grid(int n);
int launch_retract(const DevVars& cur, const DevVars& cand, const DevBand& B, const double* dl_point,
                   const double* dl_flow, cudaStream_t s);
// ---- navigation variables and visual-inertial factors (kernels_imu.cu).  nav[i] = (solver position, dimension) of every
// velocity (3) and bias (6).
int nav_grid(int type, int n);      // partial sums a linearize / error launch of a navigation factor block writes
int launch_nav_linearize(const DevBlock& blk, const DevVars& v, double* partials, cudaStream_t s);
int launch_nav_error(const DevBlock& blk, const DevVars& v, double* partials, double* per_factor, cudaStream_t s);
int launch_nav_factors(const DevBlock& blk, const DevBand& B, cudaStream_t s);
int launch_nav_model(const DevBlock& blk, const DevBand& B, double* partials, cudaStream_t s);
int launch_nav_retract(const DevVars& cur, const DevVars& cand, const DevBand& B, const int2* nav, int n, cudaStream_t s);
int launch_nav_inert(const DevBand& B, const int2* nav, int n, cudaStream_t s);

// ---- per-frame batch entry points (kernels_star.cu, kernels_ransac.cu).  Per-device state kept between calls (these entry
// points run every frame): one stream and one grow-only workspace, so a call costs copies + one launch -- no cudaMalloc /
// cudaFree / stream creation on the per-frame path.  Calls on one device serialise on mu; dynoba_batch_release frees it.
struct StarContext { std::mutex mu; cudaStream_t stream = nullptr; char* base = nullptr; size_t cap = 0; };
StarContext& star_context(int device);          // device in [0, 64)
int star_device_ready(int device);              // sm_90 check, cudaSetDevice, stream creation (call with mu held)
// a bump allocator over the workspace, 16-byte granules; with base == nullptr it only measures
struct DeviceBlock {
  char* base = nullptr; size_t used = 0;
  template <class T> T* take(size_t count) { T* p = base ? (T*)(base + used) : nullptr; used += (count*sizeof(T) + 15) & ~(size_t)15; return p; }
  bool allocate(StarContext& c) {
    const size_t need = used + 256; used = 0;
    if (need > c.cap) {
      if (c.base) { cudaFree(c.base); c.base = nullptr; c.cap = 0; }
      const size_t cap = need + need/2;
      if (cudaMalloc((void**)&c.base, cap) != cudaSuccess) { c.base = nullptr; return false; }
      c.cap = cap;
    }
    base = c.base; return true;
  }
};

}  // namespace dynoba
