// frontend.cu -- libdynofront: front-end rows a13 / a14 of SURVEY.md section 8 as sm_90a kernels (include/dynofront.h).
// Compiled with -fmad=false: the KLT arithmetic follows OpenCV's scalar float code, which is not FMA-contracted.
//
// Ordering semantics that make the reference sequential are kept exactly:
//  * trackDynamic's cv::circle side effect on the detection mask makes acceptance of feature i depend on the
//    earlier accepted features (FeatureTracker.cc:385-392,472-482): resolved in parallel as a greedy independent
//    set over the "covers" relation, in rounds, inside one CTA;
//  * the tracking mask takes the label of the LAST accepted feature that covers a pixel: max-index-wins scatter;
//  * new tracklet ids are handed out in iteration order: prefix count over the accepted features;
//  * propogateMask processes objects one after the other, each vote seeing the previous object's writes.
#include <cuda_runtime.h>
#include <math_constants.h>
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/dynofront.h"
#include "boundary.cuh"

#define FCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return -3; } } while (0)

// A grow-only device array that owns its allocation.  Growing waits for the work queued on the stream (it may still read
// the old array), frees the old array and allocates the new one; when the array is large enough, ensure() does nothing, so
// the steady state neither synchronises nor frees.
template <class T> struct DevBuf {
  T* p = nullptr; size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~DevBuf() { cudaFree(p); }
  operator T*() const { return p; }
  cudaError_t ensure(size_t n, cudaStream_t s) {
    if (n <= cap) return cudaSuccess;
    if (p) {
      const cudaError_t e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) return e;
      cudaFree(p); p = nullptr; cap = 0;
    }
    const cudaError_t e = cudaMalloc((void**)&p, n*sizeof(T));
    if (e != cudaSuccess) { p = nullptr; return e; }
    cap = n; return cudaSuccess;
  }
};
// the counters of dynofront_detect_static; (anms_off, corners, K) is the one list anms_range_tree_kernel reads, anms its count
struct DetectCounters { int candidates, corners, anms_off, K, anms, unused, features; unsigned max_eig; };

struct dynofront_ctx {
  int dev = 0, W = 0, H = 0; cudaStream_t s = nullptr; std::string err; bool have_prev = false, have_cur = false, have_pyr = false, have_pyr_cur = false;
  DevBuf<float> flow; DevBuf<int32_t> mask; DevBuf<uint8_t> det; bool has_det = false;
  DevBuf<uint8_t> det_work, trk; DevBuf<int> trk_idx; bool det_work_valid = false;
  // feature scratch
  DevBuf<double> f_kp, f_pred, f_flow; DevBuf<int32_t> f_lab, f_age, f_oage, f_olab; DevBuf<int64_t> f_tid, f_otid;
  DevBuf<int> f_x, f_y, f_state, f_next, cell; DevBuf<uint8_t> f_acc; DevBuf<long long> nextid;
  // sampling scratch
  DevBuf<int> tile_cnt, obj_tot, d_objs, d_zero, d_idx;
  // propagate scratch
  DevBuf<int32_t> pmask, cmask; DevBuf<float> pflow; DevBuf<int> pflag, pm_votes;
  // KLT; der2: Scharr derivatives of the CURRENT image (backward pass)
  std::vector<DevBuf<uint8_t>> pyr[2]; std::vector<DevBuf<short>> der, der2; std::vector<int> lw, lh;
  DevBuf<float> k_prev, k_next, k_err, k_back, k_eig; DevBuf<uint8_t> k_st, k_st2, k_keep; DevBuf<int32_t> k_age; DevBuf<int> k_count;
  DevBuf<double> st_depth;                        // stereoTrack
  // stereo matching: pyramids of its own (0: a given left image, with st_der; 1: a given right image; 2: dynofront_set_right's),
  // never the temporal pair above; LK points, compaction (input row per rank, rank per row, compacted rows), offsets, counts
  std::vector<DevBuf<uint8_t>> st_pyr[3]; std::vector<DevBuf<short>> st_der; bool has_right = false;
  DevBuf<float> sm_left, sm_right, sm_cl, sm_cr; DevBuf<uint8_t> sm_st, sm_state; DevBuf<int> sm_idx, sm_rank, sm_off, sm_cnt;
  DevBuf<double> sm_depth, sm_ru;
  // external-flow static tracker scratch
  DevBuf<double> sf_kp, sf_flow, sf_pred; DevBuf<int32_t> sf_age, sf_det, sf_oage; DevBuf<uint8_t> sf_use, sf_pass, sf_acc;
  DevBuf<int> sf_cell, sf_win, sf_win2, sf_cnt; DevBuf<long long> sf_otid;
  // ANMS work arrays and lists, sampleDynamic selection scratch
  DevBuf<int> sel_xy, sel_px, sel_py, sel_orig, sel_next, sel_out, sel_off, sel_cnt, sel_k, sel_n; DevBuf<float> sel_tol;
  DevBuf<int> sd_idx, sd_ntrack, sd_counts; DevBuf<double> sd_kp, sd_flow, sd_pred; DevBuf<long long> sd_tid; DevBuf<int32_t> sd_lab;
  // static detection (dynofront_detect_static)
  DevBuf<uint8_t> dt_gray, dt_mask, dt_clahe, dt_lut; DevBuf<float> dt_dx, dt_dy, dt_box, dt_eig, dt_pts, dt_resp;
  DevBuf<unsigned long long> dt_keys; DevBuf<int> dt_corners; DevBuf<DetectCounters> dt_cnt;
  DevBuf<double> dt_kp; DevBuf<long long> dt_tid; bool dt_valid = false;
  // depth and back-projection: the current frame's depth image (stale after set_frame / next_frame until set_depth)
  DevBuf<double> depth; bool has_frame = false, has_depth = false;
  DevBuf<double> dp_kp, dp_depth, dp_right, dp_point, dp_stereo; DevBuf<int32_t> dp_lab, dp_index; DevBuf<uint8_t> dp_flag, dp_out; DevBuf<int> dp_cnt;
  DevBuf<float> dc_xyz; DevBuf<uint8_t> dc_rgb, dc_valid; DevBuf<uint32_t> dc_label;
  // homography RANSAC: inputs, point / inlier lists, outputs, per-problem statistics (6 arrays of hm_np) and per-iteration counts
  DevBuf<int> hm_off, hm_cidx, hm_lidx, hm_stat, hm_counts; DevBuf<float> hm_src, hm_dst; DevBuf<float4> hm_inl; DevBuf<double> hm_H; DevBuf<uint8_t> hm_mask;
  int hm_np = 0, hm_cap = 0, hm_record = 0;       // problems and recorded iterations of the last call; iterations to record
  // fundamental-matrix RANSAC: inputs, outputs, per-problem statistics (9 arrays of fm_np) and the per-iteration record
  DevBuf<int> fm_off, fm_stat; DevBuf<float> fm_src, fm_dst, fm_rec; DevBuf<double> fm_F; DevBuf<uint8_t> fm_mask;
  int fm_np = 0, fm_cap = 0, fm_record = 0;
  // trackDynamicKLT (also uses the trackDynamic, KLT, detection and ANMS scratch): status rows, counters, per-object lists (tk_int:
  // bb[4][64], K, cand, off, corners, selected), tracked sort keys, eigen image, GFTT corners, output features
  DevBuf<unsigned char> tk_rows, tk_cnt; DevBuf<int> tk_int, tk_corners; DevBuf<unsigned long long> tk_keys; DevBuf<float> tk_eig;
  DevBuf<double> tk_kp; DevBuf<int32_t> tk_age, tk_lab, tk_src; DevBuf<long long> tk_tid;
  // object boundary mask (dynofront_object_boundary): T, the boundary mask until it replaces det, the extent tables and their
  // pinned host copy; mask_propagated: dynofront_propagate_mask has modified the resident current motion mask since its upload
  DevBuf<uint8_t> bd_T, bd_mask; DevBuf<int> bd_tab; int* bd_host = nullptr; bool mask_propagated = false, bd_smem_set = false;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
};
// grows each (buffer, element count) pair in turn; 0, or -3 with the error at the first allocation that fails
static int grow(dynofront_ctx*) { return 0; }
template <class T, class... R> static int grow(dynofront_ctx* h, DevBuf<T>& b, size_t n, R&&... rest) {
  const cudaError_t e = b.ensure(n, h->s);
  if (e != cudaSuccess) { h->err = std::string("device allocation: ") + cudaGetErrorString(e); return -3; }
  return grow(h, rest...);
}
// feature arrays are sized for at least this many features, so that small changes of the count do not reallocate
static size_t feature_cap(int n) { return (size_t)std::max(n, 4096); }

// ---------------------------------------------------------------------------------------------------- trackDynamic
struct Disc { int r; int hw[16]; };   // half width of the filled cv::circle per |dy|
static Disc make_disc(int r) {       // OpenCV drawing.cpp Circle(): midpoint algorithm, filled spans
  Disc d; d.r = r; for (int i = 0; i < 16; i++) d.hw[i] = -1;
  int err = 0, dx = r, dy = 0, plus = 1, minus = (r << 1) - 1;
  while (dx >= dy) {
    d.hw[dy] = std::max(d.hw[dy], dx); d.hw[dx] = std::max(d.hw[dx], dy);
    dy++; err += plus; plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask; dx += mask; minus -= mask & 2;
  }
  return d;
}
// visits the pixels (x, y) of the filled disc around (cx, cy) that lie inside the W x H image, rows top to bottom, each row
// left to right; stops after the first pixel for which visit returns true
template <class F> __device__ __forceinline__ void disc_walk(const Disc& d, int cx, int cy, int W, int H, F visit) {
  for (int dy = -d.r; dy <= d.r; dy++) {
    const int yy = cy + dy; if (yy < 0 || yy >= H) continue;
    const int hw = d.hw[dy < 0 ? -dy : dy];
    for (int dx = -hw; dx <= hw; dx++) { const int xx = cx + dx; if (xx >= 0 && xx < W && visit(xx, yy)) return; }
  }
}
__device__ __forceinline__ bool within_shrunken(double kx, double ky, int rows, int cols, int sr, int sc) {
  const int pc = (int)kx, pr = (int)ky;     // static_cast<int>
  return pr > sr && pr < rows - sr && pc > sc && pc < cols - sc;
}

__global__ void td_candidate_kernel(int n, const double* __restrict__ kp, const int32_t* __restrict__ plab, const int32_t* __restrict__ page,
                                    const float* __restrict__ flow, const int32_t* __restrict__ mask, const uint8_t* __restrict__ det, int W, int H,
                                    dynofront_track_params prm, int* fx, int* fy, int* state, double* pred, double* oflow, int32_t* oage, int32_t* olab) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double kx = kp[2*i], ky = kp[2*i + 1];
  const int x = (int)kx, y = (int)ky;
  fx[i] = x; fy[i] = y;
  int st = 2;   // 0 unknown (candidate), 1 accepted, 2 rejected
  pred[2*i] = pred[2*i+1] = oflow[2*i] = oflow[2*i+1] = 0.0; oage[i] = 0; olab[i] = 0;
  if (x >= 0 && x < W && y >= 0 && y < H) {
    const int lab = mask[(size_t)y*W + x];
    const bool det_ok = det ? det[(size_t)y*W + x] != 0 : true;
    const bool contained = kx >= 0.0 && kx < (double)W && ky >= 0.0 && ky < (double)H;
    if (det_ok && contained && lab != 0 && lab == plab[i]) {
      const double fxe = (double)flow[2*((size_t)y*W + x)], fye = (double)flow[2*((size_t)y*W + x) + 1];
      const double px = kx + fxe, py = ky + fye;
      if (within_shrunken(px, py, H, W, prm.shrink_row, prm.shrink_col) && !(fxe == 0 || fye == 0)) {
        st = 0;
        pred[2*i] = px; pred[2*i+1] = py; oflow[2*i] = fxe; oflow[2*i+1] = fye;
        oage[i] = page[i] + 1; olab[i] = lab;
      }
    }
  }
  state[i] = st;
}
__global__ void td_link_kernel(int n, const int* fx, const int* fy, const int* state, int W, int* cell, int* next) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n || state[i] != 0) return;
  next[i] = atomicExch(&cell[(size_t)fy[i]*W + fx[i]], i);
}
// greedy resolution + tracklet ids, one CTA; a candidate covered by an earlier accepted one gets state `masked`
__global__ void __launch_bounds__(1024) td_resolve_kernel(int n, const int* fx, const int* fy, int* state, const int* cell, const int* next,
                                                          int W, int H, Disc disc, int max_age, const int64_t* ptid, int32_t* oage, int64_t* otid,
                                                          uint8_t* acc, long long* nextid, int masked) {
  __shared__ int remaining;
  for (;;) {
    if (threadIdx.x == 0) remaining = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      if (state[i] != 0) continue;
      bool any_acc = false, any_unknown = false;
      disc_walk(disc, fx[i], fy[i], W, H, [&](int xx, int yy) {
        for (int j = cell[(size_t)yy*W + xx]; j >= 0; j = next[j]) {
          if (j >= i) continue;
          const int sj = ((volatile int*)state)[j];
          if (sj == 1) { any_acc = true; break; }
          if (sj == 0) any_unknown = true;
        }
        return any_acc;
      });
      if (any_acc) state[i] = masked;
      else if (!any_unknown) state[i] = 1;
      else atomicAdd(&remaining, 1);
    }
    __syncthreads();
    if (remaining == 0) break;
    __syncthreads();
  }
  if (threadIdx.x == 0) {           // tracklet ids in iteration order (FeatureTracker.cc:446-450)
    long long id = *nextid;
    for (int i = 0; i < n; i++) {
      const bool a = state[i] == 1; acc[i] = a ? 1 : 0;
      if (!a) { oage[i] = 0; otid[i] = 0; continue; }
      if (oage[i] > max_age) { otid[i] = id++; oage[i] = 0; } else otid[i] = ptid[i];
    }
    *nextid = id;
  }
}
__global__ void td_clear_rejected_kernel(int n, const uint8_t* acc, double* pred, double* oflow, int32_t* olab) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n || acc[i]) return;
  pred[2*i] = pred[2*i+1] = oflow[2*i] = oflow[2*i+1] = 0.0; olab[i] = 0;
}
__global__ void td_masks_kernel(int n, const int* fx, const int* fy, const uint8_t* acc, int W, int H, Disc disc, uint8_t* det, int* trk_idx) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n || !acc[i]) return;
  disc_walk(disc, fx[i], fy[i], W, H, [&](int xx, int yy) {
    det[(size_t)yy*W + xx] = 0;
    atomicMax(&trk_idx[(size_t)yy*W + xx], i + 1);     // last writer (largest index) wins
    return false;
  });
}
__global__ void td_trk_final_kernel(size_t npx, const int* trk_idx, const int32_t* olab, uint8_t* trk) {
  const size_t p = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  if (p >= npx) return;
  const int t = trk_idx[p];
  const int l = t ? olab[t - 1] : 0;
  trk[p] = (uint8_t)(l < 0 ? 0 : l > 255 ? 255 : l);       // cv::Scalar(label) drawn into CV_8U saturates
}
__global__ void fill_u8_kernel(uint8_t* p, size_t n, uint8_t v) { const size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; if (i < n) p[i] = v; }
__global__ void fill_i32_kernel(int* p, size_t n, int v) { const size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; if (i < n) p[i] = v; }

// ---------------------------------------------------------------------------------------------------- sampleDynamic scan
constexpr int ST_TILE = 1024, ST_MAXOBJ = 64;
// the object list of a per-object entry point: at most ST_MAXOBJ ids, each > 0 and none twice (the reference's callers pass a
// std::set<ObjectId> of detected objects); checked before anything is launched
static int check_objects(dynofront_ctx* h, int n, const int32_t* objects) {
  if (n > ST_MAXOBJ) { h->err = "at most 64 objects"; return -1; }
  for (int o = 0; o < n; o++) {
    if (objects[o] <= 0) { h->err = "object ids must be > 0 (0 is the background)"; return -1; }
    for (int q = 0; q < o; q++) if (objects[q] == objects[o]) { h->err = "object ids must be distinct"; return -1; }
  }
  return 0;
}
__device__ __forceinline__ int sample_slot(size_t p, int W, int H, const uint8_t* det, const int32_t* mask, const float* flow, const int* objs, int nobj,
                                           dynofront_track_params prm, bool* zero) {
  *zero = false;
  if (det[p] == 0) return -1;
  const int lab = mask[p];
  int slot = -1;
  for (int o = 0; o < nobj; o++) if (objs[o] == lab) { slot = o; break; }
  if (slot < 0 || lab == 0) return -1;
  const double fx = (double)flow[2*p], fy = (double)flow[2*p + 1];
  if (fx == 0 || fy == 0) { *zero = true; return -(slot + 2); }
  const int i = (int)(p / W), j = (int)(p % W);
  if (!within_shrunken((double)j, (double)i, H, W, prm.shrink_row, prm.shrink_col)) return -1;
  return slot;
}
__global__ void __launch_bounds__(ST_TILE) sc_count_kernel(size_t npx, int W, int H, const uint8_t* det, const int32_t* mask, const float* flow,
                                                           const int* objs, int nobj, dynofront_track_params prm, int* tile_cnt, int* zero_cnt) {
  __shared__ int cnt[ST_MAXOBJ], zc[ST_MAXOBJ];
  if (threadIdx.x < ST_MAXOBJ) { cnt[threadIdx.x] = 0; zc[threadIdx.x] = 0; }
  __syncthreads();
  const size_t p = (size_t)blockIdx.x*ST_TILE + threadIdx.x;
  if (p < npx) {
    bool z; const int s = sample_slot(p, W, H, det, mask, flow, objs, nobj, prm, &z);
    if (s >= 0) atomicAdd(&cnt[s], 1); else if (z) atomicAdd(&zc[-s - 2], 1);
  }
  __syncthreads();
  if ((int)threadIdx.x < nobj) { tile_cnt[(size_t)blockIdx.x*ST_MAXOBJ + threadIdx.x] = cnt[threadIdx.x]; if (zc[threadIdx.x]) atomicAdd(&zero_cnt[threadIdx.x], zc[threadIdx.x]); }
}
__global__ void sc_scan_kernel(int ntiles, int nobj, int* tile_cnt, int* obj_tot) {
  const int o = threadIdx.x;
  if (o >= nobj) return;
  int run = 0;
  for (int t = 0; t < ntiles; t++) { const int c = tile_cnt[(size_t)t*ST_MAXOBJ + o]; tile_cnt[(size_t)t*ST_MAXOBJ + o] = run; run += c; }
  obj_tot[o] = run;
}
__global__ void __launch_bounds__(ST_TILE) sc_scatter_kernel(size_t npx, int W, int H, const uint8_t* det, const int32_t* mask, const float* flow,
                                                             const int* objs, int nobj, dynofront_track_params prm, const int* tile_off,
                                                             const int* obj_off, int* indices, long long capacity) {
  __shared__ int wc[32][ST_MAXOBJ];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t p = (size_t)blockIdx.x*ST_TILE + threadIdx.x;
  int s = -1;
  if (p < npx) { bool z; s = sample_slot(p, W, H, det, mask, flow, objs, nobj, prm, &z); if (s < 0) s = -1; }
  int myrank = 0;
  for (int o = 0; o < nobj; o++) {
    const unsigned b = __ballot_sync(0xffffffffu, s == o);
    if (lane == 0) wc[warp][o] = __popc(b);
    if (s == o) myrank = __popc(b & ((1u << lane) - 1));
  }
  __syncthreads();
  if (s >= 0) {
    int base = 0;
    for (int w = 0; w < warp; w++) base += wc[w][s];
    const long long dst = (long long)obj_off[s] + tile_off[(size_t)blockIdx.x*ST_MAXOBJ + s] + base + myrank;
    if (dst < capacity) indices[dst] = (int)p;
  }
}

// ---------------------------------------------------------------------------------------------------- ANMS (range tree)
// AdaptiveNonMaximumSuppression::suppressNonMax with AnmsAlgorithmType::RangeTree (NonMaximumSupression.cc:33-116,
// anms.cc:278-362), one CTA per key-point list, every list of a frame in one launch.
//  * Order.  Both call sites hand over responses that truncate to int 0, so cv::sortIdx(SORT_DESCENDING) sorts all-equal
//    keys: libstdc++'s introsort then yields a fixed permutation P_n of the input (equal_keys_sort_position).
//  * Width.  The reference's binary search over the square half-width w, with its quadratic-formula bounds, float
//    Kmin / Kmax and the fall-back to the last computed result (which can hold more than Kmax points).
//  * Greedy.  For one w, a point is kept when no earlier KEPT point lies in the inclusive square |dx| <= w, |dy| <= w.
//    Chunks of SEL_THREADS points are first tested in parallel against the points kept by earlier chunks (a bucket grid
//    in shared memory, cells >= w so a square touches <= 3x3 cells); the survivors of a chunk are then resolved in order
//    by one warp, 32 at a time: pairwise conflicts as a bit mask, a serial 32-step scan, insertion into the grid.
// Undefined inputs of the reference, defined here: K = 0 selects nothing (the reference converts +inf to int), K = 1
// selects the first point in processing order (the reference computes 0/0).
constexpr int SEL_THREADS = 256, SEL_GRID = 4096;
__device__ __forceinline__ int equal_keys_sort_position(int e, int n) {
  int pos = e, lo = 0, hi = n;
  while (hi - lo > 16) {                                   // std::__introsort_loop; depth never reaches 2*floor(log2 n)
    const int mid = lo + (hi - lo)/2;
    if (pos == lo) pos = mid; else if (pos == mid) pos = lo;   // __move_median_to_first, every comparison false: swap(first, mid)
    if (pos != lo) pos = lo + hi - pos;                        // __unguarded_partition: reverses [lo + 1, hi)
    const int cut = lo + 1 + (hi - lo - 1)/2;
    if (pos >= cut) lo = cut; else hi = cut;                   // recurse right, loop left (insertion sort moves nothing)
  }
  return n - 1 - pos;                                          // SORT_DESCENDING reverses the ascending result
}
// upper bound of the width search, anms.cc:282-297 in the reference's types (int / long long / double), K >= 2.  Every width
// tried is <= this, so key-points with coordinate + anms_high <= 65535 never reach the u16 wrap of rangetree<u16,u16>::search.
__host__ __device__ inline int anms_high(int K, int cols, int rows) {
  const int exp1 = rows + cols + 2*K;
  const long long exp2 = 4LL*cols + 4LL*K + 4LL*rows*K + (long long)rows*rows + (long long)cols*cols - 2LL*rows*cols + 4LL*rows*cols*K;
  const double exp3 = sqrt((double)exp2), exp4 = K - 1;
  const double sol1 = -round((exp1 + exp3)/exp4), sol2 = -round((exp1 - exp3)/exp4);
  return (int)(sol1 > sol2 ? sol1 : sol2);
}
// the reference's u16 range tree wraps coordinate + width above 65535: true when a list with K >= 2 whose largest coordinate
// is max_coord could reach that, so that the call is refused rather than answered differently
static bool anms_u16_wraps(long long max_coord, int K, int cols, int rows) {
  return max_coord + std::max(anms_high(K, cols, rows), 0) > 65535;
}
struct SelGrid { int x0, y0, s, nx, ny, w; };
// Two metrics share the ordered resolver: the range tree's inclusive square |dx|, |dy| <= w, and goodFeaturesToTrack's
// strict disc dx^2 + dy^2 < w^2 (its minDistance test).
template <bool EUCLID> __device__ __forceinline__ bool sel_near(int dx, int dy, int w) {
  return EUCLID ? dx*dx + dy*dy < w*w : (dx <= w && dx >= -w && dy <= w && dy >= -w);
}
template <bool EUCLID>
__device__ __forceinline__ bool sel_conflict(const SelGrid& g, const int* head, const int* px, const int* py, const int* nxt, int x, int y) {
  const int cx0 = max(x - g.w - g.x0, 0)/g.s, cx1 = min((x + g.w - g.x0)/g.s, g.nx - 1);
  const int cy0 = max(y - g.w - g.y0, 0)/g.s, cy1 = min((y + g.w - g.y0)/g.s, g.ny - 1);
  for (int cy = cy0; cy <= cy1; cy++)
    for (int cx = cx0; cx <= cx1; cx++)
      for (int q = head[cy*g.nx + cx]; q >= 0; q = nxt[q])
        if (sel_near<EUCLID>(px[q] - x, py[q] - y, g.w)) return true;
  return false;
}
// The ordered greedy of one CTA over points 0..n-1 of px / py: a point is kept when no earlier kept point is near it, and
// the pass stops once `limit` points are kept.  sel[0..) receives the kept positions in order; returns how many (the value
// is also in *s_kept, for every thread).
template <bool EUCLID>
__device__ int sel_greedy(const SelGrid& g, int n, int limit, const int* px, const int* py, int* nxt, int* sel, int* head, uint8_t* pend, int* s_kept) {
  const int tid = threadIdx.x, lane = tid & 31;
  for (int c = tid; c < g.nx*g.ny; c += SEL_THREADS) head[c] = -1;
  if (tid == 0) *s_kept = 0;
  __syncthreads();
  int kept = 0;                                                  // (warp 0's running count)
  for (int c0 = 0; c0 < n; c0 += SEL_THREADS) {
    const int i = c0 + tid;
    pend[tid] = (i < n && !sel_conflict<EUCLID>(g, head, px, py, nxt, px[i], py[i])) ? 1 : 0;
    __syncthreads();
    if (tid < 32) {
      for (int g0 = 0; g0 < SEL_THREADS && c0 + g0 < n && kept < limit; g0 += 32) {
        const int j = c0 + g0 + lane;
        bool p = j < n && pend[g0 + lane];
        if (!__any_sync(0xffffffffu, p)) continue;
        const int x = j < n ? px[j] : 0, y = j < n ? py[j] : 0;
        if (p && g0 > 0) p = !sel_conflict<EUCLID>(g, head, px, py, nxt, x, y);      // points kept earlier in this chunk
        const unsigned M = __ballot_sync(0xffffffffu, p);
        unsigned cm = 0;
        for (int b = 0; b < 32; b++) {
          const int xb = __shfl_sync(0xffffffffu, x, b), yb = __shfl_sync(0xffffffffu, y, b);
          if (b < lane && ((M >> b) & 1u) && sel_near<EUCLID>(xb - x, yb - y, g.w)) cm |= 1u << b;
        }
        unsigned km = 0;
        for (int b = 0; b < 32; b++) {
          const unsigned cb = __shfl_sync(0xffffffffu, cm, b);
          if (((M >> b) & 1u) && !(cb & km)) km |= 1u << b;
        }
        while (__popc(km) > limit - kept) km &= ~(1u << (31 - __clz(km)));     // the count limit: later points are not reached
        if ((km >> lane) & 1u) {
          sel[kept + __popc(km & ((1u << lane) - 1u))] = j;
          nxt[j] = atomicExch(&head[((y - g.y0)/g.s)*g.nx + (x - g.x0)/g.s], j);
        }
        kept += __popc(km);
        __syncwarp();
      }
      if (tid == 0) *s_kept = kept;
    }
    __syncthreads();
    if (*s_kept >= limit) break;
  }
  return *s_kept;
}
__host__ __device__ inline SelGrid sel_make_grid(int width, int bx0, int by0, int bx1, int by1) {
  SelGrid g; g.w = width; g.x0 = bx0; g.y0 = by0;
  const int bw = bx1 - bx0 + 1, bh = by1 - by0 + 1;
  g.s = max(max(width, 1), (int)sqrt((double)bw*bh/SEL_GRID));
  while ((long long)((bw + g.s - 1)/g.s)*((bh + g.s - 1)/g.s) > SEL_GRID) g.s++;
  g.nx = (bw + g.s - 1)/g.s; g.ny = (bh + g.s - 1)/g.s;
  return g;
}
// Points of list l: pixel (lin % W, lin / W) of lin[off + e] when lin is given, else xy[off + e].  Work arrays px / py /
// porig / nxt and the result sel are indexed like the input (off + position).  sel[off + r] = index within the list of
// the r-th selected point, nsel[l] = how many (never more than the list holds).
__global__ void __launch_bounds__(SEL_THREADS, 1) anms_range_tree_kernel(const int* __restrict__ off, const int* __restrict__ cnt, const int* __restrict__ kneed,
                                                                      const float* __restrict__ tol, float tol_all, const int* __restrict__ lin,
                                                                      const int* __restrict__ xy, int W, int cols, int rows,
                                                                      int* px, int* py, int* porig, int* nxt, int* sel, int* __restrict__ nsel) {
  __shared__ int head[SEL_GRID];
  __shared__ uint8_t pend[SEL_THREADS];
  __shared__ int s_bb[4], s_kept, s_width, s_stop, s_done;   // (two flags: no thread rewrites one that a slow warp may still read)
  __shared__ SelGrid s_g;
  const int l = blockIdx.x, o = off[l], n = cnt[l], K = kneed[l], tid = threadIdx.x;
  if (n <= 0 || K <= 0) { if (tid == 0) nsel[l] = 0; return; }
  px += o; py += o; porig += o; nxt += o; sel += o;
  if (tid == 0) { s_bb[0] = s_bb[1] = 0x7fffffff; s_bb[2] = s_bb[3] = -1; }
  __syncthreads();
  int bx0 = 0x7fffffff, by0 = 0x7fffffff, bx1 = -1, by1 = -1;
  for (int e = tid; e < n; e += SEL_THREADS) {
    int x, y;
    if (lin) { const int p = lin[o + e]; x = p % W; y = p / W; } else { x = xy[2*(o + e)]; y = xy[2*(o + e) + 1]; }
    const int k = equal_keys_sort_position(e, n);
    px[k] = x; py[k] = y; porig[k] = e;
    bx0 = min(bx0, x); by0 = min(by0, y); bx1 = max(bx1, x); by1 = max(by1, y);
  }
  atomicMin(&s_bb[0], bx0); atomicMin(&s_bb[1], by0); atomicMax(&s_bb[2], bx1); atomicMax(&s_bb[3], by1);
  __syncthreads();
  if (K == 1) { if (tid == 0) { sel[0] = porig[0]; nsel[l] = 1; } return; }
  // anms.cc:282-310, same types: int / long long / double, float Kmin / Kmax
  int low = 0, high = 0, prevwidth = -1; unsigned Kmin = 0, Kmax = 0;
  if (tid == 0) {
    high = anms_high(K, cols, rows);
    low = (int)floor(sqrt((double)n/K));
    const float t = tol ? tol[l] : tol_all, Kf = (float)(unsigned)K;
    Kmin = (unsigned)roundf(Kf - Kf*t); Kmax = (unsigned)roundf(Kf + Kf*t);
    s_kept = 0;
  }
  for (;;) {
    if (tid == 0) {
      const int width = low + (high - low)/2;
      s_stop = (width == prevwidth || low > high) ? 1 : 0;         // keep the last computed result
      if (!s_stop) { s_g = sel_make_grid(width, s_bb[0], s_bb[1], s_bb[2], s_bb[3]); s_width = width; }
    }
    __syncthreads();
    if (s_stop) break;
    sel_greedy<false>(s_g, n, 0x7fffffff, px, py, nxt, sel, head, pend, &s_kept);
    if (tid == 0) {                                                // anms.cc:347-354
      const unsigned r = (unsigned)s_kept;
      s_done = 0;
      if (r >= Kmin && r <= Kmax) s_done = 1;
      else if (r < Kmin) high = s_width - 1;
      else low = s_width + 1;
      prevwidth = s_width;
    }
    __syncthreads();
    if (s_done) break;
  }
  const int m = s_kept;
  for (int r = tid; r < m; r += SEL_THREADS) sel[r] = porig[sel[r]];
  if (tid == 0) nsel[l] = m;
}

// sampleDynamic after ANMS (FeatureTracker.cc:955-1015): list offsets and the number of corners needed per object
__global__ void sd_prepare_kernel(int nobj, const int* tot, const int* num_track, int max_features, int* off, int* kneed) {
  if (threadIdx.x != 0) return;
  int run = 0;
  for (int o = 0; o < nobj; o++) { off[o] = run; run += tot[o]; kneed[o] = max(max_features - num_track[o], 0); }
}
// one CTA per object: the selected candidate pixels become features, packed object after object in the given order
__global__ void sd_construct_kernel(const int* __restrict__ off, const int* __restrict__ nsel, const int* __restrict__ sel, const int* __restrict__ idx,
                                    const float* __restrict__ flow, int W, const int* __restrict__ objs, long long base_id, double* __restrict__ okp,
                                    double* __restrict__ oflow, double* __restrict__ opred, long long* __restrict__ otid, int32_t* __restrict__ olab) {
  const int o = blockIdx.x;
  int base = 0;
  for (int q = 0; q < o; q++) base += nsel[q];
  for (int r = threadIdx.x; r < nsel[o]; r += blockDim.x) {
    const int p = idx[off[o] + sel[off[o] + r]], x = p % W, y = p / W, d = base + r;
    const double fx = (double)flow[2*(size_t)p], fy = (double)flow[2*(size_t)p + 1];
    okp[2*(size_t)d] = x; okp[2*(size_t)d + 1] = y; oflow[2*(size_t)d] = fx; oflow[2*(size_t)d + 1] = fy;
    opred[2*(size_t)d] = x + fx; opred[2*(size_t)d + 1] = y + fy;     // Feature::CalculatePredictedKeypoint
    otid[d] = base_id + d; olab[d] = objs[o];
  }
}

// ---------------------------------------------------------------------------------------------------- propogateMask
// The vote of one object is sorted[0] of std::sort(pairs, a.second > b.second) over the (label, count) pairs of a
// std::map<int, int>, i.e. in ascending label order.  pm_introsort_loop restates libstdc++'s __introsort_loop (<bits/stl_algo.h>:
// threshold 16, depth limit 2 floor(log2 n), median of three moved to the front, unguarded partition, heap sort at the depth
// limit).  The final insertion sort that follows it is stable, so sorted[0] is the first pair of largest count after the loop.
struct PmPair { int l, c; };
__device__ void pm_adjust_heap(PmPair* a, int hole, int len, PmPair v) {       // __adjust_heap + __push_heap
  const int top = hole;
  int child = hole;
  while (child < (len - 1)/2) {
    child = 2*(child + 1);
    if (a[child].c > a[child - 1].c) child--;
    a[hole] = a[child]; hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2)/2) { child = 2*(child + 1); a[hole] = a[child - 1]; hole = child - 1; }
  int parent = (hole - 1)/2;
  while (hole > top && a[parent].c > v.c) { a[hole] = a[parent]; hole = parent; parent = (hole - 1)/2; }
  a[hole] = v;
}
__device__ void pm_heap_sort(PmPair* a, int len) {                            // __partial_sort(first, last, last): make_heap, sort_heap
  for (int parent = (len - 2)/2; len >= 2; parent--) { pm_adjust_heap(a, parent, len, a[parent]); if (parent == 0) break; }
  for (int last = len - 1; last > 0; last--) { const PmPair v = a[last]; a[last] = a[0]; pm_adjust_heap(a, 0, last, v); }
}
__device__ int pm_partition_pivot(PmPair* a, int first, int last) {           // __unguarded_partition_pivot
  const int x = first + 1, y = first + (last - first)/2, z = last - 1;
  int m;
  if (a[x].c > a[y].c) m = a[y].c > a[z].c ? y : a[x].c > a[z].c ? z : x;
  else m = a[x].c > a[z].c ? x : a[y].c > a[z].c ? z : y;
  PmPair t = a[first]; a[first] = a[m]; a[m] = t;
  const int pc = a[first].c;
  int i = first + 1, j = last;
  for (;;) {
    while (a[i].c > pc) i++;
    j--;
    while (pc > a[j].c) j--;
    if (!(i < j)) return i;
    t = a[i]; a[i] = a[j]; a[j] = t;
    i++;
  }
}
__device__ void pm_introsort_loop(PmPair* a, int n) {
  // ranges still to sort; the depths on the stack fall strictly from bottom to top, so it holds at most 2*31 + 1 entries
  struct Range { int first, last, depth; } st[64];
  int top = 0;
  if (n > 1) st[top++] = Range{0, n, 2*(31 - __clz(n))};
  while (top) {
    Range r = st[--top];
    while (r.last - r.first > 16) {
      if (r.depth == 0) { pm_heap_sort(a + r.first, r.last - r.first); break; }
      r.depth--;
      const int cut = pm_partition_pivot(a, r.first, r.last);
      st[top++] = Range{cut, r.last, r.depth};
      r.last = cut;
    }
  }
}
// one CTA: the votes (current-mask labels under the object's predicted key-points, any int32) are counted into (label, count)
// pairs in ascending label order, labels in [0, 256) in a shared histogram, the others gathered into votes (n ints) and sorted;
// *flag = 1 when there are >= min_votes votes and sorted[0] is label 0.  pairs holds n pairs.
constexpr int PM_THREADS = 256, PM_SMEM = 2048;
__global__ void __launch_bounds__(PM_THREADS) pm_vote_kernel(int n, const double* kp, const int32_t* lab, int label, const int32_t* cur, int W, int H,
                                                             int min_votes, int* votes, PmPair* pairs, int* flag) {
  static_assert(PM_THREADS == 256, "one histogram bin per thread");
  __shared__ int hist[256]; __shared__ int s_v[PM_SMEM]; __shared__ int s_total, s_out, s_max, s_best;
  hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) { s_total = 0; s_out = 0; s_max = 0; s_best = 256; }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += PM_THREADS) {
    if (lab[i] != label) continue;
    const int u = (int)kp[2*i], v = (int)kp[2*i + 1];
    if (u < W && u > 0 && v < H && v > 0) {
      const int l = cur[(size_t)v*W + u];
      atomicAdd(&s_total, 1);
      if (l >= 0 && l < 256) atomicAdd(&hist[l], 1); else votes[atomicAdd(&s_out, 1)] = l;
    }
  }
  __syncthreads();
  const int c = hist[threadIdx.x], m = s_out, total = s_total;
  const int np_hist = __syncthreads_count(c > 0);
  if (total == 0 || total < min_votes) { if (threadIdx.x == 0) *flag = 0; return; }
  if (m == 0 && np_hist <= 16) {                   // std::sort of <= 16 pairs is an insertion sort: the first maximum in label order
    if (c > 0) atomicMax(&s_max, c);
    __syncthreads();
    if (c > 0 && c == s_max) atomicMin(&s_best, (int)threadIdx.x);
    __syncthreads();
    if (threadIdx.x == 0) *flag = s_best == 0 ? 1 : 0;
    return;
  }
  int* v = votes;
  if (m <= PM_SMEM) {
    for (int i = threadIdx.x; i < m; i += PM_THREADS) s_v[i] = votes[i];
    v = s_v;
    __syncthreads();
  }
  unsigned N = 1;
  while (N < (unsigned)m) N <<= 1;
  for (unsigned k = 2; k <= N; k <<= 1) {          // bitonic sort, every compare-exchange ascending: the padding up to N is +inf
    for (unsigned j = k >> 1; j > 0; j >>= 1) {
      for (unsigned i = threadIdx.x; i < N; i += PM_THREADS) {
        const unsigned l = j == k >> 1 ? i ^ (k - 1) : i ^ j;
        if (l > i && l < (unsigned)m) { const int a = v[i], b = v[l]; if (a > b) { v[i] = b; v[l] = a; } }
      }
      __syncthreads();
    }
  }
  if (threadIdx.x != 0) return;
  int np = 0, i = 0;
  auto runs = [&](bool negative) {                 // the sorted votes outside [0, 256): the negative ones, then those >= 256
    int run = 0;
    for (; i < m && (v[i] < 0) == negative; i++) {
      run++;
      if (i == m - 1 || v[i + 1] != v[i]) { pairs[np++] = PmPair{v[i], run}; run = 0; }
    }
  };
  runs(true);
  for (int l = 0; l < 256; l++) if (hist[l]) pairs[np++] = PmPair{l, hist[l]};
  runs(false);
  pm_introsort_loop(pairs, np);
  int best = 0;
  for (int q = 1; q < np; q++) if (pairs[q].c > pairs[best].c) best = q;
  *flag = pairs[best].l == 0 ? 1 : 0;
}
__global__ void pm_warp_kernel(size_t npx, int W, int H, const int32_t* pmask, const float* pflow, int label, dynofront_track_params prm,
                               const int* flag, int32_t* cur) {
  if (*flag == 0) return;
  const size_t p = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  if (p >= npx || pmask[p] != label) return;
  const double fx = (double)pflow[2*p], fy = (double)pflow[2*p + 1];
  if (fx == 0 || fy == 0) return;
  const int j = (int)(p / W), k = (int)(p % W);
  const double px = k + fx, py = j + fy;
  if (!within_shrunken(px, py, H, W, prm.shrink_row, prm.shrink_col)) return;
  if (px < W && px > 0 && py < H && py > 0) cur[(size_t)((int)py)*W + (int)px] = label;
}

// ---------------------------------------------------------------------------------------------------- pyramidal KLT
__device__ __forceinline__ int reflect101(int i, int n) { if (i < 0) i = -i; if (i >= n) i = 2*n - 2 - i; return i; }
__global__ void pyr_down_kernel(const uint8_t* __restrict__ src, int sw, int sh, uint8_t* __restrict__ dst, int dw, int dh) {
  const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  const int k[5] = { 1, 4, 6, 4, 1 };
  int sum = 0;
  for (int j = -2; j <= 2; j++) {
    const int yy = reflect101(2*y + j, sh);
    int row = 0;
    for (int i = -2; i <= 2; i++) row += k[i + 2]*src[(size_t)yy*sw + reflect101(2*x + i, sw)];
    sum += k[j + 2]*row;
  }
  dst[(size_t)y*dw + x] = (uint8_t)((sum + 128) >> 8);
}
__global__ void scharr_kernel(const uint8_t* __restrict__ src, int w, int h, short* __restrict__ dst) {
  const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int y0 = y > 0 ? y - 1 : (h > 1 ? 1 : 0), y2 = y < h - 1 ? y + 1 : (h > 1 ? h - 2 : 0);
  const int xm = x > 0 ? x - 1 : (w > 1 ? 1 : 0), xp = x < w - 1 ? x + 1 : (w > 1 ? w - 2 : 0);
  auto t0 = [&](int xx) { return (src[(size_t)y0*w + xx] + src[(size_t)y2*w + xx])*3 + src[(size_t)y*w + xx]*10; };
  auto t1 = [&](int xx) { return (int)src[(size_t)y2*w + xx] - (int)src[(size_t)y0*w + xx]; };
  dst[2*((size_t)y*w + x)] = (short)(t0(xp) - t0(xm));
  dst[2*((size_t)y*w + x) + 1] = (short)((t1(xp) + t1(xm))*3 + t1(x)*10);
}

struct KltLevels { const uint8_t* I[8]; const uint8_t* J[8]; const short* D[8]; int w[8], h[8]; int nlev; };
constexpr int KLT_WARPS = 4, KLT_MAXWIN = 31;
#define DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))

__device__ __forceinline__ int img_at(const uint8_t* I, int w, int h, int x, int y) { return I[(size_t)reflect101(y, h)*w + reflect101(x, w)]; }
__device__ __forceinline__ int der_at(const short* D, int w, int h, int x, int y, int c) { return (x < 0 || x >= w || y < 0 || y >= h) ? 0 : D[2*((size_t)y*w + x) + c]; }

__global__ void __launch_bounds__(KLT_WARPS*32) klt_kernel(KltLevels L, int n, const float* __restrict__ prevPts, float* __restrict__ nextPts,
                                                           uint8_t* __restrict__ status, float* __restrict__ err, int win, int maxCount, float eps2,
                                                           int use_initial, float minEigThreshold, float* __restrict__ eig_out) {
  extern __shared__ short ksm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pt = blockIdx.x*KLT_WARPS + warp;
  if (pt >= n) return;
  const int area = win*win;
  short* Ipatch = ksm + (size_t)warp*area*3; short* dI = Ipatch + area;
  const float halfWin = (win - 1)*0.5f;
  const float px0 = prevPts[2*pt], py0 = prevPts[2*pt + 1];
  float nx = nextPts[2*pt], ny = nextPts[2*pt + 1];
  bool st = true; float e = 0.f;
  for (int level = L.nlev - 1; level >= 0; level--) {
    const int w = L.w[level], h = L.h[level];
    const float sc = (float)(1.0/(1 << level));
    float ppx = px0*sc, ppy = py0*sc;
    if (level == L.nlev - 1) { if (use_initial) { nx = nx*sc; ny = ny*sc; } else { nx = ppx; ny = ppy; } }
    else { nx = nx*2.f; ny = ny*2.f; }
    ppx -= halfWin; ppy -= halfWin;
    const int ipx = (int)floorf(ppx), ipy = (int)floorf(ppy);
    if (ipx < -win || ipx >= w || ipy < -win || ipy >= h) { if (level == 0) { st = false; e = 0.f; } continue; }
    float a = ppx - ipx, b = ppy - ipy;
    int iw00 = __float2int_rn((1.f - a)*(1.f - b)*16384.f), iw01 = __float2int_rn(a*(1.f - b)*16384.f),
        iw10 = __float2int_rn((1.f - a)*b*16384.f), iw11 = 16384 - iw00 - iw01 - iw10;
    long long sA11 = 0, sA12 = 0, sA22 = 0;
    for (int q = lane; q < area; q += 32) {
      const int y = q/win, x = q - y*win, gx = ipx + x, gy = ipy + y;
      const int ival = DESCALE(img_at(L.I[level], w, h, gx, gy)*iw00 + img_at(L.I[level], w, h, gx + 1, gy)*iw01 +
                               img_at(L.I[level], w, h, gx, gy + 1)*iw10 + img_at(L.I[level], w, h, gx + 1, gy + 1)*iw11, 9);
      const int ixv = DESCALE(der_at(L.D[level], w, h, gx, gy, 0)*iw00 + der_at(L.D[level], w, h, gx + 1, gy, 0)*iw01 +
                              der_at(L.D[level], w, h, gx, gy + 1, 0)*iw10 + der_at(L.D[level], w, h, gx + 1, gy + 1, 0)*iw11, 14);
      const int iyv = DESCALE(der_at(L.D[level], w, h, gx, gy, 1)*iw00 + der_at(L.D[level], w, h, gx + 1, gy, 1)*iw01 +
                              der_at(L.D[level], w, h, gx, gy + 1, 1)*iw10 + der_at(L.D[level], w, h, gx + 1, gy + 1, 1)*iw11, 14);
      Ipatch[q] = (short)ival; dI[2*q] = (short)ixv; dI[2*q + 1] = (short)iyv;
      sA11 += (long long)ixv*ixv; sA12 += (long long)ixv*iyv; sA22 += (long long)iyv*iyv;
    }
    for (int o = 16; o > 0; o >>= 1) { sA11 += __shfl_xor_sync(0xffffffffu, sA11, o); sA12 += __shfl_xor_sync(0xffffffffu, sA12, o); sA22 += __shfl_xor_sync(0xffffffffu, sA22, o); }
    __syncwarp();
    const float FLT_SCALE = 1.f/(1 << 20);
    const float A11 = (float)sA11*FLT_SCALE, A12 = (float)sA12*FLT_SCALE, A22 = (float)sA22*FLT_SCALE;
    float D = A11*A22 - A12*A12;
    const float minEig = (A22 + A11 - sqrtf((A11 - A22)*(A11 - A22) + 4.f*A12*A12))/(2*win*win);
    if (eig_out && level == 0 && lane == 0) { eig_out[2*pt] = minEig; eig_out[2*pt + 1] = (A11 + A22)/(2*win*win); }
    if (minEig < minEigThreshold || D < 1.1920929e-07f) { if (level == 0) st = false; continue; }
    D = 1.f/D;
    nx -= halfWin; ny -= halfWin;
    float pdx = 0.f, pdy = 0.f;
    float outx = nx + halfWin, outy = ny + halfWin;
    for (int j = 0; j < maxCount; j++) {
      const int inx = (int)floorf(nx), iny = (int)floorf(ny);
      if (inx < -win || inx >= w || iny < -win || iny >= h) { if (level == 0) st = false; break; }
      a = nx - inx; b = ny - iny;
      iw00 = __float2int_rn((1.f - a)*(1.f - b)*16384.f); iw01 = __float2int_rn(a*(1.f - b)*16384.f);
      iw10 = __float2int_rn((1.f - a)*b*16384.f); iw11 = 16384 - iw00 - iw01 - iw10;
      long long sb1 = 0, sb2 = 0;
      for (int q = lane; q < area; q += 32) {
        const int y = q/win, x = q - y*win, gx = inx + x, gy = iny + y;
        const int diff = DESCALE(img_at(L.J[level], w, h, gx, gy)*iw00 + img_at(L.J[level], w, h, gx + 1, gy)*iw01 +
                                 img_at(L.J[level], w, h, gx, gy + 1)*iw10 + img_at(L.J[level], w, h, gx + 1, gy + 1)*iw11, 9) - Ipatch[q];
        sb1 += (long long)diff*dI[2*q]; sb2 += (long long)diff*dI[2*q + 1];
      }
      for (int o = 16; o > 0; o >>= 1) { sb1 += __shfl_xor_sync(0xffffffffu, sb1, o); sb2 += __shfl_xor_sync(0xffffffffu, sb2, o); }
      const float b1 = (float)sb1*FLT_SCALE, b2 = (float)sb2*FLT_SCALE;
      const float dx = (A12*b2 - A22*b1)*D, dy = (A12*b1 - A11*b2)*D;
      nx += dx; ny += dy;
      outx = nx + halfWin; outy = ny + halfWin;
      if (dx*dx + dy*dy <= eps2) break;
      if (j > 0 && fabsf(dx + pdx) < 0.01f && fabsf(dy + pdy) < 0.01f) { outx -= dx*0.5f; outy -= dy*0.5f; break; }
      pdx = dx; pdy = dy;
    }
    nx = outx; ny = outy;
    if (st && level == 0) {     // residual error of the final position (status can still flip here)
      const float fx = nx - halfWin, fy = ny - halfWin;
      const int inx = (int)floorf(fx), iny = (int)floorf(fy);
      if (inx < -win || inx >= w || iny < -win || iny >= h) st = false;
      else {
        const float aa = fx - inx, bb = fy - iny;
        iw00 = __float2int_rn((1.f - aa)*(1.f - bb)*16384.f); iw01 = __float2int_rn(aa*(1.f - bb)*16384.f);
        iw10 = __float2int_rn((1.f - aa)*bb*16384.f); iw11 = 16384 - iw00 - iw01 - iw10;
        long long se = 0;
        for (int q = lane; q < area; q += 32) {
          const int y = q/win, x = q - y*win, gx = inx + x, gy = iny + y;
          const int diff = DESCALE(img_at(L.J[0], w, h, gx, gy)*iw00 + img_at(L.J[0], w, h, gx + 1, gy)*iw01 +
                                   img_at(L.J[0], w, h, gx, gy + 1)*iw10 + img_at(L.J[0], w, h, gx + 1, gy + 1)*iw11, 9) - Ipatch[q];
          se += diff < 0 ? -diff : diff;
        }
        for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
        e = (float)se*(1.f/(32*win*win));
      }
    }
  }
  if (lane == 0) { nextPts[2*pt] = nx; nextPts[2*pt + 1] = ny; status[pt] = st ? 1 : 0; if (err) err[pt] = e; }
}

// ---------------------------------------------------------------------------------------------------- forward-backward KLT
// KltFeatureTracker::trackPoints after the two cv::calcOpticalFlowPyrLK calls (StaticFeatureTracker.cc:505-534): a track
// survives when both passes succeeded and the backward pass returns to within 0.5 px of where it started (float
// arithmetic, as the reference's lambda), then the per-point checks of :575-592 / :628-646 -- background label at the
// truncated key-point, inside the image and the shrunken image, age + 1 <= max_feature_track_age.
__global__ void klt_fb_filter_kernel(int n, const float* __restrict__ prev, const float* __restrict__ next, const float* __restrict__ back,
                                     const uint8_t* __restrict__ st_f, const uint8_t* __restrict__ st_b, float max_dist, uint8_t* __restrict__ status,
                                     int check, const int32_t* __restrict__ mask, int W, int H, dynofront_track_params prm, const int32_t* __restrict__ age,
                                     int max_age, uint8_t* __restrict__ keep, int* __restrict__ count) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float dx = prev[2*i] - back[2*i], dy = prev[2*i + 1] - back[2*i + 1];
  const bool ok = st_f[i] && st_b[i] && sqrtf(dx*dx + dy*dy) <= max_dist;
  status[i] = ok ? 1 : 0;
  bool k = ok;
  if (check && ok) {
    const double kx = (double)next[2*i], ky = (double)next[2*i + 1];
    const int x = (int)kx, y = (int)ky;                                       // functional_keypoint::u / v: truncation
    const bool contained = kx >= 0.0 && kx < (double)W && ky >= 0.0 && ky < (double)H;
    const bool shrunk = y > prm.shrink_row && y < H - prm.shrink_row && x > prm.shrink_col && x < W - prm.shrink_col;
    k = contained && shrunk && mask[(size_t)y*W + x] == 0 && age[i] + 1 <= max_age;
  }
  keep[i] = k ? 1 : 0;
  if (ok) atomicAdd(count, 1);
  if (k) atomicAdd(count + 1, 1);
}
__global__ void count_status_kernel(int n, const uint8_t* st, int* count) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i < n && st[i]) atomicAdd(count, 1);
}

// ---------------------------------------------------------------------------------------------------- external-flow static tracker
// ExternalFlowFeatureTracker::trackStatic / constructStaticFeature (StaticFeatureTracker.cc:70-220).  The reference walks
// the previous features in order and the FIRST one that passes every check claims its grid cell (cells are only marked by
// successful constructions): in parallel, the passing feature with the smallest index per cell wins (atomicMin).  New
// detections do the same among the cells the tracked features left free, in detection order, until the frame holds
// max_features (a prefix count); tracklet ids are handed out in that order.
// feature i: flow and predicted key-point at oflow[2i] / pred[2i]
__device__ __forceinline__ bool sf_construct(const float* flow, const int32_t* mask, int W, int H, int x, int y, double kx, double ky, int i,
                                             double* oflow, double* pred) {
  if (mask[(size_t)y*W + x] != 0) return false;
  const double fx = (double)flow[2*((size_t)y*W + x)], fy = (double)flow[2*((size_t)y*W + x) + 1];
  if (!(fx != 0 && fy != 0)) return false;
  const double px = kx + fx, py = ky + fy;
  if (!(px >= 0.0 && px < (double)W && py >= 0.0 && py < (double)H)) return false;
  oflow[2*(size_t)i] = fx; oflow[2*(size_t)i + 1] = fy; pred[2*(size_t)i] = px; pred[2*(size_t)i + 1] = py;
  return true;
}
__device__ __forceinline__ void sf_clear(int i, double* oflow, double* pred) {
  oflow[2*(size_t)i] = oflow[2*(size_t)i + 1] = pred[2*(size_t)i] = pred[2*(size_t)i + 1] = 0.0;
}
__global__ void sf_prev_kernel(int n, const double* __restrict__ kp, const uint8_t* __restrict__ usable, const float* flow, const int32_t* mask, int W, int H,
                               int cell_size, int ncols, int* __restrict__ cell, uint8_t* __restrict__ pass, double* __restrict__ oflow,
                               double* __restrict__ pred, int* __restrict__ win) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double kx = kp[2*i], ky = kp[2*i + 1];
  pass[i] = 0; cell[i] = -1;
  if (!(kx >= 0.0 && kx < (double)W && ky >= 0.0 && ky < (double)H)) return;
  const int x = (int)kx, y = (int)ky;
  const int c = (int)floor(ky/cell_size)*ncols + (int)floor(kx/cell_size);
  cell[i] = c;
  if (!usable[i]) return;
  if (!sf_construct(flow, mask, W, H, x, y, kx, ky, i, oflow, pred)) return;
  pass[i] = 1;
  atomicMin(win + c, i);
}
__global__ void sf_prev_resolve_kernel(int n, const int* cell, const uint8_t* pass, const int* win, const int32_t* age, uint8_t* acc, double* oflow,
                                       double* pred, int32_t* oage, int* cnt) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool a = pass[i] && win[cell[i]] == i;
  acc[i] = a ? 1 : 0; oage[i] = a ? age[i] + 1 : 0;
  if (!a) sf_clear(i, oflow, pred);
  else atomicAdd(cnt, 1);
}
__global__ void sf_det_kernel(int n, const int32_t* __restrict__ xy, const float* flow, const int32_t* mask, int W, int H, int cell_size, int ncols,
                              const int* __restrict__ win_prev, int* __restrict__ cell, uint8_t* __restrict__ pass, double* __restrict__ oflow,
                              double* __restrict__ pred, int* __restrict__ win) {
  const int j = blockIdx.x*blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int x = xy[2*j], y = xy[2*j + 1];
  pass[j] = 0; cell[j] = -1;
  if (x < 0 || x >= W || y < 0 || y >= H) return;
  if (mask[(size_t)y*W + x] != 0) return;
  const int c = (int)floor((double)y/cell_size)*ncols + (int)floor((double)x/cell_size);
  cell[j] = c;
  if (win_prev[c] != 0x7fffffff) return;                       // cell taken by a tracked feature
  if (!sf_construct(flow, mask, W, H, x, y, (double)x, (double)y, j, oflow, pred)) return;
  pass[j] = 1;
  atomicMin(win + c, j);
}
// In-order compaction inside one CTA of 1024 threads that walks a list in 1024-wide chunks, every thread calling this once
// per chunk: returns how many flags before this thread's are set, in this chunk and the earlier ones, and adds the chunk's
// flags to the running count `base` (the same in every thread).
__device__ __forceinline__ int cta_rank(int flag, int& base) {
  __shared__ int s_scan[1024];
  s_scan[threadIdx.x] = flag;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) { const int v = threadIdx.x >= o ? s_scan[threadIdx.x - o] : 0; __syncthreads(); s_scan[threadIdx.x] += v; __syncthreads(); }
  const int rank = base + s_scan[threadIdx.x] - flag;
  base += s_scan[1023];
  __syncthreads();
  return rank;
}
// one CTA: in-order prefix count of the accepted detections, truncated at `room`; tracklet ids follow the order
__global__ void __launch_bounds__(1024) sf_det_resolve_kernel(int n, const int* cell, const uint8_t* pass, const int* win, const int* cnt_prev, int max_features,
                                                              long long base_id, uint8_t* acc, double* oflow, double* pred, long long* otid, int* cnt_det) {
  const int room = max(0, max_features - *cnt_prev);
  int base = 0;
  for (int j0 = 0; j0 < n; j0 += 1024) {
    const int j = j0 + threadIdx.x;
    const int a = (j < n && pass[j] && win[cell[j]] == j) ? 1 : 0;
    const int rank = cta_rank(a, base);                          // accepted detections before j
    if (j < n) {
      const bool fin = a && rank < room;
      acc[j] = fin ? 1 : 0; otid[j] = fin ? base_id + rank : 0;
      if (!fin) sf_clear(j, oflow, pred);
    }
  }
  if (threadIdx.x == 0) *cnt_det = min(base, room);
}

// ---------------------------------------------------------------------------------------------------- KltFeatureTracker::detectFeatures
// StaticFeatureTracker.cc:330-418 and SparseFeatureDetector::detect (FeatureDetector.cc:187-239) with the CPU OpenCV routines
// they call (TrackerParams defaults: cv::GFTTDetector, not cv::cuda's).  Every float result reproduces cv2 bit for bit; the
// orders below were pinned against it (opencv-python 4.x on x86-64 with AVX2 dispatch):
//  * CLAHE: tiles on the BORDER_REFLECT_101-extended image when W or H is not a multiple of 8 (both sides are then padded by
//    8 - side % 8), clip max(int(2.0 * area / 256), 1), tile coordinates as y * (1.f / tile_h) - 0.5f;
//  * Sobel (scale 1 / (4 * 3 * 255) folded into the smoothing tap): the x derivative is fma(r[-1] + r[+1], s, r[0] * 2s) over
//    the exact row differences; the y derivative's row pass is the SIMD fma chain for x < (W / 32) * 32 and the scalar
//    sequential sum on the remaining columns, then the exact column difference;
//  * the unnormalised 3x3 box sum of the products: rows as (c[-1] + c[0]) + c[+1] in double, then a running double sum that
//    slides down each column (add the entering row, subtract the leaving one), rounded to float;
//  * (a + c) - sqrt((a - c)^2 + b^2) in float without FMA.
constexpr int DT_SORT_TILE = 2048, DT_TILES = 8;
__device__ __forceinline__ uint32_t f32_order(float v) { const uint32_t u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float f32_unorder(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

// detection mask: the caller's boundary mask (255 without one) AND background, then a filled cv::circle of radius r around
// every current feature, centred on cvRound of the float key-point (cv::Point2f -> cv::Point: round half to even)
__global__ void dt_mask_kernel(size_t npx, const uint8_t* __restrict__ det, const int32_t* __restrict__ mask, uint8_t* __restrict__ out) {
  const size_t p = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  if (p < npx) out[p] = (mask[p] == 0) ? (det ? det[p] : 255) : 0;
}
__global__ void dt_circles_kernel(int n, const double* __restrict__ kp, Disc disc, int W, int H, uint8_t* out) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int cx = __float2int_rn((float)kp[2*i]), cy = __float2int_rn((float)kp[2*i + 1]);
  disc_walk(disc, cx, cy, W, H, [&](int xx, int yy) { out[(size_t)yy*W + xx] = 0; return false; });
}
// CLAHE(2.0, 8x8), one CTA per tile: histogram, clip, redistribution, LUT (clahe.cpp CLAHE_CalcLut_Body)
__global__ void __launch_bounds__(256) clahe_lut_kernel(const uint8_t* __restrict__ img, int W, int H, int tw, int th, int clip, float lut_scale,
                                                        uint8_t* __restrict__ lut) {
  __shared__ int hist[256];
  const int tx = blockIdx.x, ty = blockIdx.y;
  hist[threadIdx.x] = 0;
  __syncthreads();
  for (int q = threadIdx.x; q < tw*th; q += blockDim.x) {
    int x = tx*tw + q % tw, y = ty*th + q / tw;
    if (x >= W) x = 2*W - 2 - x;                                 // the BORDER_REFLECT_101 extension (right / bottom only)
    if (y >= H) y = 2*H - 2 - y;
    atomicAdd(&hist[img[(size_t)y*W + x]], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (clip > 0) {
      int clipped = 0;
      for (int i = 0; i < 256; i++) if (hist[i] > clip) { clipped += hist[i] - clip; hist[i] = clip; }
      const int batch = clipped/256; int residual = clipped - batch*256;
      for (int i = 0; i < 256; i++) hist[i] += batch;
      if (residual != 0) { const int step = max(256/residual, 1); for (int i = 0; i < 256 && residual > 0; i += step, residual--) hist[i]++; }
    }
    int sum = 0; uint8_t* L = lut + (ty*DT_TILES + tx)*256;
    for (int i = 0; i < 256; i++) { sum += hist[i]; L[i] = (uint8_t)min(max(__float2int_rn((float)sum*lut_scale), 0), 255); }
  }
}
__global__ void clahe_apply_kernel(const uint8_t* __restrict__ img, int W, int H, float inv_tw, float inv_th, const uint8_t* __restrict__ lut,
                                   uint8_t* __restrict__ out) {
  const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const float tyf = (float)y*inv_th - 0.5f, txf = (float)x*inv_tw - 0.5f;
  int ty1 = (int)floorf(tyf), ty2 = ty1 + 1, tx1 = (int)floorf(txf), tx2 = tx1 + 1;
  const float ya = tyf - (float)ty1, ya1 = 1.0f - ya, xa = txf - (float)tx1, xa1 = 1.0f - xa;
  ty1 = max(ty1, 0); ty2 = min(ty2, DT_TILES - 1); tx1 = max(tx1, 0); tx2 = min(tx2, DT_TILES - 1);
  const int v = img[(size_t)y*W + x];
  const uint8_t *L1 = lut + ty1*DT_TILES*256, *L2 = lut + ty2*DT_TILES*256;
  const float res = ((float)L1[tx1*256 + v]*xa1 + (float)L1[tx2*256 + v]*xa)*ya1 + ((float)L2[tx1*256 + v]*xa1 + (float)L2[tx2*256 + v]*xa)*ya;
  out[(size_t)y*W + x] = (uint8_t)min(max(__float2int_rn(res), 0), 255);
}
// Sobel 3x3 of cornerEigenValsVecs (see the orders above)
__global__ void dt_sobel_kernel(const uint8_t* __restrict__ img, int W, int H, float* __restrict__ dx, float* __restrict__ dy) {
  const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const double s = 1.0/(4*3*255.0);
  const float f1 = (float)s, f0 = (float)(2*s);
  const int xm = reflect101(x - 1, W), xp = reflect101(x + 1, W), ym = reflect101(y - 1, H), yp = reflect101(y + 1, H);
  auto at = [&](int yy, int xx) { return (float)img[(size_t)yy*W + xx]; };
  auto rd = [&](int yy) { return at(yy, xp) - at(yy, xm); };
  const bool simd = x < (W/32)*32;
  auto rs = [&](int yy) { const float L = at(yy, xm), M = at(yy, x), R = at(yy, xp);
    return simd ? __fmaf_rn(R, f1, __fmaf_rn(M, f0, L*f1)) : (f1*L + f0*M) + f1*R; };
  dx[(size_t)y*W + x] = __fmaf_rn(rd(ym) + rd(yp), f1, rd(y)*f0);
  dy[(size_t)y*W + x] = rs(yp) - rs(ym);
}
// the unnormalised 3x3 box sum of one product channel (0: Ix Ix, 1: Ix Iy, 2: Iy Iy), one thread per (column, channel)
// sliding down the column as ColumnSum<double, float> does; box is [3][H][W]
__global__ void __launch_bounds__(32) dt_box_kernel(const float* __restrict__ dx, const float* __restrict__ dy, int W, int H, float* __restrict__ box) {
  const int t = blockIdx.x*blockDim.x + threadIdx.x;
  if (t >= 3*W) return;
  const int c = t / W, x = t - c*W;
  const int xm = reflect101(x - 1, W), xp = reflect101(x + 1, W);
  const float* U = c == 2 ? dy : dx; const float* V = c == 0 ? dx : dy;
  auto row = [&](int yy) {
    const size_t r = (size_t)reflect101(yy, H)*W;
    return ((double)(U[r + xm]*V[r + xm]) + (double)(U[r + x]*V[r + x])) + (double)(U[r + xp]*V[r + xp]);
  };
  float* out = box + (size_t)c*W*H + x;
  double rm = row(-1), r0 = row(0), rp = row(1), S = (0.0 + rm) + r0;
  for (int y = 0; y < H; y++) {
    const double rn = y + 2 <= H ? row(y + 2) : 0.0;            // the next row is loaded while this one is summed
    const double s0 = S + rp;
    out[(size_t)y*W] = (float)s0; S = s0 - rm;
    rm = r0; r0 = rp; rp = rn;
  }
}
// the minimum eigenvalue per pixel and the maximum of the eigen image under the detection mask (minMaxLoc), as an
// order-preserving u32
__global__ void dt_eig_kernel(const float* __restrict__ box, size_t npx, const uint8_t* __restrict__ mask, float* __restrict__ eig, unsigned* __restrict__ maxv) {
  const size_t p = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  uint32_t best = 0;
  if (p < npx) {
    const float a = box[p]*0.5f, b = box[npx + p], cc = box[2*npx + p]*0.5f;
    const float e = (a + cc) - sqrtf((a - cc)*(a - cc) + b*b);
    eig[p] = e;
    if (mask[p]) best = f32_order(e);
  }
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best) atomicMax(maxv, best);
}
// goodFeaturesToTrack candidates: THRESH_TOZERO at (float)(maxVal * quality), 3x3 local maxima (dilate) that are non-zero
// and inside the mask, the 1-px border excluded.  Key = value (order-preserving) << 32 | pixel address, sorted descending:
// greaterThanPtr (larger value first, ties: larger address first).
__global__ void dt_cand_kernel(const float* __restrict__ eig, int W, int H, const uint8_t* __restrict__ mask, const unsigned* __restrict__ maxv,
                               double quality, unsigned long long* __restrict__ keys, int* __restrict__ count) {
  const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
  if (x < 1 || y < 1 || x >= W - 1 || y >= H - 1) return;
  const float mx = *maxv ? f32_unorder(*maxv) : 0.f;             // minMaxLoc over an empty mask leaves maxVal = 0
  const float thr = (float)((double)mx*quality);
  auto tz = [&](int xx, int yy) { const float v = eig[(size_t)yy*W + xx]; return v > thr ? v : 0.f; };
  const float v = tz(x, y);
  if (v == 0.f || !mask[(size_t)y*W + x]) return;
  float d = v;
  for (int j = -1; j <= 1; j++) for (int i = -1; i <= 1; i++) d = fmaxf(d, tz(x + i, y + j));
  if (v != d) return;
  const int k = atomicAdd(count, 1);
  keys[k] = ((unsigned long long)f32_order(v) << 32) | (unsigned)(y*W + x);
}
// bitonic sort (descending) of keys[0 .. npad), npad = max(next power of two >= *count, DT_SORT_TILE); every launch reads the
// count on the device and the stages above npad return at once, so the host plans for the largest size without a readback
__device__ __forceinline__ int dt_npad(const int* count) { int n = DT_SORT_TILE; while (n < *count) n <<= 1; return n; }
__global__ void dt_sort_pad_kernel(unsigned long long* keys, const int* count, int cap) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x, n = dt_npad(count);
  if (i >= *count && i < n && i < cap) keys[i] = 0ull;
}
__device__ __forceinline__ void dt_cmpx(unsigned long long* a, unsigned long long* b, bool desc) {
  const unsigned long long x = *a, y = *b;
  if ((x < y) == desc) { *a = y; *b = x; }
}
__global__ void __launch_bounds__(DT_SORT_TILE/2) dt_sort_local_kernel(unsigned long long* keys, const int* count, int k_first, int k_last) {
  __shared__ unsigned long long s[DT_SORT_TILE];
  const int n = dt_npad(count), base = blockIdx.x*DT_SORT_TILE;
  if (base >= n || k_last > n) return;
  s[threadIdx.x] = keys[base + threadIdx.x]; s[threadIdx.x + DT_SORT_TILE/2] = keys[base + threadIdx.x + DT_SORT_TILE/2];
  __syncthreads();
  for (int k = k_first; k <= k_last; k <<= 1)
    for (int j = min(k, DT_SORT_TILE)/2; j > 0; j >>= 1) {
      const int t = threadIdx.x, i = (t/j)*2*j + (t % j);
      dt_cmpx(&s[i], &s[i + j], ((base + i) & k) == 0);
      __syncthreads();
    }
  keys[base + threadIdx.x] = s[threadIdx.x]; keys[base + threadIdx.x + DT_SORT_TILE/2] = s[threadIdx.x + DT_SORT_TILE/2];
}
__global__ void dt_sort_global_kernel(unsigned long long* keys, const int* count, int k, int j) {
  const int n = dt_npad(count), t = blockIdx.x*blockDim.x + threadIdx.x;
  if (k > n || t >= n/2) return;
  const int i = (t/j)*2*j + (t % j);
  dt_cmpx(&keys[i], &keys[i + j], (i & k) == 0);
}
// the greedy minDistance filter with the maxCorners stop (goodFeaturesToTrack), one CTA per sorted key list, through the
// ordered resolver of the ANMS with the strict Euclidean metric.  List l is keys[off[l] .. off[l] + count[l]) (one list at 0
// without off); the pixel address is key & addr_mask.  corners[2*(off[l] + c)] = (x, y) in output order, n_corners[l]; resp
// (may be NULL) = the first value of a key whose value sits in the upper 32 bits.
__global__ void __launch_bounds__(SEL_THREADS, 1) dt_gftt_select_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ off,
                                                                      const int* __restrict__ count, unsigned addr_mask, int W, int H,
                                                                      int min_dist, int max_corners, int* px, int* py, int* nxt, int* sel,
                                                                      int* __restrict__ corners, int* __restrict__ n_corners, float* __restrict__ resp) {
  __shared__ int head[SEL_GRID];
  __shared__ uint8_t pend[SEL_THREADS];
  __shared__ int s_kept;
  __shared__ SelGrid s_g;
  const int l = blockIdx.x, o = off ? off[l] : 0, n = count[l], tid = threadIdx.x;
  if (n == 0) { if (tid == 0) { n_corners[l] = 0; if (resp) *resp = 0.f; } return; }
  keys += o; px += o; py += o; nxt += o; sel += o; corners += 2*(size_t)o;
  for (int e = tid; e < n; e += SEL_THREADS) { const unsigned a = (unsigned)keys[e] & addr_mask; px[e] = (int)(a % W); py[e] = (int)(a / W); }
  if (tid == 0) s_g = sel_make_grid(min_dist, 0, 0, W - 1, H - 1);
  __syncthreads();
  const int m = sel_greedy<true>(s_g, n, max_corners > 0 ? max_corners : 0x7fffffff, px, py, nxt, sel, head, pend, &s_kept);
  for (int r = tid; r < m; r += SEL_THREADS) { corners[2*r] = px[sel[r]]; corners[2*r + 1] = py[sel[r]]; }
  if (tid == 0) { n_corners[l] = m; if (resp) *resp = f32_unorder((unsigned)(keys[0] >> 32)); }
}
// cv::getRectSubPix(img, 13x13, centre, CV_32F) as cornerSubPix calls it.  Inside the image: the four float weights, summed
// as (p a11 + q a12) + (u a21 + v a22); near the border: adjustRect's clamped rectangle (columns outside the image repeat
// the vertical interpolation of the edge column, rows outside repeat the edge row), which gives cv2's values up to the last
// bit of some entries (cv2 runs Intel IPP there; DESIGN section 4).
constexpr int SP_WIN = 5, SP_W = 2*SP_WIN + 1, SP_P = SP_W + 2;
struct SubpixMask { float m[SP_W*SP_W]; };
__device__ void dt_rect_subpix(const uint8_t* __restrict__ img, int W, int H, float cx0, float cy0, float* patch) {
  const float cx = cx0 - (SP_P - 1)*0.5f, cy = cy0 - (SP_P - 1)*0.5f;
  const int ix = (int)floorf(cx), iy = (int)floorf(cy);
  const float a = cx - (float)ix, b = cy - (float)iy;
  const float a11 = (1.f - a)*(1.f - b), a12 = a*(1.f - b), a21 = (1.f - a)*b, a22 = a*b, b1 = 1.f - b, b2 = b;
  auto px = [&](int y, int x) { return (float)img[(size_t)y*W + x]; };
  if (0 <= ix && ix < W - SP_P && 0 <= iy && iy < H - SP_P) {
    for (int i = 0; i < SP_P; i++)
      for (int j = 0; j < SP_P; j++)
        patch[i*SP_P + j] = (px(iy + i, ix + j)*a11 + px(iy + i, ix + j + 1)*a12) + (px(iy + i + 1, ix + j)*a21 + px(iy + i + 1, ix + j + 1)*a22);
    return;
  }
  int col = 0, row = 0, rx, rw, ry, rh;                          // adjustRect (imgwarp.cpp)
  if (ix >= 0) { col += ix; rx = 0; } else { rx = min(-ix, SP_P); }
  if (ix < W - SP_P) rw = SP_P; else { rw = W - ix - 1; if (rw < 0) { col += rw; rw = 0; } }
  if (iy >= 0) { row += iy; ry = 0; } else ry = -iy;
  if (iy < H - SP_P) rh = SP_P; else { rh = H - iy - 1; if (rh < 0) { row += rh; rh = 0; } }
  col -= rx;
  for (int i = 0; i < SP_P; i++) {
    int r2 = row + 1;
    if (i < ry || i >= rh) r2 -= 1;
    // rows above the image that are cut on the right repeat column W - 2, not W - 1 (what cv2's getRectSubPix returns there)
    const int cr = (i < ry && rw < SP_P) ? col + rw - 1 : col + rw;
    const float s0 = px(row, col + rx)*b1 + px(r2, col + rx)*b2, s1 = px(row, cr)*b1 + px(r2, cr)*b2;
    for (int j = 0; j < rx; j++) patch[i*SP_P + j] = s0;
    for (int j = rw; j < SP_P; j++) patch[i*SP_P + j] = s1;
    for (int j = rx; j < rw; j++) {
      const float p = px(row, col + j), q = px(row, col + j + 1);
      patch[i*SP_P + j] = r2 != row ? (p*a11 + q*a12) + (px(r2, col + j)*a21 + px(r2, col + j + 1)*a22) : p*(1.f - a) + q*a;
    }
    if (i < rh) row = r2;
  }
}
// cv::cornerSubPix(img, pts, (5,5), (-1,-1), EPS+COUNT): one thread per point, OpenCV's sequential double sums over the
// 11x11 window (the eps^2 test sees them, so their order is kept), the det <= DBL_EPSILON^2 and leave-the-image breaks, and
// the reset to the start when the point moved more than the window.  The Gaussian weights come from the host (std::exp).
// Point r is corner sel[r] (corner r without ANMS, sel == NULL), r < *cnt.
__global__ void dt_subpix_kernel(int m, const int* __restrict__ corners, const int* __restrict__ sel, const int* __restrict__ cnt,
                                 const uint8_t* __restrict__ img, int W, int H, SubpixMask mask, int max_iters, double eps2, float* __restrict__ pts) {
  const int r = blockIdx.x*blockDim.x + threadIdx.x;
  if (r >= m || r >= *cnt) return;
  const int c = sel ? sel[r] : r;
  const float tx = (float)corners[2*c], ty = (float)corners[2*c + 1];
  float ix = tx, iy = ty;
  float patch[SP_P*SP_P];
  int iter = 0; double err = 0;
  do {
    dt_rect_subpix(img, W, H, ix, iy, patch);
    double a = 0, b = 0, cc = 0, bb1 = 0, bb2 = 0;
    for (int i = 0, k = 0; i < SP_W; i++) {
      const double py = i - SP_WIN;
      const float* sp = patch + (i + 1)*SP_P + 1;
      for (int j = 0; j < SP_W; j++, k++) {
        const double mk = mask.m[k];
        const double tgx = sp[j + 1] - sp[j - 1], tgy = sp[j + SP_P] - sp[j - SP_P];
        const double gxx = tgx*tgx*mk, gxy = tgx*tgy*mk, gyy = tgy*tgy*mk, pxd = j - SP_WIN;
        a += gxx; b += gxy; cc += gyy;
        bb1 += gxx*pxd + gxy*py; bb2 += gxy*pxd + gyy*py;
      }
    }
    const double det = a*cc - b*b;
    if (fabs(det) <= 2.220446049250313e-16*2.220446049250313e-16) break;
    const double scale = 1.0/det;
    const float nx = (float)(ix + cc*scale*bb1 - b*scale*bb2), ny = (float)(iy - b*scale*bb1 + a*scale*bb2);
    err = (nx - ix)*(nx - ix) + (ny - iy)*(ny - iy);
    ix = nx; iy = ny;
    if (ix < 0 || ix >= W || iy < 0 || iy >= H) break;
  } while (++iter < max_iters && err > eps2);
  if (fabsf(ix - tx) > SP_WIN || fabsf(iy - ty) > SP_WIN) { ix = tx; iy = ty; }
  pts[2*r] = ix; pts[2*r + 1] = iy;
}
// the detected points in ANMS order become features (StaticFeatureTracker.cc:393-415): contained, inside the shrunken
// image, background at the truncated pixel; in-order prefix count, tracklet ids from base_id in that order.  One CTA.
__global__ void __launch_bounds__(1024) dt_construct_kernel(const float* __restrict__ pts, const int* __restrict__ cnt, const int32_t* __restrict__ mask,
                                                            int W, int H, dynofront_track_params prm, long long base_id, double* __restrict__ kp,
                                                            long long* __restrict__ tid, int* __restrict__ n_out) {
  const int n = *cnt;
  int base = 0;
  for (int j0 = 0; j0 < n; j0 += 1024) {
    const int j = j0 + threadIdx.x;
    double kx = 0, ky = 0; int a = 0;
    if (j < n) {
      kx = (double)pts[2*j]; ky = (double)pts[2*j + 1];
      const bool contained = kx >= 0.0 && kx < (double)W && ky >= 0.0 && ky < (double)H;
      a = (contained && within_shrunken(kx, ky, H, W, prm.shrink_row, prm.shrink_col) && mask[(size_t)((int)ky)*W + (int)kx] == 0) ? 1 : 0;
    }
    const int rank = cta_rank(a, base);
    if (a) { kp[2*(size_t)rank] = kx; kp[2*(size_t)rank + 1] = ky; tid[rank] = base_id + rank; }
  }
  if (threadIdx.x == 0) *n_out = base;
}
// the points cornerSubPix would refine when it is off: the integer corners as floats, in selection order
__global__ void dt_points_kernel(int m, const int* __restrict__ corners, const int* __restrict__ sel, const int* __restrict__ cnt, float* __restrict__ pts) {
  const int r = blockIdx.x*blockDim.x + threadIdx.x;
  if (r >= m || r >= *cnt) return;
  const int c = sel ? sel[r] : r;
  pts[2*r] = (float)corners[2*c]; pts[2*r + 1] = (float)corners[2*c + 1];
}

// ---------------------------------------------------------------------------------------------------- depth and back-projection
// Frame::updateDepths (Frame.cc:241-251,430-467), the per-feature half of RGBDInstanceFrontendModule::fillOutputPacketWithTracks
// (:391-486) and Frame::projectToDenseCloud (Frame.cc:172-238).  The camera is gtsam::PinholeCamera<Cal3_S2> at the identity
// pose (Camera.cc:39-46), calib = fx fy s u0 v0.  Every double / float operation below is one IEEE operation in the order of
// the reference (the library is built with -fmad=false, so nothing is contracted into an FMA).
struct Calib5 { double fx, fy, s, u0, v0; };
struct Pose12 { double m[12]; };     // row-major R, then t
// Cal3_S2::calibrate in GTSAM 4.2's operation order, then PinholeBase::BackprojectFromCamera (x d, y d, d)
__device__ __forceinline__ void backproject_cam(const Calib5& K, double u, double v, double d, double* p) {
  const double du = u - K.u0, dv = v - K.v0;
  const double inv_fx = 1.0/K.fx, inv_fy = 1.0/K.fy;
  const double ify_dv = inv_fy*dv;
  const double x = inv_fx*(du - K.s*ify_dv), y = ify_dv;
  p[0] = x*d; p[1] = y*d; p[2] = d;
}
// Pose3::transformFrom: q_i = ((R_i0 p0 + R_i1 p1) + R_i2 p2) + t_i
__device__ __forceinline__ void transform_from(const Pose12& X, double* p) {
  double q[3];
  for (int r = 0; r < 3; r++) q[r] = ((X.m[3*r]*p[0] + X.m[3*r + 1]*p[1]) + X.m[3*r + 2]*p[2]) + X.m[9 + r];
  p[0] = q[0]; p[1] = q[1]; p[2] = q[2];
}
// Color::uniqueId(size_t(label), 0.5f, 0.95f) (Colour.cc:178-185) through Color::fromHSV / rgbFromChromaHue (:73-100), with
// the reference's mix of float and double: fmod(float, int) and the terms around it are double, x is rounded to float
__device__ __forceinline__ void unique_id_rgb(int32_t label, uint8_t* rgb) {
  const float phi = (float)((1.0 + sqrt(5.0))/2.0);
  const float t = (float)(unsigned long long)(long long)label*phi;
  const float n = t - floorf(t);
  float hue = (float)(floor((double)n*256.0)/255.0);
  hue = fminf(fmaxf(hue, 0.0f), 1.0f);
  const float value = 0.95f, chroma = value*0.5f;
  const float hp = hue*6.0f;
  const float x = (float)((double)chroma*(1.0 - fabs(fmod((double)hp, 2.0) - 1.0)));
  float r1 = chroma, g1 = 0.0f, b1 = x;
  if (hp < 1.0f) { r1 = chroma; g1 = x; b1 = 0.0f; }
  else if (hp < 2.0f) { r1 = x; g1 = chroma; b1 = 0.0f; }
  else if (hp < 3.0f) { r1 = 0.0f; g1 = chroma; b1 = x; }
  else if (hp < 4.0f) { r1 = 0.0f; g1 = x; b1 = chroma; }
  else if (hp < 5.0f) { r1 = x; g1 = 0.0f; b1 = chroma; }
  const float m = value - chroma;
  rgb[0] = (uint8_t)((r1 + m)*255.0f); rgb[1] = (uint8_t)((g1 + m)*255.0f); rgb[2] = (uint8_t)((b1 + m)*255.0f);
}
// updateDepthsFeatureContainer: d = depth(int(v), int(u)); invalid (NaN depth) when d > max || d <= 0, so a NaN depth stays
// valid without depth.  A truncated pixel outside the image (undefined in the reference) is invalid with NaN depth; the test
// -1 < u < W is the truncation test without converting an out-of-range double to int.  cnt[0] invalid, cnt[1] outside.
__global__ void ud_kernel(int n, const double* __restrict__ kp, const int32_t* __restrict__ lab, const double* __restrict__ depth, int W, int H,
                          double max_bg, double max_obj, double* __restrict__ dout, uint8_t* __restrict__ valid, int* cnt) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double kx = kp[2*i], ky = kp[2*i + 1];
  const bool inside = kx > -1.0 && kx < (double)W && ky > -1.0 && ky < (double)H;
  const double mx = lab[i] == 0 ? max_bg : max_obj;
  const double d = inside ? depth[(size_t)(int)ky*W + (int)kx] : 0.0;
  const bool ok = inside && !(d > mx || d <= 0.0);
  dout[i] = ok ? d : CUDART_NAN;
  valid[i] = ok ? 1 : 0;
  if (!ok) atomicAdd(&cnt[0], 1);
  if (!inside) atomicAdd(&cnt[1], 1);
}
// fill_camera_measurements over the usable features in input order, one CTA: landmark when the depth is not NaN (hasDepth),
// stereo (uL, uR, v) from the given right key-point, else with rgbd and depth uR = uL - fx b / d, an outlier (dropped) when
// uR < 0 || uR > W.  Emitted measurements are compacted in input order; the first `capacity` are written, *m counts all.
__global__ void __launch_bounds__(1024) bp_kernel(int n, const double* __restrict__ kp, const double* __restrict__ depth, const uint8_t* __restrict__ usable,
                                                  const double* __restrict__ right_u, Calib5 K, double fx_b, int rgbd, int W, Pose12 X, int use_X, int capacity,
                                                  int32_t* index, double* point, double* stereo, uint8_t* outlier, int* m) {
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    int emit = 0; uint8_t out = 0;
    double p[3] = {CUDART_NAN, CUDART_NAN, CUDART_NAN}, st[3] = {CUDART_NAN, CUDART_NAN, CUDART_NAN};
    if (i < n && usable[i]) {
      const double u = kp[2*i], v = kp[2*i + 1], d = depth[i];
      const bool has_depth = !isnan(d);
      if (has_depth) { backproject_cam(K, u, v, d, p); if (use_X) transform_from(X, p); }
      const double ur_given = right_u ? right_u[i] : CUDART_NAN;
      if (!isnan(ur_given)) { st[0] = u; st[1] = ur_given; st[2] = v; }
      else if (rgbd && has_depth) {
        const double ur = u - fx_b/d;
        if (ur < 0.0 || ur > (double)W) out = 1;
        else { st[0] = u; st[1] = ur; st[2] = v; }
      }
      emit = !out;
    }
    if (i < n) outlier[i] = out;
    const int rank = cta_rank(emit, base);
    if (emit && rank < capacity) {
      index[rank] = i;
      for (int c = 0; c < 3; c++) { point[3*(size_t)rank + c] = p[c]; stereo[3*(size_t)rank + c] = st[c]; }
    }
  }
  if (threadIdx.x == 0) *m = base;
}
// projectToDenseCloud, one thread per pixel: pixels outside the boundary mask, or with depth > thresh || depth <= 0 || !finite
// (thresh by background / object label) are zero; the others hold the camera-frame point rounded to float, black (background)
// or Color::uniqueId(label), the label and valid = 1.  *count = number of valid pixels.
__global__ void dc_kernel(size_t npx, int W, const double* __restrict__ depth, const int32_t* __restrict__ mask, const uint8_t* __restrict__ det,
                          Calib5 K, double max_bg, double max_obj, float* xyz, uint8_t* rgb, uint32_t* label, uint8_t* valid, int* count) {
  const size_t p = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  bool ok = false;
  if (p < npx) {
    float q[3] = {0.f, 0.f, 0.f}; uint8_t c[3] = {0, 0, 0}; uint32_t l = 0;
    if (!det || det[p] != 0) {
      const int32_t oid = mask[p]; const double d = depth[p];
      const double thresh = oid == 0 ? max_bg : max_obj;
      if (!(d > thresh || d <= 0.0 || !isfinite(d))) {
        double pt[3];
        backproject_cam(K, (double)(int)(p % W), (double)(int)(p / W), d, pt);
        q[0] = (float)pt[0]; q[1] = (float)pt[1]; q[2] = (float)pt[2];
        if (oid != 0) unique_id_rgb(oid, c);
        l = (uint32_t)oid; ok = true;
      }
    }
    for (int k = 0; k < 3; k++) { xyz[3*p + k] = q[k]; rgb[3*p + k] = c[k]; }
    label[p] = l; valid[p] = ok ? 1 : 0;
  }
  const int nv = __syncthreads_count(ok);
  if (threadIdx.x == 0 && nv) atomicAdd(count, nv);
}

// ---------------------------------------------------------------------------------------------------- homography RANSAC
// cv::findHomography(src, dst, RANSAC, thr, mask, max_iters, confidence) as KltFeatureTracker::geometricVerification calls it
// (StaticFeatureTracker.cc:627-639), one persistent CTA per problem.  OpenCV's orders, pinned against cv2 by tests/test_homography.py
// (tests/homography_oracle.py restates them):
//  * draws: cv::RNG((uint64)-1) (multiply-with-carry), uniform(0, n) = next() % n, groups of 4 distinct indices with duplicates
//    re-drawn at once.  The split of the stream into groups does not depend on the subset test, so one lane cuts a chunk of
//    groups and the subset tests and 4-point models run in parallel, one thread per group;
//  * an iteration takes groups until one passes checkSubset; 10 000 rejections in a row end the loop (fail it in iteration 0);
//  * model: runKernel (centroid / mean absolute deviation normalisation, LtL summed in point order, OpenCV's Jacobi, the
//    eigenvector of the smallest eigenvalue, invHnorm * H0 * Hnorm2, times 1 / H22); error in float with H cast to float;
//  * thread 0 replays the sequential best-model / RANSACUpdateNumIters loop over each chunk's counts, so nothing depends on the
//    chunk size (32, 64, 128, then 256 groups);
//  * after RANSAC: in-order compaction of the inliers, runKernel over them (each of the 4 centroid / deviation sums and the 45 LtL
//    sums sequential in point order on one lane), OpenCV 4's 10-step Levenberg-Marquardt control over the 8 free entries (normal
//    equations by a fixed-order block reduction, a Cholesky solve, lambda from the host's C library), H / H22, and the returned
//    mask recomputed as err(H) <= thr^2 over all points.
// The problem's points are the rows of [off[p], off[p+1]) whose sel is non-zero (all rows without sel), in row order; the mask is
// written at the rows (0 on unselected rows).
#define HOM_THREADS 256
#define HOM_WARPS (HOM_THREADS/32)
#define HOM_CHUNK 256
#define HOM_MAX_ATTEMPTS 10000
#define HOM_NRED 45                      // 36 entries of the upper triangle of J^T J, 8 of J^T r, S
enum { HOM_OK = 0, HOM_TOO_FEW = 1, HOM_FOUR_POINT = 2, HOM_RANSAC_FAILED = 3 };

struct HomBatch {
  const int* off; const float* src; const float* dst; const uint8_t* sel;
  int* cidx; int* lidx;                  // per row: the problem's point list (row of each rank), then its inlier list (ranks)
  float4* inl;                           // per row: the inliers gathered in order (src x, src y, dst x, dst y)
  float thr2; double conf; int max_iters, refine;
  double* H; uint8_t* mask; int* n_inl; int* status; int* iters; int* groups; int* rejected; int* best;
  int* counts; int counts_cap;           // per-iteration inlier counts (parity hook), the first counts_cap iterations; NULL: none
  double lam[33];                        // the LM's lambda = exp(lg * log(10.)), lg = -16 .. 16, from the host's C library as OpenCV
};

__device__ __forceinline__ double cv_hypot(double a, double b) {      // OpenCV lapack.cpp hypot
  a = fabs(a); b = fabs(b);
  if (a > b) { b /= a; return a*sqrt(1 + b*b); }
  if (b > 0) { a /= b; return b*sqrt(1 + a*a); }
  return 0;
}
// cv::eigen of the symmetric 9x9 A (upper triangle read, destroyed) by JacobiImpl_; returns the row of V holding the eigenvector of
// the smallest eigenvalue after OpenCV's descending selection sort (tracked as a permutation instead of swapping rows).
__device__ int cv_jacobi9(double* A, double* V) {
  const int n = 9; double W[9]; int indR[9], indC[9];
  for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) V[i*n + j] = i == j ? 1.0 : 0.0;
  for (int k = 0; k < n; k++) {
    W[k] = A[(n + 1)*k];
    if (k < n - 1) { int m = k + 1; double mv = fabs(A[n*k + m]); for (int i = k + 2; i < n; i++) { const double v = fabs(A[n*k + i]); if (mv < v) mv = v, m = i; } indR[k] = m; }
    if (k > 0) { int m = 0; double mv = fabs(A[k]); for (int i = 1; i < k; i++) { const double v = fabs(A[n*i + k]); if (mv < v) mv = v, m = i; } indC[k] = m; }
  }
  for (int iters = 0; iters < n*n*30; iters++) {
    int k = 0; double mv = fabs(A[indR[0]]);
    for (int i = 1; i < n - 1; i++) { const double v = fabs(A[n*i + indR[i]]); if (mv < v) mv = v, k = i; }
    int l = indR[k];
    for (int i = 1; i < n; i++) { const double v = fabs(A[n*indC[i] + i]); if (mv < v) mv = v, k = indC[i], l = i; }
    const double p = A[n*k + l];
    if (fabs(p) <= DBL_EPSILON) break;
    const double y = (W[l] - W[k])*0.5;
    double t = fabs(y) + cv_hypot(p, y);
    double s = cv_hypot(p, t);
    const double c = t/s;
    s = p/s; t = (p/t)*p;
    if (y < 0) s = -s, t = -t;
    A[n*k + l] = 0;
    W[k] -= t; W[l] += t;
    double a0, b0;
#define HOM_ROT(v0, v1) a0 = v0, b0 = v1, v0 = a0*c - b0*s, v1 = a0*s + b0*c
    for (int i = 0; i < k; i++) HOM_ROT(A[n*i + k], A[n*i + l]);
    for (int i = k + 1; i < l; i++) HOM_ROT(A[n*k + i], A[n*i + l]);
    for (int i = l + 1; i < n; i++) HOM_ROT(A[n*k + i], A[n*l + i]);
    for (int i = 0; i < n; i++) HOM_ROT(V[n*k + i], V[n*l + i]);
#undef HOM_ROT
    for (int j = 0; j < 2; j++) {
      const int idx = j == 0 ? k : l;
      if (idx < n - 1) { int m = idx + 1; double mv2 = fabs(A[n*idx + m]); for (int i = idx + 2; i < n; i++) { const double v = fabs(A[n*idx + i]); if (mv2 < v) mv2 = v, m = i; } indR[idx] = m; }
      if (idx > 0) { int m = 0; double mv2 = fabs(A[idx]); for (int i = 1; i < idx; i++) { const double v = fabs(A[n*i + idx]); if (mv2 < v) mv2 = v, m = i; } indC[idx] = m; }
    }
  }
  int perm[9]; for (int i = 0; i < n; i++) perm[i] = i;
  for (int k = 0; k < n - 1; k++) {
    int m = k; for (int i = k + 1; i < n; i++) if (W[m] < W[i]) m = i;
    if (k != m) { const double w = W[m]; W[m] = W[k]; W[k] = w; const int q = perm[m]; perm[m] = perm[k]; perm[k] = q; }
  }
  return perm[n - 1];
}
// the tail of runKernel: Jacobi on LtL (upper triangle), H = invHnorm * H0 * Hnorm2, times 1 / H22
__device__ void hom_from_ltl(double* L, const double c[4], const double s[4], double* H) {
  // c = (cm.x, cm.y, cM.x, cM.y), s = (sm.x, sm.y, sM.x, sM.y) after s = count / sum
  double V[81];
  const int r = cv_jacobi9(L, V);
  const double* H0 = V + 9*r;
  const double inv[9] = {1./s[0], 0, c[0], 0, 1./s[1], c[1], 0, 0, 1};
  const double h2[9] = {s[2], 0, -c[2]*s[2], 0, s[3], -c[3]*s[3], 0, 0, 1};
  double T[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) T[3*i + j] = (inv[3*i]*H0[j] + inv[3*i + 1]*H0[3 + j]) + inv[3*i + 2]*H0[6 + j];
  double R[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[3*i + j] = (T[3*i]*h2[j] + T[3*i + 1]*h2[3 + j]) + T[3*i + 2]*h2[6 + j];
  const double sc = 1./R[8];
  for (int e = 0; e < 9; e++) H[e] = R[e]*sc;
}
__device__ __forceinline__ void hom_ltl_add(double* L, double x, double y, double X, double Y) {
  const double Lx[9] = {X, Y, 1, 0, 0, 0, -x*X, -x*Y, -x}, Ly[9] = {0, 0, 0, X, Y, 1, -y*X, -y*Y, -y};
  for (int j = 0; j < 9; j++) for (int k = j; k < 9; k++) L[9*j + k] += Lx[j]*Lx[k] + Ly[j]*Ly[k];
}
// runKernel on 4 correspondences (one thread); false = no model
__device__ bool hom_kernel4(const float* Ms, const float* ms, double* H) {
  double c[4] = {0, 0, 0, 0}, s[4] = {0, 0, 0, 0};
  for (int i = 0; i < 4; i++) { c[0] += ms[2*i]; c[1] += ms[2*i + 1]; c[2] += Ms[2*i]; c[3] += Ms[2*i + 1]; }
  for (int e = 0; e < 4; e++) c[e] /= 4;
  for (int i = 0; i < 4; i++) {
    s[0] += fabs(ms[2*i] - c[0]); s[1] += fabs(ms[2*i + 1] - c[1]); s[2] += fabs(Ms[2*i] - c[2]); s[3] += fabs(Ms[2*i + 1] - c[3]);
  }
  for (int e = 0; e < 4; e++) if (fabs(s[e]) < DBL_EPSILON) return false;
  for (int e = 0; e < 4; e++) s[e] = 4/s[e];
  double L[81];
  for (int e = 0; e < 81; e++) L[e] = 0;
  for (int i = 0; i < 4; i++)
    hom_ltl_add(L, (ms[2*i] - c[0])*s[0], (ms[2*i + 1] - c[1])*s[1], (Ms[2*i] - c[2])*s[2], (Ms[2*i + 1] - c[3])*s[3]);
  hom_from_ltl(L, c, s, H);
  return true;
}
// haveCollinearPoints(ms, K): triples (j, k, K-1), k < j, float differences, double products
template <int K> __device__ bool hom_collinear(const float* p) {
  const int i = K - 1;
  for (int j = 0; j < i; j++) {
    const double dx1 = p[2*j] - p[2*i], dy1 = p[2*j + 1] - p[2*i + 1];
    for (int k = 0; k < j; k++) {
      const double dx2 = p[2*k] - p[2*i], dy2 = p[2*k + 1] - p[2*i + 1];
      if (fabs(dx2*dy1 - dy2*dx1) <= FLT_EPSILON*(fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2))) return true;
    }
  }
  return false;
}
__device__ __forceinline__ double hom_det3(const float* p, int a, int b, int c) {   // determinant(Matx33d) of rows (x, y, 1)
  const double a00 = p[2*a], a01 = p[2*a + 1], a10 = p[2*b], a11 = p[2*b + 1], a20 = p[2*c], a21 = p[2*c + 1];
  return a00*(a11*1.0 - a21*1.0) - a01*(a10*1.0 - a20*1.0) + 1.0*(a10*a21 - a20*a11);
}
__device__ bool hom_check_subset(const float* S, const float* D) {
  if (hom_collinear<4>(S) || hom_collinear<4>(D)) return false;
  const int tt[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {0, 1, 3}};
  int neg = 0;
  for (int i = 0; i < 4; i++) neg += hom_det3(S, tt[i][0], tt[i][1], tt[i][2])*hom_det3(D, tt[i][0], tt[i][1], tt[i][2]) < 0;
  return neg == 0 || neg == 4;
}
__device__ __forceinline__ float hom_err(const float* Hf, float x, float y, float u, float v) {   // computeError
  const float ww = 1.f/(Hf[6]*x + Hf[7]*y + 1.f);
  const float dx = (Hf[0]*x + Hf[1]*y + Hf[2])*ww - u, dy = (Hf[3]*x + Hf[4]*y + Hf[5])*ww - v;
  return dx*dx + dy*dy;
}
// RANSACUpdateNumIters(p, ep, model_points, niters)
__device__ int hom_update_iters(double p, double ep, int model_points, int max_iters) {
  p = fmin(fmax(p, 0.), 1.); ep = fmin(fmax(ep, 0.), 1.);
  double num = fmax(1. - p, DBL_MIN), denom = 1. - pow(1. - ep, (double)model_points);
  if (denom < DBL_MIN) return 0;
  num = log(num); denom = log(denom);
  return denom >= 0 || -num >= max_iters*(-denom) ? max_iters : __double2int_rn(num/denom);
}
// HomographyRefineCallback::compute for one correspondence: residuals (2) and, with J, the two Jacobian rows
__device__ __forceinline__ void hom_resid(const double* h, double Mx, double My, double mx, double my, double* r, double* J) {
  double ww = h[6]*Mx + h[7]*My + 1.;
  ww = fabs(ww) > DBL_EPSILON ? 1./ww : 0;
  const double xi = (h[0]*Mx + h[1]*My + h[2])*ww, yi = (h[3]*Mx + h[4]*My + h[5])*ww;
  r[0] = xi - mx; r[1] = yi - my;
  if (J) {
    J[0] = Mx*ww; J[1] = My*ww; J[2] = ww; J[3] = J[4] = J[5] = 0.; J[6] = -Mx*ww*xi; J[7] = -My*ww*xi;
    J[8] = J[9] = J[10] = 0.; J[11] = Mx*ww; J[12] = My*ww; J[13] = ww; J[14] = -Mx*ww*yi; J[15] = -My*ww*yi;
  }
}
// block-wide sum of NV doubles per thread in a fixed order (warp butterflies, then warps in order on thread 0) into out
template <int NV> __device__ void hom_block_sum(double* v, double (*red)[HOM_NRED], double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int e = 0; e < NV; e++) {
    double x = v[e];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    v[e] = x;
  }
  if (lane == 0) for (int e = 0; e < NV; e++) red[warp][e] = v[e];
  __syncthreads();
  if (threadIdx.x == 0) for (int e = 0; e < NV; e++) { double x = red[0][e]; for (int w = 1; w < HOM_WARPS; w++) x += red[w][e]; out[e] = x; }
  __syncthreads();
}
// in-order compaction inside the CTA: out[k] = value(i) of the k-th i in [0, n) with flag(i); returns the count (all threads)
template <class F, class G> __device__ int hom_compact(int n, F flag, G value, int* out, int* sh_wcnt) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += HOM_THREADS) {
    const int i = i0 + threadIdx.x;
    const bool f = i < n && flag(i);
    const unsigned b = __ballot_sync(0xffffffffu, f);
    if (lane == 0) sh_wcnt[warp] = __popc(b);
    __syncthreads();
    int before = base;
    for (int w = 0; w < warp; w++) before += sh_wcnt[w];
    if (f) out[before + __popc(b & ((1u << lane) - 1))] = value(i);
    int tot = 0; for (int w = 0; w < HOM_WARPS; w++) tot += sh_wcnt[w];
    base += tot;
    __syncthreads();
  }
  return base;
}
// the next `count` groups of K distinct indices in [0, n) from cv::RNG state st (getSubset: a duplicate is re-drawn at once) into
// grp[count][K]; returns the new state
template <int K> __device__ unsigned long long hom_draw_groups(unsigned long long st, int n, int count, int* grp) {
  for (int g = 0; g < count; g++)
    for (int i = 0; i < K;) {
      st = (unsigned long long)(unsigned)st*4164903690ull + (st >> 32);
      const int k = (int)((unsigned)st % (unsigned)n);
      bool dup = false; for (int j = 0; j < i; j++) dup |= grp[K*g + j] == k;
      if (!dup) grp[K*g + i++] = k;
    }
  return st;
}

__global__ void __launch_bounds__(HOM_THREADS) hom_ransac_kernel(HomBatch B) {
  __shared__ int sh_grp[HOM_CHUNK][4];
  __shared__ int sh_cnt[HOM_CHUNK];              // -2: rejected by the subset test, -1: no model, else the inlier count
  __shared__ double sh_H[HOM_CHUNK][9];
  __shared__ float4 sh_tile[HOM_THREADS];        // (src x, src y, dst x, dst y)
  __shared__ double sh_red[HOM_WARPS][HOM_NRED];
  __shared__ double sh_best[9], sh_x[9], sh_xd[9], sh_sum[HOM_NRED], sh_A[64], sh_v[8], sh_S, sh_Sd, sh_c[4], sh_s[4], sh_L[81];
  __shared__ int sh_wcnt[HOM_WARPS];
  __shared__ unsigned long long sh_rng;
  __shared__ int sh_it, sh_niters, sh_best_cnt, sh_best_it, sh_groups, sh_rej, sh_run, sh_done, sh_fail, sh_ninl, sh_ok, sh_lm_go;
  const int pb = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int r0 = B.off[pb], nrows = B.off[pb + 1] - r0;
  int* cidx = B.cidx + r0; int* lidx = B.lidx + r0;
  const float2* src = reinterpret_cast<const float2*>(B.src); const float2* dst = reinterpret_cast<const float2*>(B.dst);
  for (int i = t; i < nrows; i += HOM_THREADS) B.mask[r0 + i] = 0;
  const uint8_t* sel = B.sel;
  const int n = sel ? hom_compact(nrows, [&](int i) { return sel[r0 + i] != 0; }, [&](int i) { return r0 + i; }, cidx, sh_wcnt)
                    : hom_compact(nrows, [&](int) { return true; }, [&](int i) { return r0 + i; }, cidx, sh_wcnt);
  double* Hout = B.H + 9*(size_t)pb;
  if (n < 4) {                                   // geometricVerification: fewer than 4 points are all inliers
    for (int i = t; i < n; i += HOM_THREADS) B.mask[cidx[i]] = 1;
    if (t < 9) Hout[t] = 0;
    if (t == 0) { B.status[pb] = HOM_TOO_FEW; B.n_inl[pb] = n; B.iters[pb] = 0; B.groups[pb] = 0; B.rejected[pb] = 0; B.best[pb] = -1; }
    return;
  }
  if (n == 4) {                                  // findHomography: runKernel only, no RANSAC and no refinement
    if (t == 0) {
      float Ms[8], ms[8];
      for (int i = 0; i < 4; i++) { const float2 a = src[cidx[i]], b = dst[cidx[i]]; Ms[2*i] = a.x; Ms[2*i + 1] = a.y; ms[2*i] = b.x; ms[2*i + 1] = b.y; }
      double H[9]; const bool ok = hom_kernel4(Ms, ms, H);
      for (int e = 0; e < 9; e++) Hout[e] = ok ? H[e] : 0;
      for (int i = 0; i < 4; i++) B.mask[cidx[i]] = ok ? 1 : 0;
      B.status[pb] = HOM_FOUR_POINT; B.n_inl[pb] = ok ? 4 : 0; B.iters[pb] = 0; B.groups[pb] = 0; B.rejected[pb] = 0; B.best[pb] = -1;
    }
    return;
  }
  if (t == 0) {
    sh_rng = ~0ull; sh_it = 0; sh_niters = max(B.max_iters, 1); sh_best_cnt = 0; sh_best_it = -1; sh_groups = 0; sh_rej = 0; sh_run = 0;
    sh_done = 0; sh_fail = 0;
  }
  __syncthreads();
  int* counts = B.counts ? B.counts + (size_t)pb*B.counts_cap : nullptr;
  for (int c = 0; !sh_done; c++) {
    const int nch = min(HOM_CHUNK, 32 << min(c, 3));
    if (t == 0) sh_rng = hom_draw_groups<4>(sh_rng, n, nch, &sh_grp[0][0]);     // the draw stream, cut into groups of 4
    __syncthreads();
    if (t < nch) {                               // subset test and 4-point model, one thread per group
      float Ms[8], ms[8];
      for (int i = 0; i < 4; i++) { const int r = cidx[sh_grp[t][i]]; const float2 a = src[r], b = dst[r]; Ms[2*i] = a.x; Ms[2*i + 1] = a.y; ms[2*i] = b.x; ms[2*i + 1] = b.y; }
      int cnt = -2;
      if (hom_check_subset(Ms, ms)) cnt = hom_kernel4(Ms, ms, sh_H[t]) ? 0 : -1;
      sh_cnt[t] = cnt;
    }
    for (int tile0 = 0; tile0 < n; tile0 += HOM_THREADS) {    // inlier counts, points staged through shared memory
      const int tn = min(HOM_THREADS, n - tile0);
      __syncthreads();
      if (t < tn) { const int r = cidx[tile0 + t]; const float2 a = src[r], b = dst[r]; sh_tile[t] = make_float4(a.x, a.y, b.x, b.y); }
      __syncthreads();
      for (int m = warp; m < nch; m += HOM_WARPS) {
        if (sh_cnt[m] < 0) continue;
        float Hf[8]; for (int e = 0; e < 8; e++) Hf[e] = (float)sh_H[m][e];
        int cnt = 0;
        for (int j0 = 0; j0 < tn; j0 += 32) {
          const int j = j0 + lane;
          bool in = false;
          if (j < tn) { const float4 q = sh_tile[j]; in = hom_err(Hf, q.x, q.y, q.z, q.w) <= B.thr2; }
          cnt += __popc(__ballot_sync(0xffffffffu, in));
        }
        if (lane == 0) sh_cnt[m] += cnt;
      }
    }
    __syncthreads();
    if (t == 0) {                                // the sequential loop of RANSACPointSetRegistrator::run over this chunk
      int it = sh_it, niters = sh_niters, best = sh_best_cnt, run = sh_run, groups = sh_groups, rej = sh_rej;
      bool done = false;
      for (int m = 0; m < nch; m++) {
        groups++;
        if (sh_cnt[m] == -2) {
          rej++;
          if (++run >= HOM_MAX_ATTEMPTS) { done = true; if (it == 0) sh_fail = 1; break; }
          continue;
        }
        run = 0;
        const int cnt = sh_cnt[m];
        if (counts && it < B.counts_cap) counts[it] = cnt;
        if (cnt > max(best, 3)) {
          best = cnt; sh_best_it = it;
          for (int e = 0; e < 9; e++) sh_best[e] = sh_H[m][e];
          niters = hom_update_iters(B.conf, (double)(n - cnt)/n, 4, niters);
        }
        if (++it >= niters) { done = true; break; }
      }
      sh_it = it; sh_niters = niters; sh_best_cnt = best; sh_run = run; sh_groups = groups; sh_rej = rej; sh_done = done;
    }
    __syncthreads();
  }
  const bool model = !sh_fail && sh_best_cnt > 0;
  if (!model) {                                  // RANSAC failed: no H, all zeros
    if (t < 9) Hout[t] = 0;
    if (t == 0) { B.status[pb] = HOM_RANSAC_FAILED; B.n_inl[pb] = 0; B.iters[pb] = sh_fail ? 0 : sh_it; B.groups[pb] = sh_groups; B.rejected[pb] = sh_rej; B.best[pb] = -1; }
    return;
  }
  if (B.refine) {
    // the RANSAC mask, compacted in order (ranks)
    float Hb[8]; for (int e = 0; e < 8; e++) Hb[e] = (float)sh_best[e];
    const int m = hom_compact(n, [&](int i) { const float2 a = src[cidx[i]], b = dst[cidx[i]]; return hom_err(Hb, a.x, a.y, b.x, b.y) <= B.thr2; },
                              [&](int i) { return i; }, lidx, sh_wcnt);
    float4* Q = B.inl + r0;                     // the inliers, gathered in order: the sequential sums below read them contiguously
    for (int i = t; i < m; i += HOM_THREADS) { const int r = cidx[lidx[i]]; const float2 a = src[r], b = dst[r]; Q[i] = make_float4(a.x, a.y, b.x, b.y); }
    __syncthreads();
    // runKernel over the inliers: 4 centroid sums, 4 deviation sums, then the 45 LtL sums, each sequential in point order on one lane
    auto coord = [](const float4& q, int e) { return e == 0 ? q.z : e == 1 ? q.w : e == 2 ? q.x : q.y; };   // (m.x, m.y, M.x, M.y)
    if (t < 4) {
      double a = 0;
      for (int i = 0; i < m; i++) a += coord(Q[i], t);
      sh_c[t] = a/m;
    }
    __syncthreads();
    if (t < 4) {
      double a = 0; const double cc = sh_c[t];
      for (int i = 0; i < m; i++) a += fabs(coord(Q[i], t) - cc);
      sh_s[t] = a;
    }
    __syncthreads();
    const bool ok = fabs(sh_s[0]) >= DBL_EPSILON && fabs(sh_s[1]) >= DBL_EPSILON && fabs(sh_s[2]) >= DBL_EPSILON && fabs(sh_s[3]) >= DBL_EPSILON;
    if (ok) {
      double s[4]; for (int e = 0; e < 4; e++) s[e] = m/sh_s[e];
      if (t < HOM_NRED) {
        int j = 0, k = t; while (k >= 9 - j) { k -= 9 - j; j++; } k += j;        // t -> (j, k), k >= j
        double a = 0;
        for (int i = 0; i < m; i++) {
          const float4 q = Q[i];
          const double x = (q.z - sh_c[0])*s[0], y = (q.w - sh_c[1])*s[1], X = (q.x - sh_c[2])*s[2], Y = (q.y - sh_c[3])*s[3];
          const double Lx[9] = {X, Y, 1, 0, 0, 0, -x*X, -x*Y, -x}, Ly[9] = {0, 0, 0, X, Y, 1, -y*X, -y*Y, -y};
          a += Lx[j]*Lx[k] + Ly[j]*Ly[k];
        }
        sh_L[9*j + k] = a;
      }
      __syncthreads();
      if (t == 0) { double c4[4] = {sh_c[0], sh_c[1], sh_c[2], sh_c[3]}; hom_from_ltl(sh_L, c4, s, sh_x); }
    } else if (t < 9) sh_x[t] = sh_best[t];       // (runKernel's result is not checked: H stays the RANSAC model)
    __syncthreads();
    // Levenberg-Marquardt over H[0..7] (OpenCV 4 LMSolver, 10 steps): J^T J, J^T r and S by a fixed-order block reduction
    int lg = -3, it = 0;
    auto normal_eq = [&](const double* h) {
      double acc[HOM_NRED]; for (int e = 0; e < HOM_NRED; e++) acc[e] = 0;
      for (int i = t; i < m; i += HOM_THREADS) {
        const float4 q = Q[i];
        double rr[2], J[16]; hom_resid(h, q.x, q.y, q.z, q.w, rr, J);
        for (int row = 0; row < 2; row++) {
          const double* Jr = J + 8*row; int e = 0;
          for (int a = 0; a < 8; a++) for (int b = a; b < 8; b++) acc[e++] += Jr[a]*Jr[b];
          for (int a = 0; a < 8; a++) acc[36 + a] += Jr[a]*rr[row];
          acc[44] += rr[row]*rr[row];
        }
      }
      hom_block_sum<HOM_NRED>(acc, sh_red, sh_sum);
      if (t == 0) {
        int e = 0;
        for (int a = 0; a < 8; a++) for (int b = a; b < 8; b++) { sh_A[8*a + b] = sh_sum[e]; sh_A[8*b + a] = sh_sum[e]; e++; }
        for (int a = 0; a < 8; a++) sh_v[a] = sh_sum[36 + a];
        sh_S = sh_sum[44];
      }
      __syncthreads();
    };
    normal_eq(sh_x);
    for (;;) {
      double dmax = 0;
      if (t == 0) {                              // (A + lambda diag A) d = v by Cholesky, xd = x - d
        const double lambda = B.lam[lg + 16];
        double Ap[64], d[8];
        for (int e = 0; e < 64; e++) Ap[e] = sh_A[e];
        for (int a = 0; a < 8; a++) Ap[9*a] *= 1 + lambda;
        for (int j = 0; j < 8; j++) {
          double s = Ap[9*j]; for (int k = 0; k < j; k++) s -= Ap[8*j + k]*Ap[8*j + k];
          const double lj = sqrt(fmax(s, 0.0)); Ap[9*j] = lj;
          for (int i = j + 1; i < 8; i++) { double q = Ap[8*i + j]; for (int k = 0; k < j; k++) q -= Ap[8*i + k]*Ap[8*j + k]; Ap[8*i + j] = lj > 0 ? q/lj : 0; }
        }
        for (int i = 0; i < 8; i++) { double q = sh_v[i]; for (int k = 0; k < i; k++) q -= Ap[8*i + k]*d[k]; d[i] = Ap[9*i] > 0 ? q/Ap[9*i] : 0; }
        for (int i = 7; i >= 0; i--) { double q = d[i]; for (int k = i + 1; k < 8; k++) q -= Ap[8*k + i]*d[k]; d[i] = Ap[9*i] > 0 ? q/Ap[9*i] : 0; }
        for (int e = 0; e < 8; e++) { sh_xd[e] = sh_x[e] - d[e]; dmax = fmax(dmax, fabs(d[e])); }
        sh_xd[8] = sh_x[8];
      }
      __syncthreads();
      {
        double acc[1] = {0};
        for (int i = t; i < m; i += HOM_THREADS) {
          const float4 q = Q[i];
          double rr[2]; hom_resid(sh_xd, q.x, q.y, q.z, q.w, rr, nullptr);
          acc[0] += rr[0]*rr[0]; acc[0] += rr[1]*rr[1];
        }
        hom_block_sum<1>(acc, sh_red, &sh_Sd);
      }
      bool better = false;
      if (t == 0) {
        better = sh_Sd < sh_S;
        if (better) { lg = max(lg - 1, -16); it++; for (int e = 0; e < 9; e++) sh_x[e] = sh_xd[e]; }
        else { it += lg == 16; lg = min(lg + 1, 16); }
        sh_ok = better;
      }
      __syncthreads();
      if (sh_ok) normal_eq(sh_x);                // (S becomes Sd)
      if (t == 0) sh_lm_go = it < 10 && dmax >= FLT_EPSILON && sh_S >= (double)FLT_EPSILON*FLT_EPSILON;
      __syncthreads();
      if (!sh_lm_go) break;
    }
    if (t == 0) {
      const double sc = fabs(sh_x[8]) > FLT_EPSILON ? 1./sh_x[8] : 1.;
      for (int e = 0; e < 9; e++) sh_best[e] = sh_x[e]*sc;
    }
    __syncthreads();
  }
  // the returned mask: err(H) <= thr^2 over all points
  if (t == 0) sh_ninl = 0;
  __syncthreads();
  float Hf[8]; for (int e = 0; e < 8; e++) Hf[e] = (float)sh_best[e];
  int cnt = 0;
  for (int i = t; i < n; i += HOM_THREADS) {
    const int r = cidx[i]; const float2 a = src[r], b = dst[r];
    const bool in = hom_err(Hf, a.x, a.y, b.x, b.y) <= B.thr2;
    B.mask[r] = in; cnt += in;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) atomicAdd(&sh_ninl, cnt);
  __syncthreads();
  if (t < 9) Hout[t] = sh_best[t];
  if (t == 0) { B.status[pb] = HOM_OK; B.n_inl[pb] = sh_ninl; B.iters[pb] = sh_it; B.groups[pb] = sh_groups; B.rejected[pb] = sh_rej; B.best[pb] = sh_best_it; }
}
// ---------------------------------------------------------------------------------------------------- fundamental-matrix RANSAC
// cv::findFundamentalMat(p1, p2, FM_RANSAC, thr, conf, max_iters) as FeatureTracker::stereoTrack calls it (FeatureTracker.cc:279-281),
// one persistent CTA per problem.  tests/fundamental_oracle.py restates the orders, tests/test_fundamental.py pins them against cv2:
//  * draws: the homography's cv::RNG stream and duplicate rule, groups of 7; subset test = haveCollinearPoints on either set; 10 000
//    (RANSAC) or 1000 (LMedS) rejections in a row end the loop (fail it in iteration 0);
//  * model: run7Point, one thread per draw: Hartley normalisation, OpenCV's one-sided Jacobi SVD of the 7x9 system with the null
//    space rows completed from cv::RNG(0x12345678), the determinant cubic, cv::solveCubic, per root lambda / mu scaling,
//    de-normalisation and F / F22;
//  * n >= 15: RANSAC.  Warps count the inliers of every (draw, root) model over points staged through shared memory; thread 0
//    replays the loop in (draw, root) order (best when count > max(best, 6), then RANSACUpdateNumIters(conf, ., 7, niters)), so
//    nothing depends on the chunk size;
//  * 8 <= n < 15: LMedS.  One thread per model takes the (n/2)-th smallest float error (n is at most 14); a strictly smaller median
//    wins; the mask is err <= sigma^2 with OpenCV's sigma;
//  * n == 7: run7Point alone (up to 3 models, mask all ones); n < 7: no model.
// A draw whose cubic counts as all zero (solveCubic returns -1, which cv2 4.13 does not guard and raises on) has no model.
#define FUND_THREADS 128
#define FUND_WARPS (FUND_THREADS/32)
#define FUND_CHUNK 128
enum { FUND_OK = 0, FUND_LMEDS = 1, FUND_SEVEN_POINT = 2, FUND_TOO_FEW = 3, FUND_FAILED = 4 };

struct FundBatch {
  const int* off; const float* src; const float* dst;
  float thr2; double conf; int max_iters;
  double* F; uint8_t* mask;                      // F[P][27]: up to 3 models, row-major
  int* stat;                                     // 9 arrays of P: n_models, n_inliers, status, iterations, groups, rejected, best, best_root, success
  float* rec; int rec_cap;                       // parity hook: per iteration (models, score of root 0, 1, 2), the first rec_cap iterations
};

// cv::solveCubic (OpenCV 4.13) of (a0, a1, a2, a3): the number of roots (-1: every coefficient counts as 0), roots in x.
// Every coefficient is 0 when max|a_i| < DBL_EPSILON; a leading coefficient with |a_i * (1 / max|a_j|)| < DBL_EPSILON counts as
// 0, cascading down; the quadratic / linear branches use the unscaled coefficients, the cubic branch the scaled ones.
__device__ int cv_solve_cubic(double a0, double a1, double a2, double a3, double* x) {
  x[0] = x[1] = x[2] = 0;
  const double m = fmax(fmax(fabs(a0), fabs(a1)), fmax(fabs(a2), fabs(a3)));
  if (!(m >= DBL_EPSILON)) return -1;
  const double inv = 1./m;
  auto small = [inv](double v) { return fabs(v*inv) < DBL_EPSILON; };
  if (!small(a0)) { a0 *= inv; a1 *= inv; a2 *= inv; a3 *= inv; }
  else { a0 = 0; if (small(a1)) { a1 = 0; if (small(a2)) { a2 = 0; if (small(a3)) a3 = 0; } } }
  if (a0 == 0) {
    if (a1 == 0) {
      if (a2 == 0) return a3 == 0 ? -1 : 0;
      x[0] = -a3/a2; return 1;
    }
    double d = a2*a2 - 4*a1*a3;
    if (d < 0) return 0;
    d = sqrt(d);
    const double q1 = (-a2 + d)*0.5, q2 = (a2 + d)*-0.5;
    if (fabs(q1) > fabs(q2)) { x[0] = q1/a1; x[1] = a3/q1; } else { x[0] = q2/a1; x[1] = a3/q2; }
    return d > 0 ? 2 : 1;
  }
  a0 = 1./a0; a1 *= a0; a2 *= a0; a3 *= a0;
  const double Q = (a1*a1 - 3*a2)*(1./9);
  const double R = (a1*(2*a1*a1 - 9*a2) + 27*a3)*(1./54);
  const double Qcubed = Q*Q*Q;
  double d = (a1*a1*(a2*a2 - 4*a1*a3) + 2*a2*(9*a1*a3 - 2*a2*a2) - 27*a3*a3)*(1./108);
  if (d > 0) {
    const double theta = acos(R/sqrt(Qcubed)), t0 = -2*sqrt(Q), t1 = theta*(1./3), t2 = a1*(1./3);
    x[0] = t0*cos(t1) - t2; x[1] = t0*cos(t1 + (2.*CUDART_PI/3)) - t2; x[2] = t0*cos(t1 + (4.*CUDART_PI/3)) - t2;
    return 3;
  }
  if (d == 0) {
    if (R >= 0) { x[0] = -2*pow(R, 1./3) - a1/3; x[1] = pow(R, 1./3) - a1/3; }
    else { x[0] = 2*pow(-R, 1./3) - a1/3; x[1] = -pow(-R, 1./3) - a1/3; }
    const bool one = x[0] == x[1];
    if (one) x[1] = 0;
    return one ? 1 : 2;
  }
  d = sqrt(-d);
  double e = pow(d + fabs(R), 1./3);
  if (R > 0) e = -e;
  x[0] = (e + Q/e) - a1*(1./3);
  return 1;
}
// JacobiSVDImpl_'s completion of row i of U[9][9] from the generator state st (the rows before it are orthonormal)
__device__ void cv_svd_complete(double* U, int i, unsigned long long& st) {
  const double eps = DBL_EPSILON*10;
  double sd = 0;
  for (int ii = 0; ii < 100 && sd <= DBL_MIN; ii++) {
    for (int k = 0; k < 9; k++) {
      st = (unsigned long long)(unsigned)st*4164903690ull + (st >> 32);
      U[9*i + k] = ((unsigned)st & 256) != 0 ? 1./9 : -(1./9);
    }
    for (int it = 0; it < 2; it++)
      for (int j = 0; j < i; j++) {
        sd = 0; for (int k = 0; k < 9; k++) sd += U[9*i + k]*U[9*j + k];
        double asum = 0;
        for (int k = 0; k < 9; k++) { const double t = U[9*i + k] - sd*U[9*j + k]; U[9*i + k] = t; asum += fabs(t); }
        asum = asum > eps*100 ? 1/asum : 0;
        for (int k = 0; k < 9; k++) U[9*i + k] *= asum;
      }
    sd = 0; for (int k = 0; k < 9; k++) sd += U[9*i + k]*U[9*i + k];
    sd = sqrt(sd);
  }
  const double s = sd > DBL_MIN ? 1/sd : 0.;
  for (int k = 0; k < 9; k++) U[9*i + k] *= s;
}
// SVDecomp(A, W, U, Vt, MODIFY_A | FULL_UV) of the 7x9 A held in U's first 7 rows: U becomes Vt (9x9).  OpenCV transposes the
// problem, so the one-sided Jacobi rotates the 7 rows; rows past the rank come from cv::RNG(0x12345678).
__device__ void cv_svd7x9(double* U) {
  const double eps = DBL_EPSILON*10;
  double W[7];
  for (int i = 0; i < 7; i++) { double s = 0; for (int k = 0; k < 9; k++) s += U[9*i + k]*U[9*i + k]; W[i] = s; }
  for (int iter = 0; iter < 30; iter++) {
    bool changed = false;
    for (int i = 0; i < 6; i++)
      for (int j = i + 1; j < 7; j++) {
        double* Ai = U + 9*i; double* Aj = U + 9*j;
        const double a = W[i], b = W[j];
        double p = 0; for (int k = 0; k < 9; k++) p += Ai[k]*Aj[k];
        if (fabs(p) <= eps*sqrt(a*b)) continue;
        p *= 2;
        const double beta = a - b, gamma = cv_hypot(p, beta);
        double c, s;
        if (beta < 0) { const double delta = (gamma - beta)*0.5; s = sqrt(delta/gamma); c = p/(gamma*s*2); }
        else { c = sqrt((gamma + beta)/(gamma*2)); s = p/(gamma*c*2); }
        double na = 0, nb = 0;
        for (int k = 0; k < 9; k++) {
          const double t0 = c*Ai[k] + s*Aj[k], t1 = -s*Ai[k] + c*Aj[k];
          Ai[k] = t0; Aj[k] = t1; na += t0*t0; nb += t1*t1;
        }
        W[i] = na; W[j] = nb;
        changed = true;
      }
    if (!changed) break;
  }
  for (int i = 0; i < 7; i++) { double s = 0; for (int k = 0; k < 9; k++) s += U[9*i + k]*U[9*i + k]; W[i] = sqrt(s); }
  for (int i = 0; i < 6; i++) {
    int j = i; for (int k = i + 1; k < 7; k++) if (W[j] < W[k]) j = k;
    if (i != j) { const double w = W[i]; W[i] = W[j]; W[j] = w; for (int k = 0; k < 9; k++) { const double q = U[9*i + k]; U[9*i + k] = U[9*j + k]; U[9*j + k] = q; } }
  }
  unsigned long long st = 0x12345678ull;
  for (int i = 0; i < 9; i++) {
    const double sd = i < 7 ? W[i] : 0;
    if (sd <= DBL_MIN) cv_svd_complete(U, i, st);
    else { const double s = 1/sd; for (int k = 0; k < 9; k++) U[9*i + k] *= s; }
  }
}
// run7Point on 7 correspondences P1 -> P2 ([7][2] float): the number of models written to F[3][9] (-1: all-zero cubic, 0: none)
__device__ int fund_run7(const float* P1, const float* P2, double* F) {
  double c1x = 0, c1y = 0, c2x = 0, c2y = 0;
  for (int i = 0; i < 7; i++) { c1x += P1[2*i]; c1y += P1[2*i + 1]; c2x += P2[2*i]; c2y += P2[2*i + 1]; }
  const double t = 1./7;
  c1x *= t; c1y *= t; c2x *= t; c2y *= t;
  double s1 = 0, s2 = 0;
  for (int i = 0; i < 7; i++) {
    const double dx1 = P1[2*i] - c1x, dy1 = P1[2*i + 1] - c1y, dx2 = P2[2*i] - c2x, dy2 = P2[2*i + 1] - c2y;
    s1 += sqrt(dx1*dx1 + dy1*dy1); s2 += sqrt(dx2*dx2 + dy2*dy2);
  }
  s1 *= t; s2 *= t;
  if (s1 < FLT_EPSILON || s2 < FLT_EPSILON) return 0;
  s1 = sqrt(2.)/s1; s2 = sqrt(2.)/s2;
  double U[81];
  for (int i = 0; i < 7; i++) {
    const double x0 = (P1[2*i] - c1x)*s1, y0 = (P1[2*i + 1] - c1y)*s1, x1 = (P2[2*i] - c2x)*s2, y1 = (P2[2*i + 1] - c2y)*s2;
    double* a = U + 9*i;
    a[0] = x1*x0; a[1] = x1*y0; a[2] = x1; a[3] = y1*x0; a[4] = y1*y0; a[5] = y1; a[6] = x0; a[7] = y0; a[8] = 1;
  }
  cv_svd7x9(U);
  double f1[9], f2[9];
  for (int i = 0; i < 9; i++) { f2[i] = U[72 + i]; f1[i] = U[63 + i] - f2[i]; }
  double t0 = f2[4]*f2[8] - f2[5]*f2[7], t1 = f2[3]*f2[8] - f2[5]*f2[6], t2 = f2[3]*f2[7] - f2[4]*f2[6];
  const double c3 = f2[0]*t0 - f2[1]*t1 + f2[2]*t2;
  const double c2 = f1[0]*t0 - f1[1]*t1 + f1[2]*t2 - f1[3]*(f2[1]*f2[8] - f2[2]*f2[7]) + f1[4]*(f2[0]*f2[8] - f2[2]*f2[6])
                  - f1[5]*(f2[0]*f2[7] - f2[1]*f2[6]) + f1[6]*(f2[1]*f2[5] - f2[2]*f2[4]) - f1[7]*(f2[0]*f2[5] - f2[2]*f2[3])
                  + f1[8]*(f2[0]*f2[4] - f2[1]*f2[3]);
  t0 = f1[4]*f1[8] - f1[5]*f1[7]; t1 = f1[3]*f1[8] - f1[5]*f1[6]; t2 = f1[3]*f1[7] - f1[4]*f1[6];
  const double c1 = f2[0]*t0 - f2[1]*t1 + f2[2]*t2 - f2[3]*(f1[1]*f1[8] - f1[2]*f1[7]) + f2[4]*(f1[0]*f1[8] - f1[2]*f1[6])
                  - f2[5]*(f1[0]*f1[7] - f1[1]*f1[6]) + f2[6]*(f1[1]*f1[5] - f1[2]*f1[4]) - f2[7]*(f1[0]*f1[5] - f1[2]*f1[3])
                  + f2[8]*(f1[0]*f1[4] - f1[1]*f1[3]);
  const double c0 = f1[0]*t0 - f1[1]*t1 + f1[2]*t2;
  double r[3];
  const int n = cv_solve_cubic(c0, c1, c2, c3, r);
  if (n < 1 || n > 3) return n;
  const double T1[9] = {s1, 0, -s1*c1x, 0, s1, -s1*c1y, 0, 0, 1};
  const double T2t[9] = {s2, 0, 0, 0, s2, 0, -s2*c2x, -s2*c2y, 1};
  for (int k = 0; k < n; k++) {
    double lambda = r[k], mu = 1., fm[9];
    const double s = f1[8]*r[k] + f2[8];
    if (fabs(s) > DBL_EPSILON) { mu = 1./s; lambda *= mu; fm[8] = 1.; } else fm[8] = 0.;
    for (int i = 0; i < 8; i++) fm[i] = f1[i]*lambda + f2[i]*mu;
    double T[9], R[9];                           // (T2^T F) T1, Matx products (sums from 0, left to right)
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double a = 0; for (int q = 0; q < 3; q++) a += T2t[3*i + q]*fm[3*q + j]; T[3*i + j] = a; }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double a = 0; for (int q = 0; q < 3; q++) a += T[3*i + q]*T1[3*q + j]; R[3*i + j] = a; }
    if (fabs(R[8]) > FLT_EPSILON) { const double inv = 1./R[8]; for (int e = 0; e < 9; e++) R[e] *= inv; }
    for (int e = 0; e < 9; e++) F[9*k + e] = R[e];
  }
  return n;
}
// computeError: the larger squared distance to the two epipolar lines, in double, stored as float
__device__ __forceinline__ float fund_err(const double* F, float x1f, float y1f, float x2f, float y2f) {
  const double x1 = x1f, y1 = y1f, x2 = x2f, y2 = y2f;
  double a = F[0]*x1 + F[1]*y1 + F[2], b = F[3]*x1 + F[4]*y1 + F[5], c = F[6]*x1 + F[7]*y1 + F[8];
  const double s2 = 1./(a*a + b*b), d2 = x2*a + y2*b + c;
  a = F[0]*x2 + F[3]*y2 + F[6]; b = F[1]*x2 + F[4]*y2 + F[7]; c = F[2]*x2 + F[5]*y2 + F[8];
  const double s1 = 1./(a*a + b*b), d1 = x1*a + y1*b + c;
  const double e1 = d1*d1*s1, e2 = d2*d2*s2;
  return (float)(e1 < e2 ? e2 : e1);             // std::max(e1, e2)
}

__global__ void __launch_bounds__(FUND_THREADS) fund_ransac_kernel(FundBatch B) {
  __shared__ int sh_grp[FUND_CHUNK][7];
  __shared__ int sh_nm[FUND_CHUNK];              // -2: rejected by the subset test, else run7Point's root count
  __shared__ double sh_F[FUND_CHUNK][27];
  __shared__ float sh_score[FUND_CHUNK][3];      // inlier count (RANSAC) or median (LMedS) per model
  __shared__ float4 sh_tile[FUND_THREADS];
  __shared__ double sh_best[9];
  __shared__ float sh_best_med;
  __shared__ unsigned long long sh_rng;
  __shared__ int sh_it, sh_niters, sh_best_cnt, sh_best_it, sh_best_root, sh_groups, sh_rej, sh_run, sh_done, sh_fail, sh_ninl;
  const int pb = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int r0 = B.off[pb], n = B.off[pb + 1] - r0;
  const float2* src = reinterpret_cast<const float2*>(B.src) + r0; const float2* dst = reinterpret_cast<const float2*>(B.dst) + r0;
  uint8_t* mask = B.mask + r0;
  double* Fout = B.F + 27*(size_t)pb;
  const size_t P = gridDim.x;
  int* n_models = B.stat; int* n_inl = B.stat + P; int* status = B.stat + 2*P; int* iters = B.stat + 3*P; int* groups = B.stat + 4*P;
  int* rejected = B.stat + 5*P; int* best = B.stat + 6*P; int* best_root = B.stat + 7*P; int* success = B.stat + 8*P;
  for (int i = t; i < n; i += FUND_THREADS) mask[i] = 0;
  for (int e = t; e < 27; e += FUND_THREADS) Fout[e] = 0;
  __syncthreads();                               // the zeros above land before any thread writes the outputs below
  if (n <= 7) {                                  // fewer than 7: no model; exactly 7: run7Point alone
    if (t == 0) {
      int nm = 0;
      if (n == 7) {
        float P1[14], P2[14];
        for (int i = 0; i < 7; i++) { P1[2*i] = src[i].x; P1[2*i + 1] = src[i].y; P2[2*i] = dst[i].x; P2[2*i + 1] = dst[i].y; }
        double F[27]; nm = fund_run7(P1, P2, F);
        if (nm > 0) for (int e = 0; e < 9*nm; e++) Fout[e] = F[e];
        if (B.rec && B.rec_cap > 0) { float* rc = B.rec + (size_t)pb*4*B.rec_cap; rc[0] = (float)nm; }
      }
      const int m = nm > 0 ? nm : 0;
      for (int i = 0; i < n; i++) mask[i] = m > 0;
      n_models[pb] = m; n_inl[pb] = m > 0 ? n : 0; status[pb] = n == 7 ? FUND_SEVEN_POINT : FUND_TOO_FEW; iters[pb] = 0; groups[pb] = 0;
      rejected[pb] = 0; best[pb] = -1; best_root[pb] = -1; success[pb] = m > 0;
    }
    return;
  }
  const bool lmeds = n < 15;
  const int attempts = lmeds ? 1000 : 10000;
  if (t == 0) {
    sh_rng = ~0ull; sh_it = 0; sh_best_cnt = 0; sh_best_it = -1; sh_best_root = -1; sh_groups = 0; sh_rej = 0; sh_run = 0;
    sh_done = 0; sh_fail = 0; sh_best_med = CUDART_INF_F;
    sh_niters = lmeds ? max(hom_update_iters(B.conf, 0.45, 7, B.max_iters), 3) : max(B.max_iters, 1);
  }
  __syncthreads();
  float* rec = B.rec ? B.rec + (size_t)pb*4*B.rec_cap : nullptr;
  for (int c = 0; !sh_done; c++) {
    const int nch = min(FUND_CHUNK, 32 << min(c, 2));
    if (t == 0) sh_rng = hom_draw_groups<7>(sh_rng, n, nch, &sh_grp[0][0]);
    __syncthreads();
    if (t < nch) {                               // subset test and run7Point, one thread per draw
      float P1[14], P2[14];
      for (int i = 0; i < 7; i++) { const int r = sh_grp[t][i]; P1[2*i] = src[r].x; P1[2*i + 1] = src[r].y; P2[2*i] = dst[r].x; P2[2*i + 1] = dst[r].y; }
      int nm = -2;
      if (!hom_collinear<7>(P1) && !hom_collinear<7>(P2)) nm = fund_run7(P1, P2, sh_F[t]);
      sh_nm[t] = nm;
      for (int r = 0; r < 3; r++) sh_score[t][r] = 0;
      if (lmeds) {                               // the (n/2)-th smallest error of each model (n <= 14), ordered by bit pattern
        for (int r = 0; r < nm; r++) {
          int e[14];
          for (int i = 0; i < n; i++) {
            const int v = __float_as_int(fund_err(sh_F[t] + 9*r, src[i].x, src[i].y, dst[i].x, dst[i].y));
            int j = i; while (j > 0 && e[j - 1] > v) { e[j] = e[j - 1]; j--; }
            e[j] = v;
          }
          sh_score[t][r] = __int_as_float(e[n/2]);
        }
      }
    }
    if (!lmeds) {
      for (int tile0 = 0; tile0 < n; tile0 += FUND_THREADS) {   // inlier counts, points staged through shared memory
        const int tn = min(FUND_THREADS, n - tile0);
        __syncthreads();
        if (t < tn) { const float2 a = src[tile0 + t], b = dst[tile0 + t]; sh_tile[t] = make_float4(a.x, a.y, b.x, b.y); }
        __syncthreads();
        for (int q = warp; q < 3*nch; q += FUND_WARPS) {
          const int m = q/3, r = q - 3*m;
          if (r >= sh_nm[m]) continue;
          const double* F = sh_F[m] + 9*r;
          int cnt = 0;
          for (int j0 = 0; j0 < tn; j0 += 32) {
            const int j = j0 + lane;
            bool in = false;
            if (j < tn) { const float4 p = sh_tile[j]; in = fund_err(F, p.x, p.y, p.z, p.w) <= B.thr2; }
            cnt += __popc(__ballot_sync(0xffffffffu, in));
          }
          if (lane == 0) sh_score[m][r] += (float)cnt;
        }
      }
    }
    __syncthreads();
    if (t == 0) {                                // the sequential loop over this chunk in (draw, root) order
      int it = sh_it, niters = sh_niters, bcnt = sh_best_cnt, run = sh_run, grp = sh_groups, rej = sh_rej;
      float bmed = sh_best_med;
      bool done = false;
      for (int m = 0; m < nch; m++) {
        grp++;
        if (sh_nm[m] == -2) {
          rej++;
          if (++run >= attempts) { done = true; if (it == 0) sh_fail = 1; break; }
          continue;
        }
        run = 0;
        const int nm = sh_nm[m];
        if (rec && it < B.rec_cap) { float* rc = rec + 4*(size_t)it; rc[0] = (float)nm; for (int r = 0; r < nm; r++) rc[1 + r] = sh_score[m][r]; }
        for (int r = 0; r < nm; r++) {
          const float sc = sh_score[m][r];
          bool take;
          if (lmeds) { take = sc < bmed; if (take) bmed = sc; }
          else {
            const int cnt = (int)sc;
            take = cnt > max(bcnt, 6);
            if (take) { bcnt = cnt; niters = hom_update_iters(B.conf, (double)(n - cnt)/n, 7, niters); }
          }
          if (take) { sh_best_it = it; sh_best_root = r; for (int e = 0; e < 9; e++) sh_best[e] = sh_F[m][9*r + e]; }
        }
        if (++it >= niters) { done = true; break; }
      }
      sh_it = it; sh_niters = niters; sh_best_cnt = bcnt; sh_best_med = bmed; sh_run = run; sh_groups = grp; sh_rej = rej; sh_done = done;
    }
    __syncthreads();
  }
  if (sh_fail || sh_best_it < 0) {               // no model: F = 0, mask all zeros
    if (t == 0) {
      n_models[pb] = 0; n_inl[pb] = 0; status[pb] = FUND_FAILED; iters[pb] = sh_fail ? 0 : sh_it; groups[pb] = sh_groups;
      rejected[pb] = sh_rej; best[pb] = -1; best_root[pb] = -1; success[pb] = 0;
    }
    return;
  }
  float thr2 = B.thr2;
  if (lmeds) {
    double sigma = 2.5*1.4826*(1 + 5./(n - 7))*sqrt((double)sh_best_med);
    sigma = fmax(sigma, 0.001);
    thr2 = (float)(sigma*sigma);
  }
  if (t == 0) sh_ninl = 0;
  __syncthreads();
  int cnt = 0;
  for (int i = t; i < n; i += FUND_THREADS) {
    const bool in = fund_err(sh_best, src[i].x, src[i].y, dst[i].x, dst[i].y) <= thr2;
    mask[i] = in; cnt += in;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) atomicAdd(&sh_ninl, cnt);
  __syncthreads();
  if (t < 9) Fout[t] = sh_best[t];
  if (t == 0) {
    n_models[pb] = 1; n_inl[pb] = sh_ninl; status[pb] = lmeds ? FUND_LMEDS : FUND_OK; iters[pb] = sh_it; groups[pb] = sh_groups;
    rejected[pb] = sh_rej; best[pb] = sh_best_it; best_root[pb] = sh_best_root; success[pb] = lmeds ? sh_ninl >= 7 : 1;
  }
}

// klt_track_points: verified = the homography mask (0 on rows the forward-backward test dropped), keep = keep && verified
__global__ void ktp_post_kernel(int n, const uint8_t* __restrict__ verified, uint8_t* __restrict__ keep, int check, int* __restrict__ count) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool v = verified[i] != 0;
  if (check) keep[i] = keep[i] && v;
  if (v) atomicAdd(count, 1);
  if (check && keep[i]) atomicAdd(count + 1, 1);
}

// ---------------------------------------------------------------------------------------------------- trackDynamicKLT
// FeatureTracker::trackDynamicKLT with requiresSampling (FeatureTracker.cc:500-862,1018-1149) after the forward LK:
//  * a status-good point whose truncated pixel is outside the image is dropped and counted apart (cv::Mat::at out of range in
//    the reference);
//  * the detection-mask test reads detection_mask_impl as the feature is visited: the boundary mask, then the discs of the EARLIER
//    accepted features.  A point that would be accepted is a candidate of the greedy resolution of trackDynamic (td_link /
//    td_resolve, which marks a covered candidate TK_MASKED); any other point is TK_PENDING until the resolution is known and
//    then TK_MASKED when an earlier accepted disc covers its pixel, else TK_REJECTED.  Only TK_TRACKED and TK_REJECTED points are
//    counted, under their predicted label (integer atomics: order-independent);
//  * the tracked features leave ordered by (label, index) keys (tracks_per_object is an ordered map), through the bitonic sort;
//  * requiresSampling: one thread per detected object, from the per-label counters, the geriatric count and the float bounding
//    box (cv::boundingRect: floor of the extremes, width floor(max) - floor(min) + 1) against the inner bounding box (cv::Rect
//    intersection, int areas, calculateIoU);
//  * goodFeaturesToTrack(mono, max_features, quality, min_distance, (motion_mask == id) & detection_mask_impl) per sampled object:
//    the eigen image is computed once (the stages of dynofront_detect_static, no CLAHE).  Under THRESH_TOZERO a pixel is a corner
//    candidate iff it is a 3x3 local maximum of the raw eigen image above the object's threshold (the threshold is >= 0 whenever a
//    masked pixel can pass it), so one local-maximum pass serves every object; the per-object parts are the masked maximum, the
//    threshold and the candidate lists, sorted together with keys (object rank, value, address);
//  * the minDistance / maxCorners filter one CTA per list, the range-tree ANMS of every sampled object in one launch (response 1
//    for all, KeyPoint::convert: the visiting order is P_n), then the new features in objects order, each in ANMS order, the
//    shrunken-image test before an id is taken.
enum { TK_CAND = 0, TK_TRACKED = 1, TK_MASKED = 2, TK_REJECTED = 3, TK_OUTSIDE = 4, TK_LOST = 5, TK_PENDING = 6 };
constexpr int TK_ADDR_BITS = 26;          // pixel address bits of the corner keys: images up to 2^26 pixels
// one status row: rows[0] is label 0, rows[1 + o] objects[o]
struct TkRow { int exists, prev, track, shrunk, diff, bg, geri; unsigned bx0, by0, bx1, by1, max_eig; int is_new, resampled, sampled, num_sampled; };
struct TkCounters { int tracked, outside, cand, features; };
struct TkParams {
  dynofront_track_params track; int max_age, expiry, max_features, min_tracks; double quality, min_iou;
};
__device__ __forceinline__ int tk_slot(const int* objs, int nobj, int lab) {
  for (int o = 0; o < nobj; o++) if (objs[o] == lab) return o;
  return -1;
}
__global__ void tk_init_kernel(int nrows, TkRow* rows, TkCounters* cnt, int* cand) {
  const int r = threadIdx.x;
  if (r < nrows) { TkRow z = {}; z.bx0 = z.by0 = 0xffffffffu; rows[r] = z; }
  if (r < ST_MAXOBJ) cand[r] = 0;
  if (r == 0) *cnt = TkCounters{};
}
__global__ void tk_gather_kernel(int n, const float* __restrict__ next, const uint8_t* __restrict__ st, const int32_t* __restrict__ plab,
                                 const int32_t* __restrict__ page, const int32_t* __restrict__ mask, const uint8_t* __restrict__ det, int W, int H,
                                 TkParams P, int* fx, int* fy, int* state, int32_t* oage, int32_t* olab) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double kx = (double)next[2*i], ky = (double)next[2*i + 1];
  int s = TK_LOST, x = 0, y = 0, lab = 0;
  if (st[i]) {
    s = TK_OUTSIDE;
    if (kx > -1.0 && kx < (double)W && ky > -1.0 && ky < (double)H) {       // the truncated pixel is inside the image
      x = (int)kx; y = (int)ky;
      lab = mask[(size_t)y*W + x];
      if (det && det[(size_t)y*W + x] == 0) s = TK_MASKED;                   // the boundary mask: not counted
      else {
        const bool contained = kx >= 0.0 && kx < (double)W && ky >= 0.0 && ky < (double)H;
        const bool ok = contained && lab != 0 && lab == plab[i] && within_shrunken(kx, ky, H, W, P.track.shrink_row, P.track.shrink_col) &&
                        page[i] + 1 <= P.max_age;
        s = ok ? TK_CAND : TK_PENDING;
      }
    }
  }
  fx[i] = x; fy[i] = y; state[i] = s; oage[i] = page[i] + 1; olab[i] = lab;
}
// after td_resolve: the pending points learn whether an earlier accepted disc covers them, the counted points are counted, the
// accepted ones get their sort key; measured flow = kp_current - keypoint in double
__global__ void tk_count_kernel(int n, const float* __restrict__ prev, const float* __restrict__ next, const int* __restrict__ fx, const int* __restrict__ fy,
                                int* state, const int* __restrict__ cell, const int* __restrict__ lnext, Disc disc, int W, int H,
                                const int32_t* __restrict__ plab, const int32_t* __restrict__ oage, const int32_t* __restrict__ olab,
                                const int* __restrict__ objs, int nobj, TkParams P, TkRow* rows, TkCounters* cnt, unsigned long long* keys, double* flow) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  int s = state[i];
  if (s == TK_PENDING) {
    bool covered = false;
    disc_walk(disc, fx[i], fy[i], W, H, [&](int xx, int yy) {
      for (int j = cell[(size_t)yy*W + xx]; j >= 0; j = lnext[j]) if (j < i && state[j] == TK_TRACKED) { covered = true; break; }
      return covered;
    });
    s = covered ? TK_MASKED : TK_REJECTED;
    state[i] = s;
  }
  const double kx = (double)next[2*i], ky = (double)next[2*i + 1];
  flow[2*i] = s == TK_TRACKED ? kx - (double)prev[2*i] : 0.0;
  flow[2*i + 1] = s == TK_TRACKED ? ky - (double)prev[2*i + 1] : 0.0;
  if (s == TK_OUTSIDE) atomicAdd(&cnt->outside, 1);
  if (s != TK_TRACKED && s != TK_REJECTED) return;
  const int lab = olab[i];
  if (s == TK_TRACKED) {
    const unsigned long long a = ((unsigned long long)((unsigned)lab ^ 0x80000000u) << 32) | (unsigned)i;   // ascending (label, index)
    keys[atomicAdd(&cnt->tracked, 1)] = ~a;                                                                  // (the sort is descending)
  }
  const int o = lab == 0 ? -1 : tk_slot(objs, nobj, lab);
  if (lab != 0 && o < 0) return;                                   // a label that is not listed has no row in the output
  TkRow* r = rows + (o + 1);
  const bool contained = kx >= 0.0 && kx < (double)W && ky >= 0.0 && ky < (double)H;
  r->exists = 1;
  atomicAdd(&r->prev, 1);
  if (lab == 0) atomicAdd(&r->bg, 1);
  if (lab != plab[i]) atomicAdd(&r->diff, 1);
  if (contained && lab != 0 && lab == plab[i] && !within_shrunken(kx, ky, H, W, P.track.shrink_row, P.track.shrink_col)) atomicAdd(&r->shrunk, 1);
  if (s == TK_TRACKED) {
    atomicAdd(&r->track, 1);
    if (oage[i] > P.expiry) atomicAdd(&r->geri, 1);
    atomicMin(&r->bx0, f32_order(next[2*i])); atomicMax(&r->bx1, f32_order(next[2*i]));
    atomicMin(&r->by0, f32_order(next[2*i + 1])); atomicMax(&r->by1, f32_order(next[2*i + 1]));
  }
}
// requiresSampling, one thread per detected object in the given order; K[o] = corners needed (0: not sampled)
__global__ void tk_decide_kernel(int nobj, const int* __restrict__ bb, TkParams P, TkRow* rows, int* K) {
  const int o = threadIdx.x;
  if (o >= nobj) return;
  TkRow* r = rows + 1 + o;
  bool sample;
  if (!r->exists) { sample = true; r->exists = 1; r->is_new = 1; }          // getObjectStatus makes the row
  else if (r->track == 0) sample = false;                                    // a row but no tracked feature: skipped
  else {
    const bool old = (double)r->geri/(double)r->track > 0.8;
    const bool few = r->track < P.min_tracks;
    const int tx = (int)floorf(f32_unorder(r->bx0)), ty = (int)floorf(f32_unorder(r->by0));
    const int tw = (int)floorf(f32_unorder(r->bx1)) - tx + 1, th = (int)floorf(f32_unorder(r->by1)) - ty + 1;
    const int ax = bb[4*o], ay = bb[4*o + 1], aw = bb[4*o + 2], ah = bb[4*o + 3];
    int iw = 0, ih = 0;                                                      // cv::Rect operator& (empty: Rect())
    if (aw > 0 && ah > 0 && tw > 0 && th > 0) {
      iw = min(ax + aw, tx + tw) - max(ax, tx); ih = min(ay + ah, ty + th) - max(ay, ty);
      if (iw <= 0 || ih <= 0) iw = ih = 0;
    }
    const double inter = (double)(iw*ih), uni = (double)(aw*ah + tw*th) - inter;
    const double iou = uni == 0 ? 0.0 : inter/uni;
    sample = old || few || iou < P.min_iou;
  }
  if (sample) r->resampled = 1;
  r->sampled = sample ? 1 : 0;
  K[o] = sample ? max(P.max_features - r->track, 0) : 0;
}
// the minimum eigenvalue per pixel and, per sampled object, its maximum under (motion_mask == id) & detection_mask_impl
__global__ void tk_eig_kernel(const float* __restrict__ box, size_t npx, const int32_t* __restrict__ mask, const uint8_t* __restrict__ det,
                              const int* __restrict__ objs, int nobj, TkRow* rows, float* __restrict__ eig) {
  __shared__ int s_obj[ST_MAXOBJ]; __shared__ unsigned s_max[ST_MAXOBJ];
  if (threadIdx.x < ST_MAXOBJ) { s_obj[threadIdx.x] = threadIdx.x < nobj && rows[1 + threadIdx.x].sampled ? objs[threadIdx.x] : 0; s_max[threadIdx.x] = 0; }
  __syncthreads();
  const size_t p = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  if (p < npx) {
    const float a = box[p]*0.5f, b = box[npx + p], cc = box[2*npx + p]*0.5f;
    const float e = (a + cc) - sqrtf((a - cc)*(a - cc) + b*b);
    eig[p] = e;
    const int lab = mask[p];
    const int o = (lab != 0 && det[p]) ? tk_slot(s_obj, nobj, lab) : -1;
    if (o >= 0) atomicMax(&s_max[o], f32_order(e));
  }
  __syncthreads();
  if ((int)threadIdx.x < nobj && s_max[threadIdx.x]) atomicMax(&rows[1 + threadIdx.x].max_eig, s_max[threadIdx.x]);
}
// the candidates of every sampled object: a masked 3x3 local maximum of the raw eigen image above (float)(maxVal * quality), the
// 1-px border excluded; key = (63 - object rank) << 58 | value (order-preserving) << 26 | address, sorted descending
__global__ void tk_cand_kernel(const float* __restrict__ eig, int W, int H, const int32_t* __restrict__ mask, const uint8_t* __restrict__ det,
                               const int* __restrict__ objs, int nobj, const TkRow* __restrict__ rows, double quality, unsigned long long* __restrict__ keys,
                               TkCounters* cnt, int* __restrict__ cand) {
  __shared__ int s_obj[ST_MAXOBJ]; __shared__ float s_thr[ST_MAXOBJ];
  const int t = threadIdx.y*blockDim.x + threadIdx.x;
  if (t < ST_MAXOBJ) {
    s_obj[t] = t < nobj && rows[1 + t].sampled ? objs[t] : 0;
    const unsigned m = t < nobj ? rows[1 + t].max_eig : 0u;
    s_thr[t] = (float)((double)(m ? f32_unorder(m) : 0.f)*quality);          // minMaxLoc over an empty mask leaves maxVal = 0
  }
  __syncthreads();
  const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
  if (x < 1 || y < 1 || x >= W - 1 || y >= H - 1) return;
  const size_t p = (size_t)y*W + x;
  const int lab = mask[p];
  if (lab == 0 || !det[p]) return;
  const int o = tk_slot(s_obj, nobj, lab);
  if (o < 0) return;
  const float v = eig[p];
  if (!(v > s_thr[o])) return;
  float d = v;
  for (int j = -1; j <= 1; j++) for (int i = -1; i <= 1; i++) d = fmaxf(d, eig[(size_t)(y + j)*W + x + i]);
  if (v != d) return;
  atomicAdd(&cand[o], 1);
  keys[atomicAdd(&cnt->cand, 1)] = ((unsigned long long)(63 - o) << 58) | ((unsigned long long)f32_order(v) << TK_ADDR_BITS) | (unsigned long long)p;
}
__global__ void tk_offsets_kernel(int nobj, const int* cand, int* off) {
  if (threadIdx.x != 0) return;
  int run = 0;
  for (int o = 0; o < nobj; o++) { off[o] = run; run += cand[o]; }
}
// the output features, one CTA: the tracked ones in (label, index) order, then the new ones object after object in ANMS order,
// the shrunken-image test before an id is taken; tracklet ids count up from base_id
__global__ void __launch_bounds__(1024) tk_construct_kernel(const unsigned long long* __restrict__ tkeys, const float* __restrict__ next,
                                                            const int32_t* __restrict__ oage, const int32_t* __restrict__ olab, const int64_t* __restrict__ ptid,
                                                            const int* __restrict__ objs, int nobj, const int* __restrict__ off, const int* __restrict__ nsel,
                                                            const int* __restrict__ sel, const int* __restrict__ corners, int W, int H, TkParams P,
                                                            long long base_id, TkRow* rows, TkCounters* cnt, double* okp, int32_t* oage_out,
                                                            long long* otid, int32_t* olab_out, int32_t* osrc) {
  __shared__ int s_pre[ST_MAXOBJ + 1];
  const int ntr = cnt->tracked;
  for (int q = threadIdx.x; q < ntr; q += 1024) {
    const int i = (int)~(unsigned)tkeys[q];
    okp[2*(size_t)q] = (double)next[2*i]; okp[2*(size_t)q + 1] = (double)next[2*i + 1];
    oage_out[q] = oage[i]; otid[q] = ptid[i]; olab_out[q] = olab[i]; osrc[q] = i;
  }
  if (threadIdx.x == 0) {
    int run = 0;
    for (int o = 0; o < nobj; o++) { s_pre[o] = run; run += nsel[o]; rows[1 + o].num_sampled = nsel[o]; }
    s_pre[nobj] = run;
  }
  __syncthreads();
  const int S = s_pre[nobj];
  int base = 0;
  for (int q0 = 0; q0 < S; q0 += 1024) {
    const int q = q0 + threadIdx.x;
    int a = 0, x = 0, y = 0, o = 0;
    if (q < S) {
      while (q >= s_pre[o + 1]) o++;
      const int c = sel[off[o] + (q - s_pre[o])];
      x = corners[2*(off[o] + c)]; y = corners[2*(off[o] + c) + 1];
      a = within_shrunken((double)x, (double)y, H, W, P.track.shrink_row, P.track.shrink_col) ? 1 : 0;
    }
    const int rank = cta_rank(a, base);
    if (a) {
      const size_t d = (size_t)ntr + rank;
      okp[2*d] = x; okp[2*d + 1] = y; oage_out[d] = 0; otid[d] = base_id + rank; olab_out[d] = objs[o]; osrc[d] = -1;
    }
  }
  if (threadIdx.x == 0) cnt->features = ntr + base;
}

// ---------------------------------------------------------------------------------------------------- object boundary mask
// vision_tools::computeObjectMaskBoundaryMask on the resident current motion mask, in the restatement of boundary.cuh.  Both
// kernels work on 64 x 32 pixel tiles with 256 threads; the per-label extents are folded per thread (runs of one label down
// its column), then per CTA in shared memory, then once per (CTA, label) into the global tables with atomicMax, which makes
// them independent of the order.  Global table: [0, 1024) the extents of M == j, [1024, 2048) those of erode(T) == j, [2048]
// the flag of a label outside [0, 255].
#define BD_TW 64
#define BD_TH 32
#define BD_THREADS 256
#define BD_RS (BD_THREADS/BD_TW)          // row step between the pixels of one thread
#define BD_PP (BD_TH/BD_RS)               // pixels per thread
#define BD_TAB (8*(BOUNDARY_MAX_LABEL + 1) + 1)
#define BD_CHUNKS ((BD_TW + 2*BOUNDARY_MAX_THICKNESS + 31)/32)   // 32-column chunks of the widest tile row
#define BD_LEVELS 8                       // sparse-table levels of the widest run, 2*BOUNDARY_MAX_THICKNESS + 1 pixels
struct BdRows {                           // one element: radius, top level, row half widths per |dy|, and the |dy| range [lo, hi] whose
  int r, top, hw[BOUNDARY_MAX_THICKNESS + 1], lo[BD_LEVELS], hi[BD_LEVELS];     // runs take each level (hw falls with |dy|)
};
struct BdElem { BdRows in, out; };        // E_10 (erosion) and E_t (dilation)
__device__ __forceinline__ void bd_run_add(int (*s)[4], int lab, int W, int H, int x, int y0, int y1) {
  atomicMax(&s[lab][0], W - x); atomicMax(&s[lab][1], H - y0); atomicMax(&s[lab][2], x + 1); atomicMax(&s[lab][3], y1 + 1);
}
__device__ __forceinline__ void bd_flush(int (*s)[4], int* g) {
  __syncthreads();
  for (int l = threadIdx.x; l <= BOUNDARY_MAX_LABEL; l += BD_THREADS)
    if (s[l][2]) for (int f = 0; f < 4; f++) atomicMax(&g[4*l + f], s[l][f]);
}
// T (the 1x11 column max), the label check and the extents of M == j
__global__ void __launch_bounds__(BD_THREADS) bd_scan_kernel(const int32_t* __restrict__ M, int W, int H, uint8_t* __restrict__ T, int* tab) {
  __shared__ int s[BOUNDARY_MAX_LABEL + 1][4];
  for (int i = threadIdx.x; i < 4*(BOUNDARY_MAX_LABEL + 1); i += BD_THREADS) (&s[0][0])[i] = 0;
  __syncthreads();
  const int x = blockIdx.x*BD_TW + threadIdx.x % BD_TW, y0 = blockIdx.y*BD_TH + (threadIdx.x/BD_TW)*BD_PP;
  bool bad = false;
  if (x < W) {
    int run = 0, ry0 = 0, ry1 = 0;
    for (int y = y0; y < min(y0 + BD_PP, H); y++) {
      T[(size_t)y*W + x] = (uint8_t)boundary_column_max(M, W, H, x, y);
      const int32_t v = M[(size_t)y*W + x];
      bad |= !boundary_label_ok(v);
      const int lab = boundary_label_ok(v) ? v : 0;
      if (lab == run) { ry1 = y; continue; }
      if (run) bd_run_add(s, run, W, H, x, ry0, ry1);
      run = lab; ry0 = ry1 = y;
    }
    if (run) bd_run_add(s, run, W, H, x, ry0, ry1);
  }
  if (bad) tab[BD_TAB - 1] = 1;
  bd_flush(s, tab);
}
// One morphology pass over the tile: the max (dilation) or min (erosion) of T over the element of radius r, into acc.  The tile
// and a halo of r are loaded with a border value that never wins; then, level by level, a sparse table of row maxima / minima is
// built in place (level k holds the op over 2^k pixels starting at each column) and every element row whose run 2w+1 takes
// level k is answered with two overlapping windows: O(r) per pixel rather than O(r^2).
template <bool MAX>
__device__ void bd_pass(uint8_t* buf, const uint8_t* __restrict__ T, int W, int H, int X0, int Y0, const BdRows& E, int tx, int ty0, int* acc) {
  const int r = E.r, BW = BD_TW + 2*r, BH = BD_TH + 2*r;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int row = warp; row < BH; row += BD_THREADS/32) {     // one warp per row, all of its loads in flight at once
    const int gy = Y0 - r + row;
    const bool in_y = gy >= 0 && gy < H;
    uint8_t* rp = buf + row*BW;
    int v[BD_CHUNKS];
#pragma unroll
    for (int c = 0; c < BD_CHUNKS; c++) {
      const int bx = 32*c + lane, gx = X0 - r + bx;
      v[c] = (in_y && bx < BW && gx >= 0 && gx < W) ? T[(size_t)gy*W + gx] : (MAX ? 0 : 255);
    }
#pragma unroll
    for (int c = 0; c < BD_CHUNKS; c++) if (32*c + lane < BW) rp[32*c + lane] = (uint8_t)v[c];
  }
  __syncthreads();
  for (int k = 0; k <= E.top; k++) {
    if (k > 0) {                          // one warp per row: the whole row of level k - 1 is read before level k is written
      const int half = 1 << (k - 1), last = BW - (1 << k);
      for (int row = warp; row < BH; row += BD_THREADS/32) {
        uint8_t* rp = buf + row*BW;
        int v[BD_CHUNKS];
#pragma unroll
        for (int c = 0; c < BD_CHUNKS; c++) {
          const int x = 32*c + lane;
          v[c] = x <= last ? (MAX ? max(rp[x], rp[x + half]) : min(rp[x], rp[x + half])) : 0;
        }
        __syncwarp();
#pragma unroll
        for (int c = 0; c < BD_CHUNKS; c++) if (32*c + lane <= last) rp[32*c + lane] = (uint8_t)v[c];
        __syncwarp();
      }
      __syncthreads();
    }
    for (int a = E.lo[k]; a <= E.hi[k]; a++) {
      const int o1 = -E.hw[a], o2 = E.hw[a] - (1 << k) + 1;
      for (int dy = -a; dy <= a; dy += (a ? 2*a : 1)) {
        const uint8_t* rp = buf + (ty0 + r + dy)*BW + tx + r;
#pragma unroll
        for (int j = 0; j < BD_PP; j++) {
          const int v1 = rp[j*BD_RS*BW + o1], v2 = rp[j*BD_RS*BW + o2];
          acc[j] = MAX ? max(acc[j], max(v1, v2)) : min(acc[j], min(v1, v2));
        }
      }
    }
    __syncthreads();
  }
}
// the boundary mask and the extents of erode(T) == j
__global__ void __launch_bounds__(BD_THREADS) bd_morph_kernel(const uint8_t* __restrict__ T, int W, int H, const __grid_constant__ BdElem E,
                                                              uint8_t* __restrict__ out, int* tab) {
  extern __shared__ uint8_t bd_buf[];
  __shared__ int s[BOUNDARY_MAX_LABEL + 1][4];
  for (int i = threadIdx.x; i < 4*(BOUNDARY_MAX_LABEL + 1); i += BD_THREADS) (&s[0][0])[i] = 0;
  const int X0 = blockIdx.x*BD_TW, Y0 = blockIdx.y*BD_TH, tx = threadIdx.x % BD_TW, ty0 = threadIdx.x/BD_TW;
  int ero[BD_PP], dil[BD_PP];
#pragma unroll
  for (int j = 0; j < BD_PP; j++) { ero[j] = 255; dil[j] = 0; }
  bd_pass<false>(bd_buf, T, W, H, X0, Y0, E.in, tx, ty0, ero);
  bd_pass<true>(bd_buf, T, W, H, X0, Y0, E.out, tx, ty0, dil);
  const int x = X0 + tx;
  int run = 0, ry0 = 0, ry1 = 0;
#pragma unroll
  for (int j = 0; j < BD_PP; j++) {
    const int y = Y0 + ty0 + j*BD_RS;
    if (x >= W || y >= H) continue;
    const size_t p = (size_t)y*W + x;
    out[p] = boundary_value(T[p], dil[j], ero[j]);
    const int lab = ero[j];
    if (lab == run) { ry1 = y; continue; }
    if (run) bd_run_add(s, run, W, H, x, ry0, ry1);
    run = lab; ry0 = ry1 = y;
  }
  if (run) bd_run_add(s, run, W, H, x, ry0, ry1);
  bd_flush(s, tab + 4*(BOUNDARY_MAX_LABEL + 1));
}
static BdRows bd_rows(int r) {
  BdRows e; e.r = r; e.top = boundary_level(r);
  for (int k = 0; k < BD_LEVELS; k++) { e.lo[k] = r + 1; e.hi[k] = -1; }
  for (int a = 0; a <= r; a++) {
    e.hw[a] = boundary_ellipse_hw(r, a);
    const int k = boundary_level(e.hw[a]);
    e.lo[k] = std::min(e.lo[k], a); e.hi[k] = std::max(e.hi[k], a);
  }
  return e;
}
static size_t bd_smem(int t) { const int R = std::max(t, BOUNDARY_INNER); return (size_t)(BD_TW + 2*R)*(BD_TH + 2*R); }

// ---------------------------------------------------------------------------------------------------- host API
extern "C" {

const char* dynofront_last_error(dynofront_handle h) { return h ? h->err.c_str() : "null handle"; }

int dynofront_create(int device, int width, int height, dynofront_handle* out) {
  if (!out || width <= 0 || height <= 0) return -1;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return -3;
  cudaDeviceProp prop; if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) return -3;   // sm_90a code only
  dynofront_ctx* h = new dynofront_ctx(); h->dev = device; h->W = width; h->H = height;
  cudaSetDevice(device);
  if (cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking) != cudaSuccess) { delete h; return -3; }
  cudaEventCreate(&h->e0); cudaEventCreate(&h->e1);
  const size_t npx = (size_t)width*height;
  if (grow(h, h->flow, 2*npx, h->mask, npx, h->det, npx, h->det_work, npx, h->trk, npx, h->trk_idx, npx, h->cell, npx, h->nextid, 1,
           h->tile_cnt, ((npx + ST_TILE - 1)/ST_TILE)*ST_MAXOBJ, h->obj_tot, ST_MAXOBJ, h->d_objs, ST_MAXOBJ, h->d_zero, ST_MAXOBJ,
           h->pmask, npx, h->pflow, 2*npx, h->cmask, npx, h->pflag, 1)) { dynofront_destroy(h); return -3; }
  *out = h;
  return 0;
}
int dynofront_destroy(dynofront_handle h) {
  if (!h) return -1;
  cudaSetDevice(h->dev);
  if (h->e0) cudaEventDestroy(h->e0); if (h->e1) cudaEventDestroy(h->e1);
  if (h->s) cudaStreamDestroy(h->s);
  if (h->bd_host) cudaFreeHost(h->bd_host);
  delete h; return 0;                                           // (the buffers free their device memory)
}
int dynofront_set_frame(dynofront_handle h, const float* flow, const int32_t* motion_mask, const uint8_t* detection_mask) {
  if (!h) return -1; cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H;
  if (flow) FCK(cudaMemcpyAsync(h->flow, flow, 2*npx*sizeof(float), cudaMemcpyHostToDevice, h->s));
  if (motion_mask) FCK(cudaMemcpyAsync(h->mask, motion_mask, npx*sizeof(int32_t), cudaMemcpyHostToDevice, h->s));
  if (detection_mask) { FCK(cudaMemcpyAsync(h->det, detection_mask, npx, cudaMemcpyHostToDevice, h->s)); h->has_det = true; }
  else h->has_det = false;
  h->det_work_valid = false;
  h->has_depth = false; h->has_right = false; h->has_frame = h->has_frame || motion_mask;
  if (motion_mask) h->mask_propagated = false;
  FCK(cudaStreamSynchronize(h->s));
  return 0;
}
static int build_pyramid(dynofront_ctx* h, int which, const uint8_t* host_img, int max_level, int win, bool with_deriv);
// Streaming: the frame that was current becomes the previous one WITHOUT moving data (the device buffers swap roles:
// flow / motion mask for propogateMask, gray pyramid + Scharr derivatives for the KLT), then only the new frame's images
// cross PCIe (asynchronously when the host buffers are pinned, dynofront_pin_host) and only its pyramid is built.
int dynofront_next_frame(dynofront_handle h, const uint8_t* gray, const float* flow, const int32_t* motion_mask, const uint8_t* detection_mask) {
  if (!h || !gray || !flow || !motion_mask) return -1;
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H;
  std::swap(h->flow, h->pflow); std::swap(h->mask, h->pmask);
  FCK(cudaMemcpyAsync(h->flow, flow, 2*npx*sizeof(float), cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->mask, motion_mask, npx*sizeof(int32_t), cudaMemcpyHostToDevice, h->s));
  if (detection_mask) { FCK(cudaMemcpyAsync(h->det, detection_mask, npx, cudaMemcpyHostToDevice, h->s)); h->has_det = true; } else h->has_det = false;
  h->det_work_valid = false;
  h->has_depth = false; h->has_frame = true; h->mask_propagated = false;
  h->have_prev = h->have_cur; h->have_cur = true;
  if (!h->lw.empty()) { std::swap(h->pyr[0], h->pyr[1]); std::swap(h->der, h->der2); }
  h->have_pyr = h->have_pyr_cur; h->have_pyr_cur = true;
  if (build_pyramid(h, 1, gray, 5, 21, true)) return -3;       // (levels that are too small for a window are simply never read)
  return 0;                                                     // no synchronisation: the next call's work is ordered behind on the stream
}
static void prepare_det_work(dynofront_ctx* h) {
  const size_t npx = (size_t)h->W*h->H;
  if (h->has_det) cudaMemcpyAsync(h->det_work, h->det, npx, cudaMemcpyDeviceToDevice, h->s);
  else fill_u8_kernel<<<(unsigned)((npx + 255)/256), 256, 0, h->s>>>(h->det_work, npx, 255);
  h->det_work_valid = true;
}

int dynofront_track_dynamic(dynofront_handle h, int32_t n, const double* kp, const int32_t* lab, const int32_t* age, const int64_t* tid,
                            const dynofront_track_params* prm, int64_t* next_tracklet_id, uint8_t* accepted, double* pred_kp, double* flow_out,
                            int32_t* oage, int64_t* otid, int32_t* olab, uint8_t* det_out, uint8_t* trk_out) {
  if (!h || !prm || n < 0 || !next_tracklet_id) return -1;
  if (prm->min_distance < 0 || prm->min_distance > 15) { h->err = "min_distance must be in [0,15]"; return -1; }
  cudaSetDevice(h->dev);
  const size_t cap = feature_cap(n);
  if (grow(h, h->f_kp, 2*cap, h->f_lab, cap, h->f_age, cap, h->f_tid, cap, h->f_x, cap, h->f_y, cap, h->f_state, cap, h->f_next, cap,
           h->f_pred, 2*cap, h->f_flow, 2*cap, h->f_oage, cap, h->f_otid, cap, h->f_olab, cap, h->f_acc, cap)) return -3;
  const size_t npx = (size_t)h->W*h->H; const int W = h->W, H = h->H;
  const Disc disc = make_disc(prm->min_distance);
  FCK(cudaMemcpyAsync(h->f_kp, kp, 2*(size_t)n*8, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->f_lab, lab, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->f_age, age, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->f_tid, tid, (size_t)n*8, cudaMemcpyHostToDevice, h->s));
  long long nid = *next_tracklet_id;
  FCK(cudaMemcpyAsync(h->nextid, &nid, 8, cudaMemcpyHostToDevice, h->s));
  prepare_det_work(h);
  fill_i32_kernel<<<(unsigned)((npx + 255)/256), 256, 0, h->s>>>(h->cell, npx, -1);
  fill_i32_kernel<<<(unsigned)((npx + 255)/256), 256, 0, h->s>>>(h->trk_idx, npx, 0);
  if (n > 0) {
    const int g = (n + 127)/128;
    td_candidate_kernel<<<g, 128, 0, h->s>>>(n, h->f_kp, h->f_lab, h->f_age, h->flow, h->mask, h->has_det ? h->det.p : nullptr, W, H, *prm,
                                             h->f_x, h->f_y, h->f_state, h->f_pred, h->f_flow, h->f_oage, h->f_olab);
    td_link_kernel<<<g, 128, 0, h->s>>>(n, h->f_x, h->f_y, h->f_state, W, h->cell, h->f_next);
    td_resolve_kernel<<<1, 1024, 0, h->s>>>(n, h->f_x, h->f_y, h->f_state, h->cell, h->f_next, W, H, disc, prm->max_dynamic_feature_age,
                                            h->f_tid, h->f_oage, h->f_otid, h->f_acc, h->nextid, 2);
    td_clear_rejected_kernel<<<g, 128, 0, h->s>>>(n, h->f_acc, h->f_pred, h->f_flow, h->f_olab);
    td_masks_kernel<<<g, 128, 0, h->s>>>(n, h->f_x, h->f_y, h->f_acc, W, H, disc, h->det_work, h->trk_idx);
  }
  td_trk_final_kernel<<<(unsigned)((npx + 255)/256), 256, 0, h->s>>>(npx, h->trk_idx, h->f_olab, h->trk);
  if (n) {
    if (pred_kp) FCK(cudaMemcpyAsync(pred_kp, h->f_pred, 2*(size_t)n*8, cudaMemcpyDeviceToHost, h->s));
    if (flow_out) FCK(cudaMemcpyAsync(flow_out, h->f_flow, 2*(size_t)n*8, cudaMemcpyDeviceToHost, h->s));
    if (accepted) FCK(cudaMemcpyAsync(accepted, h->f_acc, n, cudaMemcpyDeviceToHost, h->s));
    if (oage) FCK(cudaMemcpyAsync(oage, h->f_oage, (size_t)n*4, cudaMemcpyDeviceToHost, h->s));
    if (otid) FCK(cudaMemcpyAsync(otid, h->f_otid, (size_t)n*8, cudaMemcpyDeviceToHost, h->s));
    if (olab) FCK(cudaMemcpyAsync(olab, h->f_olab, (size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  }
  FCK(cudaMemcpyAsync(&nid, h->nextid, 8, cudaMemcpyDeviceToHost, h->s));
  if (det_out) FCK(cudaMemcpyAsync(det_out, h->det_work, npx, cudaMemcpyDeviceToHost, h->s));
  if (trk_out) FCK(cudaMemcpyAsync(trk_out, h->trk, npx, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  *next_tracklet_id = nid;
  return 0;
}

int dynofront_sample_candidates(dynofront_handle h, int32_t nobj, const int32_t* objects, const dynofront_track_params* prm, int32_t* counts,
                                int32_t* offsets, int32_t* zero_flow, int32_t* indices, int64_t capacity) {
  if (!h || !prm || nobj < 0 || !counts || !offsets || (nobj && !objects)) return -1;
  if (check_objects(h, nobj, objects)) return -1;
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H; const int ntiles = (int)((npx + ST_TILE - 1)/ST_TILE);
  if (!h->det_work_valid) prepare_det_work(h);
  if (grow(h, h->d_idx, (size_t)capacity)) return -3;
  FCK(cudaMemcpyAsync(h->d_objs, objects, (size_t)nobj*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemsetAsync(h->d_zero, 0, ST_MAXOBJ*4, h->s));
  sc_count_kernel<<<ntiles, ST_TILE, 0, h->s>>>(npx, h->W, h->H, h->det_work, h->mask, h->flow, h->d_objs, nobj, *prm, h->tile_cnt, h->d_zero);
  sc_scan_kernel<<<1, ST_MAXOBJ, 0, h->s>>>(ntiles, nobj, h->tile_cnt, h->obj_tot);
  std::vector<int> tot(ST_MAXOBJ), zc(ST_MAXOBJ);
  FCK(cudaMemcpyAsync(tot.data(), h->obj_tot, ST_MAXOBJ*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(zc.data(), h->d_zero, ST_MAXOBJ*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaStreamSynchronize(h->s));
  int run = 0;
  for (int o = 0; o < nobj; o++) { counts[o] = tot[o]; offsets[o] = run; run += tot[o]; if (zero_flow) zero_flow[o] = zc[o]; }
  if (indices && capacity > 0) {
    FCK(cudaMemcpyAsync(h->obj_tot, offsets, (size_t)nobj*4, cudaMemcpyHostToDevice, h->s));
    sc_scatter_kernel<<<ntiles, ST_TILE, 0, h->s>>>(npx, h->W, h->H, h->det_work, h->mask, h->flow, h->d_objs, nobj, *prm, h->tile_cnt, h->obj_tot,
                                                    h->d_idx, (long long)capacity);
    const size_t ncopy = std::min<size_t>((size_t)run, (size_t)capacity);
    FCK(cudaMemcpyAsync(indices, h->d_idx, ncopy*4, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaStreamSynchronize(h->s));
  }
  FCK(cudaGetLastError());
  return 0;
}

// the work arrays of the ordered resolver (anms_range_tree_kernel, dt_gftt_select_kernel) hold at least a frame of points,
// indexed by int
static int grow_resolver(dynofront_ctx* h, size_t points) {
  const size_t cap = std::max(points, (size_t)h->W*h->H);
  if (cap > 0x7fffffff) { h->err = "too many key-points"; return -3; }
  return grow(h, h->sel_px, cap, h->sel_py, cap, h->sel_orig, cap, h->sel_next, cap, h->sel_out, cap);
}

int dynofront_anms_range_tree(dynofront_handle h, int32_t n_lists, const int32_t* offsets, const int32_t* xy, const int32_t* k_needed,
                              const float* tolerance, int32_t cols, int32_t rows, int32_t* selected, int32_t* n_selected, float* ms_device) {
  if (!h || n_lists < 0 || (n_lists && (!offsets || !k_needed || !tolerance || !n_selected)) || cols <= 0 || rows <= 0) return -1;
  cudaSetDevice(h->dev);
  if (n_lists == 0) return 0;
  if (offsets[0] != 0) { h->err = "offsets[0] must be 0"; return -1; }
  std::vector<int> cnt(n_lists);
  for (int l = 0; l < n_lists; l++) {
    cnt[l] = offsets[l + 1] - offsets[l];
    if (cnt[l] < 0) { h->err = "offsets must not decrease"; return -1; }
    if (k_needed[l] < 0) { h->err = "k_needed must be >= 0"; return -1; }
  }
  const size_t total = (size_t)offsets[n_lists];
  if (total && (!xy || !selected)) return -1;
  for (size_t i = 0; i < 2*total; i++) if (xy[i] < 0 || xy[i] > 65535) { h->err = "key-point coordinates must be in [0, 65535]"; return -1; }
  for (int l = 0; l < n_lists; l++) {
    if (cnt[l] == 0 || k_needed[l] < 2) continue;
    int cmax = 0;
    for (int i = 2*offsets[l]; i < 2*offsets[l + 1]; i++) cmax = std::max(cmax, (int)xy[i]);
    if (anms_u16_wraps(cmax, k_needed[l], cols, rows)) { h->err = "key-point coordinate + search width exceeds 65535 (u16 range tree)"; return -1; }
  }
  const size_t lists = std::max(n_lists, ST_MAXOBJ);
  if (grow_resolver(h, total) || grow(h, h->sel_xy, 2*std::max(total, (size_t)h->W*h->H), h->sel_off, lists, h->sel_cnt, lists, h->sel_k, lists,
                                      h->sel_n, lists, h->sel_tol, lists)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  FCK(cudaMemcpyAsync(h->sel_off, offsets, (size_t)n_lists*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->sel_cnt, cnt.data(), (size_t)n_lists*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->sel_k, k_needed, (size_t)n_lists*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->sel_tol, tolerance, (size_t)n_lists*4, cudaMemcpyHostToDevice, h->s));
  if (total) FCK(cudaMemcpyAsync(h->sel_xy, xy, 2*total*4, cudaMemcpyHostToDevice, h->s));
  anms_range_tree_kernel<<<n_lists, SEL_THREADS, 0, h->s>>>(h->sel_off, h->sel_cnt, h->sel_k, h->sel_tol, 0.f, nullptr, h->sel_xy, 0, cols, rows,
                                                            h->sel_px, h->sel_py, h->sel_orig, h->sel_next, h->sel_out, h->sel_n);
  FCK(cudaGetLastError());
  if (total) FCK(cudaMemcpyAsync(selected, h->sel_out, total*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(n_selected, h->sel_n, (size_t)n_lists*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

int dynofront_sample_dynamic(dynofront_handle h, int32_t nobj, const int32_t* objects, const int32_t* num_track, int32_t max_features,
                             const dynofront_track_params* prm, int64_t* next_tracklet_id, int32_t* counts, int32_t* num_sampled, int32_t* zero_flow,
                             int32_t capacity, double* keypoint, double* flow_out, double* predicted, int64_t* tracklet, int32_t* label,
                             int32_t* n_features, float* ms_device) {
  if (!h || !prm || nobj < 0 || capacity < 0 || !next_tracklet_id || !num_sampled || !n_features) return -1;
  if (nobj && (!objects || !num_track)) return -1;
  if (check_objects(h, nobj, objects)) return -1;
  if (capacity && (!keypoint || !flow_out || !predicted || !tracklet)) { h->err = "null feature array"; return -1; }
  const long long cmax = std::max(h->W, h->H) - 1;       // no width of the search, for any K the objects can need, may wrap
  bool wraps = cmax > 65535;
  for (int k = 2; k <= max_features && !wraps; k++) wraps = anms_u16_wraps(cmax, k, h->W, h->H);
  if (wraps) { h->err = "image too large for the u16 range tree of the reference"; return -1; }
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H; const int ntiles = (int)((npx + ST_TILE - 1)/ST_TILE);
  if (grow_resolver(h, npx) || grow(h, h->sel_off, ST_MAXOBJ, h->sel_k, ST_MAXOBJ, h->sd_idx, npx, h->sd_ntrack, ST_MAXOBJ, h->sd_counts, 3*ST_MAXOBJ)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  if (!h->det_work_valid) prepare_det_work(h);
  *n_features = 0;
  int oc[3][ST_MAXOBJ] = {};                              // per object: candidates, zero-flow pixels, selected (sd_counts)
  int* const d_tot = h->sd_counts; int* const d_zero = d_tot + ST_MAXOBJ; int* const d_nsel = d_tot + 2*ST_MAXOBJ;
  if (nobj > 0) {
    FCK(cudaMemcpyAsync(h->d_objs, objects, (size_t)nobj*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->sd_ntrack, num_track, (size_t)nobj*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemsetAsync(d_zero, 0, ST_MAXOBJ*4, h->s));
    // (1) the candidate scan of dynofront_sample_candidates, its compaction kept on the device
    sc_count_kernel<<<ntiles, ST_TILE, 0, h->s>>>(npx, h->W, h->H, h->det_work, h->mask, h->flow, h->d_objs, nobj, *prm, h->tile_cnt, d_zero);
    sc_scan_kernel<<<1, ST_MAXOBJ, 0, h->s>>>(ntiles, nobj, h->tile_cnt, d_tot);
    sd_prepare_kernel<<<1, 32, 0, h->s>>>(nobj, d_tot, h->sd_ntrack, max_features, h->sel_off, h->sel_k);
    sc_scatter_kernel<<<ntiles, ST_TILE, 0, h->s>>>(npx, h->W, h->H, h->det_work, h->mask, h->flow, h->d_objs, nobj, *prm, h->tile_cnt, h->sel_off,
                                                    h->sd_idx, (long long)npx);
    // (2) + (3) P_n and the range-tree ANMS per object, K = max(max_features - num_track, 0), tolerance 0.01 (FeatureTracker.cc:955-980)
    anms_range_tree_kernel<<<nobj, SEL_THREADS, 0, h->s>>>(h->sel_off, d_tot, h->sel_k, nullptr, 0.01f, h->sd_idx, nullptr, h->W, h->W, h->H,
                                                           h->sel_px, h->sel_py, h->sel_orig, h->sel_next, h->sel_out, d_nsel);
    FCK(cudaGetLastError());
    FCK(cudaMemcpyAsync(oc, h->sd_counts, sizeof(oc), cudaMemcpyDeviceToHost, h->s));
    FCK(cudaStreamSynchronize(h->s));
  }
  int S = 0;
  for (int o = 0; o < nobj; o++) { if (counts) counts[o] = oc[0][o]; if (zero_flow) zero_flow[o] = oc[1][o]; num_sampled[o] = oc[2][o]; S += oc[2][o]; }
  const size_t cap = feature_cap(S);
  if (grow(h, h->sd_kp, 2*cap, h->sd_flow, 2*cap, h->sd_pred, 2*cap, h->sd_tid, cap, h->sd_lab, cap)) return -3;
  const long long base_id = *next_tracklet_id;
  const int ncopy = std::min(S, capacity);
  if (S > 0) {
    // (4) the features, tracklet ids in object order then ANMS order
    sd_construct_kernel<<<nobj, 128, 0, h->s>>>(h->sel_off, d_nsel, h->sel_out, h->sd_idx, h->flow, h->W, h->d_objs, base_id, h->sd_kp, h->sd_flow,
                                                h->sd_pred, h->sd_tid, h->sd_lab);
    FCK(cudaGetLastError());
    if (ncopy) {
      FCK(cudaMemcpyAsync(keypoint, h->sd_kp, 2*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
      FCK(cudaMemcpyAsync(flow_out, h->sd_flow, 2*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
      FCK(cudaMemcpyAsync(predicted, h->sd_pred, 2*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
      FCK(cudaMemcpyAsync(tracklet, h->sd_tid, (size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
      if (label) FCK(cudaMemcpyAsync(label, h->sd_lab, (size_t)ncopy*4, cudaMemcpyDeviceToHost, h->s));
    }
  }
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  *next_tracklet_id = base_id + S;
  *n_features = S;
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

// the descending bitonic sort of keys[0 .. *count) (dt_sort_*), planned for cap keys (a power of two >= DT_SORT_TILE): every launch
// reads the count on the device, so nothing is read back
static void sort_keys_desc(dynofront_ctx* h, unsigned long long* keys, const int* count, size_t keycap) {
  const int cap = (int)keycap, nb = cap/DT_SORT_TILE;
  dt_sort_pad_kernel<<<(cap + 255)/256, 256, 0, h->s>>>(keys, count, cap);
  dt_sort_local_kernel<<<nb, DT_SORT_TILE/2, 0, h->s>>>(keys, count, 2, DT_SORT_TILE);
  for (int k = 2*DT_SORT_TILE; k <= cap; k <<= 1) {
    for (int j = k/2; j >= DT_SORT_TILE; j >>= 1) dt_sort_global_kernel<<<(cap/2 + 255)/256, 256, 0, h->s>>>(keys, count, k, j);
    dt_sort_local_kernel<<<nb, DT_SORT_TILE/2, 0, h->s>>>(keys, count, k, k);
  }
}
static size_t sort_cap(size_t n) { size_t c = DT_SORT_TILE; while (c < n) c <<= 1; return c; }

int dynofront_detect_static(dynofront_handle h, const uint8_t* gray, int32_t n_cur, const double* cur_kp, const dynofront_detect_params* prm,
                            int64_t* next_tracklet_id, int32_t capacity, double* keypoint, int64_t* tracklet, int32_t* n_features,
                            int32_t* n_corners, float* ms_device) {
  if (!h || !prm || !next_tracklet_id || !n_features || n_cur < 0 || capacity < 0 || (n_cur && !cur_kp)) return -1;
  if (capacity && (!keypoint || !tracklet)) { h->err = "null feature array"; return -1; }
  if (prm->use_harris) { h->err = "the Harris response is not supported (TrackerParams: use_harris_corner_detector = false)"; return -1; }
  if (prm->block_size != 3) { h->err = "block_size must be 3"; return -1; }
  if (prm->min_distance < 0 || prm->min_distance > 15) { h->err = "min_distance must be in [0,15]"; return -1; }
  if (prm->use_subpix && prm->subpix_win != SP_WIN) { h->err = "subpix_win must be 5"; return -1; }
  if (!(prm->quality_level > 0.0)) { h->err = "quality_level must be > 0"; return -1; }
  const int W = h->W, H = h->H; const size_t npx = (size_t)W*H;
  if (W < SP_P + 2 || H < SP_P + 2) { h->err = "image smaller than the cornerSubPix window"; return -1; }
  const int K = std::max(prm->max_features - n_cur, 0);
  if (prm->use_anms && K >= 2 && anms_u16_wraps(std::max(W, H) - 1, K, W, H)) { h->err = "image too large for the u16 range tree of the reference"; return -1; }
  if (!gray && !h->have_pyr_cur) { h->err = "no current frame on the device"; return -2; }
  cudaSetDevice(h->dev);
  const size_t keycap = sort_cap(npx);
  if (grow(h, h->dt_gray, npx, h->dt_mask, npx, h->dt_clahe, npx, h->dt_lut, DT_TILES*DT_TILES*256, h->dt_dx, npx, h->dt_dy, npx, h->dt_box, 3*npx,
           h->dt_eig, npx, h->dt_keys, keycap, h->dt_corners, 2*npx, h->dt_cnt, 1, h->dt_pts, 2*npx, h->dt_resp, 1, h->dt_kp, 2*npx, h->dt_tid, npx,
           h->f_kp, 2*feature_cap(n_cur)) || grow_resolver(h, npx)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  const uint8_t* img = gray ? h->dt_gray : h->pyr[1][0];
  if (gray) FCK(cudaMemcpyAsync(h->dt_gray, gray, npx, cudaMemcpyHostToDevice, h->s));
  if (n_cur) FCK(cudaMemcpyAsync(h->f_kp, cur_kp, 2*(size_t)n_cur*8, cudaMemcpyHostToDevice, h->s));
  DetectCounters init = {}; init.K = K;
  FCK(cudaMemcpyAsync(h->dt_cnt, &init, sizeof(init), cudaMemcpyHostToDevice, h->s));
  DetectCounters* const c = h->dt_cnt;                          // (device addresses of the counters)
  const unsigned g1 = (unsigned)((npx + 255)/256); const dim3 blk(32, 8), grd((W + 31)/32, (H + 7)/8);
  // (1) detection mask: boundary mask AND background, circles around the current features
  dt_mask_kernel<<<g1, 256, 0, h->s>>>(npx, h->has_det ? h->det.p : nullptr, h->mask, h->dt_mask);
  if (n_cur) dt_circles_kernel<<<(n_cur + 127)/128, 128, 0, h->s>>>(n_cur, h->f_kp, make_disc(prm->min_distance), W, H, h->dt_mask);
  // (2) CLAHE(2.0, 8x8) on the plain mono image
  if (prm->use_clahe) {
    const bool exact = W % DT_TILES == 0 && H % DT_TILES == 0;
    const int tw = exact ? W/DT_TILES : (W + DT_TILES - W % DT_TILES)/DT_TILES, th = exact ? H/DT_TILES : (H + DT_TILES - H % DT_TILES)/DT_TILES;
    const int area = tw*th, clip = std::max((int)(2.0*area/256), 1);
    clahe_lut_kernel<<<dim3(DT_TILES, DT_TILES), 256, 0, h->s>>>(img, W, H, tw, th, clip, 255.0f/(float)area, h->dt_lut);
    clahe_apply_kernel<<<grd, blk, 0, h->s>>>(img, W, H, 1.0f/(float)tw, 1.0f/(float)th, h->dt_lut, h->dt_clahe);
  } else FCK(cudaMemcpyAsync(h->dt_clahe, img, npx, cudaMemcpyDeviceToDevice, h->s));
  // (3) cornerMinEigenVal(3, 3), its maximum under the mask, the candidates, their order, the minDistance / maxCorners filter
  dt_sobel_kernel<<<grd, blk, 0, h->s>>>(h->dt_clahe, W, H, h->dt_dx, h->dt_dy);
  dt_box_kernel<<<(3*W + 31)/32, 32, 0, h->s>>>(h->dt_dx, h->dt_dy, W, H, h->dt_box);
  dt_eig_kernel<<<g1, 256, 0, h->s>>>(h->dt_box, npx, h->dt_mask, h->dt_eig, &c->max_eig);
  dt_cand_kernel<<<grd, blk, 0, h->s>>>(h->dt_eig, W, H, h->dt_mask, &c->max_eig, prm->quality_level, h->dt_keys, &c->candidates);
  sort_keys_desc(h, h->dt_keys, &c->candidates, keycap);
  dt_gftt_select_kernel<<<1, SEL_THREADS, 0, h->s>>>(h->dt_keys, nullptr, &c->candidates, 0xffffffffu, W, H, prm->min_distance, prm->max_corners, h->sel_px,
                                                     h->sel_py, h->sel_next, h->sel_orig, h->dt_corners, &c->corners, h->dt_resp);
  // (4) range-tree ANMS, K = max(max_features - n_cur, 0), tolerance 0.1 (FeatureDetector.cc:206-224)
  const int* sel = nullptr; const int* cnt = &c->corners;
  if (prm->use_anms) {
    anms_range_tree_kernel<<<1, SEL_THREADS, 0, h->s>>>(&c->anms_off, &c->corners, &c->K, nullptr, 0.1f, nullptr, h->dt_corners, 0, W, H,
                                                         h->sel_px, h->sel_py, h->sel_orig, h->sel_next, h->sel_out, &c->anms);
    sel = h->sel_out; cnt = &c->anms;
  }
  // (5) cornerSubPix in ANMS order, (6) the features
  const int mcap = prm->max_corners > 0 ? (int)std::min<size_t>((size_t)prm->max_corners, npx) : (int)npx;
  if (prm->use_subpix) {
    SubpixMask sm;                                            // cornersubpix.cpp: the Gaussian weights, std::exp in float
    for (int i = 0; i < SP_W; i++) {
      const float y = (float)(i - SP_WIN)/SP_WIN, vy = std::exp(-y*y);
      for (int j = 0; j < SP_W; j++) { const float x = (float)(j - SP_WIN)/SP_WIN; sm.m[i*SP_W + j] = (float)(vy*std::exp(-x*x)); }
    }
    const int iters = std::min(std::max(prm->subpix_max_iter, 1), 100); const double eps = std::max(prm->subpix_eps, 0.0);
    dt_subpix_kernel<<<(mcap + 127)/128, 128, 0, h->s>>>(mcap, h->dt_corners, sel, cnt, h->dt_clahe, W, H, sm, iters, eps*eps, h->dt_pts);
  } else dt_points_kernel<<<(mcap + 255)/256, 256, 0, h->s>>>(mcap, h->dt_corners, sel, cnt, h->dt_pts);
  const long long base_id = *next_tracklet_id;
  dt_construct_kernel<<<1, 1024, 0, h->s>>>(h->dt_pts, cnt, h->mask, W, H, prm->track, base_id, h->dt_kp, h->dt_tid, &c->features);
  FCK(cudaGetLastError());
  DetectCounters res; float resp = 0.f;
  FCK(cudaMemcpyAsync(&res, c, sizeof(res), cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(&resp, h->dt_resp, 4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaStreamSynchronize(h->s));
  h->dt_valid = true;
  // suppressNonMax truncates the responses to int (NonMaximumSupression.cc:47-53); the visiting order P_n assumes they are
  // all 0.  For blockSize 3 on 8-bit input |Ix|, |Iy| <= 1/3 after OpenCV's scale, so a, c <= 9 * (1/9) / 2 and the minimum
  // eigenvalue (a + c) - sqrt((a - c)^2 + b^2) <= 2 min(a, c) <= 1, with equality impossible (a step that is maximal in x
  // and in y over the whole 3x3 window would need its corner pixel to be 0 and 255).  Checked rather than assumed.
  if (prm->use_anms && res.corners > 0 && resp >= 1.0f) { h->err = "a GFTT response >= 1.0: the ANMS order of the reference would differ"; return -1; }
  const int total = res.features, ncopy = std::min(total, capacity);
  if (ncopy) {
    FCK(cudaMemcpyAsync(keypoint, h->dt_kp, 2*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(tracklet, h->dt_tid, (size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
  }
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  *next_tracklet_id = base_id + total; *n_features = total;
  if (n_corners) *n_corners = res.corners;
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}
int dynofront_detect_last_stages(dynofront_handle h, uint8_t* clahe, float* eig, int32_t* corners_xy, int32_t* n_corners) {
  if (!h || !n_corners) return -1;
  if (!h->dt_valid) { h->err = "no detection on this handle yet"; return -2; }
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H;
  int nc = 0;
  FCK(cudaMemcpy(&nc, &h->dt_cnt.p->corners, 4, cudaMemcpyDeviceToHost));
  if (clahe) FCK(cudaMemcpy(clahe, h->dt_clahe, npx, cudaMemcpyDeviceToHost));
  if (eig) FCK(cudaMemcpy(eig, h->dt_eig, npx*4, cudaMemcpyDeviceToHost));
  if (corners_xy && nc) FCK(cudaMemcpy(corners_xy, h->dt_corners, 2*(size_t)nc*4, cudaMemcpyDeviceToHost));
  *n_corners = nc;
  return 0;
}

int dynofront_propagate_mask(dynofront_handle h, int32_t n, const double* kp, const int32_t* lab, const int32_t* prev_mask, const float* prev_flow,
                             const dynofront_track_params* prm, int32_t min_votes, int32_t* current_mask) {
  if (!h || !prm || n < 0) return -1;
  const bool resident = !prev_mask && !prev_flow && !current_mask;       // previous / current frame already on the device (dynofront_next_frame)
  if (!resident && (!prev_mask || !prev_flow || !current_mask)) { h->err = "pass all three images, or none for the resident frames"; return -1; }
  if (resident && !h->have_prev) { h->err = "no previous frame on the device"; return -2; }
  cudaSetDevice(h->dev);
  const size_t cap = feature_cap(n);
  if (grow(h, h->f_kp, 2*cap, h->f_lab, cap, h->pm_votes, 3*cap)) return -3;
  PmPair* const pairs = reinterpret_cast<PmPair*>(h->pm_votes.p + cap);
  const size_t npx = (size_t)h->W*h->H;
  FCK(cudaMemcpyAsync(h->f_kp, kp, 2*(size_t)n*8, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->f_lab, lab, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
  const int32_t* pmask = h->pmask; const float* pflow = h->pflow; int32_t* cmask = resident ? h->mask : h->cmask;
  if (!resident) {
    FCK(cudaMemcpyAsync(h->pmask, prev_mask, npx*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->pflow, prev_flow, 2*npx*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->cmask, current_mask, npx*4, cudaMemcpyHostToDevice, h->s));
    h->have_prev = false;               // the resident previous frame was overwritten
  }
  std::vector<int32_t> labels(lab, lab + n);
  std::sort(labels.begin(), labels.end()); labels.erase(std::unique(labels.begin(), labels.end()), labels.end());
  for (int32_t l : labels) {      // objects in ascending label order, sequentially (FeatureTracker.cc:1262)
    pm_vote_kernel<<<1, PM_THREADS, 0, h->s>>>(n, h->f_kp, h->f_lab, l, cmask, h->W, h->H, min_votes, h->pm_votes, pairs, h->pflag);
    pm_warp_kernel<<<(unsigned)((npx + 255)/256), 256, 0, h->s>>>(npx, h->W, h->H, pmask, pflow, l, *prm, h->pflag, cmask);
  }
  if (!resident) FCK(cudaMemcpyAsync(current_mask, h->cmask, npx*4, cudaMemcpyDeviceToHost, h->s));
  else h->mask_propagated = true;
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  return 0;
}
int dynofront_get_motion_mask(dynofront_handle h, int32_t* out) {
  if (!h || !out) return -1;
  cudaSetDevice(h->dev);
  FCK(cudaMemcpyAsync(out, h->mask, (size_t)h->W*h->H*4, cudaMemcpyDeviceToHost, h->s)); FCK(cudaStreamSynchronize(h->s));
  return 0;
}
int dynofront_object_boundary(dynofront_handle h, int32_t thickness, int32_t capacity, int32_t* n_objects, int32_t* objects, int32_t* bb,
                              int32_t* inner_bb, uint8_t* boundary_out, float* ms_device) {
  if (!h) return -1;
  if (!n_objects || capacity < 0 || (capacity > 0 && (!objects || !bb || !inner_bb))) {
    h->err = "object_boundary: n_objects is required, and objects / bb / inner_bb when capacity > 0"; return -1;
  }
  if (!h->has_frame) { h->err = "object_boundary: no motion mask on the device (dynofront_set_frame / dynofront_next_frame)"; return -1; }
  if (h->mask_propagated) {
    h->err = "object_boundary: dynofront_propagate_mask has modified this frame's motion mask; the boundary mask is computed before it";
    return -1;
  }
  const int W = h->W, H = h->H, t = thickness < 0 ? boundary_thickness(W, H) : thickness;
  if (t > BOUNDARY_MAX_THICKNESS) {
    h->err = "object_boundary: thickness " + std::to_string(t) + " exceeds " + std::to_string(BOUNDARY_MAX_THICKNESS); return -1;
  }
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)W*H;
  if (grow(h, h->bd_T, npx, h->bd_mask, npx, h->bd_tab, BD_TAB)) return -3;
  if (!h->bd_host) FCK(cudaMallocHost((void**)&h->bd_host, BD_TAB*sizeof(int)));
  if (!h->bd_smem_set) {                // the largest tile (thickness BOUNDARY_MAX_THICKNESS) needs more than the default 48 KB
    FCK(cudaFuncSetAttribute(bd_morph_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bd_smem(BOUNDARY_MAX_THICKNESS)));
    h->bd_smem_set = true;
  }
  const BdElem E{bd_rows(BOUNDARY_INNER), bd_rows(t)};
  const dim3 grid((unsigned)((W + BD_TW - 1)/BD_TW), (unsigned)((H + BD_TH - 1)/BD_TH));
  cudaEventRecord(h->e0, h->s);
  FCK(cudaMemsetAsync(h->bd_tab, 0, BD_TAB*sizeof(int), h->s));
  bd_scan_kernel<<<grid, BD_THREADS, 0, h->s>>>(h->mask, W, H, h->bd_T, h->bd_tab);
  bd_morph_kernel<<<grid, BD_THREADS, bd_smem(t), h->s>>>(h->bd_T, W, H, E, h->bd_mask, h->bd_tab);
  cudaEventRecord(h->e1, h->s);
  FCK(cudaMemcpyAsync(h->bd_host, h->bd_tab, BD_TAB*sizeof(int), cudaMemcpyDeviceToHost, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  if (h->bd_host[BD_TAB - 1]) {
    h->err = "object_boundary: a motion-mask label is outside [0, 255] (the reference CHECKs labels > 255 and draws a negative one as 0)";
    return -1;
  }
  *n_objects = boundary_finish(h->bd_host, h->bd_host + 4*(BOUNDARY_MAX_LABEL + 1), W, H, capacity, objects, bb, inner_bb);
  std::swap(h->det, h->bd_mask);       // the boundary mask becomes the current frame's, as an upload through next_frame would
  h->has_det = true; h->det_work_valid = false;
  if (ms_device) cudaEventElapsedTime(ms_device, h->e0, h->e1);
  if (boundary_out) { FCK(cudaMemcpyAsync(boundary_out, h->det, npx, cudaMemcpyDeviceToHost, h->s)); FCK(cudaStreamSynchronize(h->s)); }
  return 0;
}
int dynofront_pin_host(dynofront_handle h, void* ptr, size_t bytes) {
  if (!h || !ptr) return -1;
  cudaSetDevice(h->dev);
  FCK(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
  return 0;
}
int dynofront_unpin_host(dynofront_handle h, void* ptr) {
  if (!h || !ptr) return -1;
  cudaSetDevice(h->dev);
  FCK(cudaHostUnregister(ptr));
  return 0;
}
// the level sizes of every pyramid of the handle (levels down to 2 px)
static void pyramid_sizes(dynofront_ctx* h) {
  if (!h->lw.empty()) return;
  for (int l = 0, w = h->W, hh = h->H; l < 8; l++) {
    h->lw.push_back(w); h->lh.push_back(hh);
    w = (w + 1)/2; hh = (hh + 1)/2;
    if (w < 2 || hh < 2) break;
  }
  const size_t L = h->lw.size();
  h->pyr[0].resize(L); h->pyr[1].resize(L); h->der.resize(L); h->der2.resize(L);
}
// uploads host_img into level 0 of pyr and builds levels 1..max_level (and the Scharr derivatives of levels 0..max_level into der
// when it is given); the arrays must be allocated
static int build_levels(dynofront_ctx* h, std::vector<DevBuf<uint8_t>>& pyr, std::vector<DevBuf<short>>* der, const uint8_t* host_img, int max_level) {
  FCK(cudaMemcpyAsync(pyr[0], host_img, (size_t)h->W*h->H, cudaMemcpyHostToDevice, h->s));
  const dim3 blk(32, 8);
  for (int l = 0; l <= max_level && l < (int)h->lw.size(); l++) {
    const int w = h->lw[l], hh = h->lh[l];
    if (l > 0) pyr_down_kernel<<<dim3((w + 31)/32, (hh + 7)/8), blk, 0, h->s>>>(pyr[l-1], h->lw[l-1], h->lh[l-1], pyr[l], w, hh);
    if (der) scharr_kernel<<<dim3((w + 31)/32, (hh + 7)/8), blk, 0, h->s>>>(pyr[l], w, hh, (*der)[l]);
  }
  return 0;
}
static int build_pyramid(dynofront_ctx* h, int which, const uint8_t* host_img, int max_level, int win, bool with_deriv) {
  pyramid_sizes(h);
  for (size_t l = 0; l < h->lw.size(); l++) {
    const size_t n = (size_t)h->lw[l]*h->lh[l];
    if (grow(h, h->pyr[0][l], n, h->pyr[1][l], n, h->der[l], 2*n, h->der2[l], 2*n)) return -3;
  }
  if (which == 1) h->has_right = false;                         // a new current image: the right image no longer belongs to it
  return build_levels(h, h->pyr[which], with_deriv ? (which == 0 ? &h->der : &h->der2) : nullptr, host_img, max_level);
}
// a stereo slot of its own (st_pyr[slot], with st_der when with_deriv), never the temporal pair
static int build_stereo_pyramid(dynofront_ctx* h, int slot, const uint8_t* host_img, int max_level, bool with_deriv) {
  pyramid_sizes(h);
  std::vector<DevBuf<uint8_t>>& pyr = h->st_pyr[slot];
  pyr.resize(h->lw.size());
  if (with_deriv) h->st_der.resize(h->lw.size());
  for (size_t l = 0; l < h->lw.size(); l++) {
    const size_t n = (size_t)h->lw[l]*h->lh[l];
    if (grow(h, pyr[l], n)) return -3;
    if (with_deriv && grow(h, h->st_der[l], 2*n)) return -3;
  }
  return build_levels(h, pyr, with_deriv ? &h->st_der : nullptr, host_img, max_level);
}

// buildOpticalFlowPyramid's top level: stop when a level is not larger than the window (lkpyramid.cpp)
static int klt_top_level(const dynofront_ctx* h, int max_level, int win) {
  int levels = 0, w = h->W, hh = h->H;
  for (int l = 0; l <= max_level && l < 8; l++) {
    levels = l;
    if (l < max_level) { const int w2 = (w + 1)/2, h2 = (hh + 1)/2; if (w2 <= win || h2 <= win) break; w = w2; hh = h2; }
  }
  return levels;
}
// klt_kernel reaches level-0 window pixels from -win to W + win - 1 (and H likewise) through one reflect101, which stays inside
// the image only when both sides are at least win + 1; cv2 would loop its borderInterpolate there, no dataset frame is that
// small, so such a frame is refused
static int klt_check_frame(dynofront_ctx* h, int win) {
  if (h->W < win + 1 || h->H < win + 1) { h->err = "frame smaller than the LK window: width and height must be at least win + 1"; return -1; }
  return 0;
}
// levels 0..top of one direction: I = pyramid `from` with its derivatives (der for pyramid 0, der2 for pyramid 1), J = the other
static KltLevels klt_levels(const dynofront_ctx* h, int top, int from) {
  KltLevels L; L.nlev = top + 1;
  for (int l = 0; l <= top; l++) {
    L.I[l] = h->pyr[from][l]; L.J[l] = h->pyr[1 - from][l]; L.D[l] = from == 0 ? h->der[l] : h->der2[l]; L.w[l] = h->lw[l]; L.h[l] = h->lh[l];
  }
  return L;
}
// cv::calcOpticalFlowPyrLK's criteria (max_count clamped to [0, 100], epsilon to [0, 10]), one warp per point; errors to k_err
static void klt_launch(dynofront_ctx* h, const KltLevels& L, int n, const float* from, float* to, uint8_t* st, int win, int max_count, double epsilon,
                       int use_initial, float min_eig, float* eig) {
  if (n == 0) return;
  const int mc = std::min(std::max(max_count, 0), 100);
  double eps = std::min(std::max(epsilon, 0.0), 10.0); eps *= eps;
  klt_kernel<<<(n + KLT_WARPS - 1)/KLT_WARPS, KLT_WARPS*32, (size_t)KLT_WARPS*win*win*3*sizeof(short), h->s>>>(L, n, from, to, st, h->k_err, win, mc,
                                                                                                              (float)eps, use_initial, min_eig, eig);
}

int dynofront_klt_track(dynofront_handle h, const uint8_t* prev_gray, const uint8_t* cur_gray, int32_t n, const float* prev_pts, float* next_pts,
                        uint8_t* status, float* err, int32_t win, int32_t max_level, int32_t max_count, double epsilon, int32_t use_initial,
                        double min_eig, float* ms_device) {
  if (!h || !prev_gray || !cur_gray || n < 0 || !prev_pts || !next_pts || !status) return -1;
  if (win < 3 || win > KLT_MAXWIN || max_level < 0) { h->err = "win must be in [3,31]"; return -1; }
  if (klt_check_frame(h, win)) return -1;
  cudaSetDevice(h->dev);
  const int levels = klt_top_level(h, max_level, win);
  const size_t cap = feature_cap(n);
  if (grow(h, h->k_prev, 2*cap, h->k_next, 2*cap, h->k_st, cap, h->k_err, cap, h->k_eig, 2*cap)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  if (build_pyramid(h, 0, prev_gray, levels, win, true)) return -3;
  if (build_pyramid(h, 1, cur_gray, levels, win, false)) return -3;
  h->have_pyr = h->have_pyr_cur = false;      // (the resident pyramids of the streaming mode were overwritten)
  FCK(cudaMemcpyAsync(h->k_prev, prev_pts, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->k_next, use_initial ? next_pts : prev_pts, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
  klt_launch(h, klt_levels(h, levels, 0), n, h->k_prev, h->k_next, h->k_st, win, max_count, epsilon, use_initial, (float)min_eig, h->k_eig);
  FCK(cudaMemcpyAsync(next_pts, h->k_next, 2*(size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(status, h->k_st, n, cudaMemcpyDeviceToHost, h->s));
  if (err) FCK(cudaMemcpyAsync(err, h->k_err, (size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

static int klt_fb_stages(dynofront_ctx* h, bool resident, const uint8_t* prev_gray, const uint8_t* cur_gray, int32_t n, const float* prev_pts,
                         const float* next_pts, const dynofront_klt_fb_params* P, const int32_t* prev_age);
int dynofront_klt_track_fb(dynofront_handle h, const uint8_t* prev_gray, const uint8_t* cur_gray, int32_t n, const float* prev_pts, float* next_pts,
                           uint8_t* status, float* back_pts, const dynofront_klt_fb_params* P, const int32_t* prev_age, uint8_t* keep,
                           int32_t* n_status, int32_t* n_keep, float* ms_device) {
  if (!h || n < 0 || !prev_pts || !next_pts || !status || !P) return -1;
  const bool resident = !prev_gray && !cur_gray;           // both pyramids already on the device (dynofront_next_frame, twice)
  if (!resident && (!prev_gray || !cur_gray)) { h->err = "pass both images, or none for the resident frames"; return -1; }
  if (resident && !(h->have_pyr && h->have_pyr_cur)) { h->err = "two frames are needed on the device"; return -2; }
  if (P->win < 3 || P->win > KLT_MAXWIN || P->win_back < 3 || P->win_back > KLT_MAXWIN || P->max_level < 0 || P->max_level_back < 0) { h->err = "win must be in [3,31]"; return -1; }
  if (P->check_static && (!prev_age || !keep)) { h->err = "check_static needs prev_age and keep"; return -1; }
  if (klt_check_frame(h, std::max(P->win, P->win_back))) return -1;
  if (int rc = klt_fb_stages(h, resident, prev_gray, cur_gray, n, prev_pts, next_pts, P, prev_age)) return rc;
  int counts[2] = {0, 0};
  FCK(cudaMemcpyAsync(next_pts, h->k_next, 2*(size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(status, h->k_st, n, cudaMemcpyDeviceToHost, h->s));
  if (back_pts) FCK(cudaMemcpyAsync(back_pts, h->k_back, 2*(size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  if (keep) FCK(cudaMemcpyAsync(keep, h->k_keep, n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(counts, h->k_count, sizeof(counts), cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  if (n_status) *n_status = counts[0]; if (n_keep) *n_keep = counts[1];
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

// the device stages of dynofront_klt_track_fb, queued from event e0 on: status in k_st, keep in k_keep, counts in k_count
static int klt_fb_stages(dynofront_ctx* h, bool resident, const uint8_t* prev_gray, const uint8_t* cur_gray, int32_t n, const float* prev_pts,
                         const float* next_pts, const dynofront_klt_fb_params* P, const int32_t* prev_age) {
  cudaSetDevice(h->dev);
  const int lf = klt_top_level(h, P->max_level, P->win), lb = klt_top_level(h, P->max_level_back, P->win_back), lmax = std::max(lf, lb);
  const size_t cap = feature_cap(n);
  if (grow(h, h->k_prev, 2*cap, h->k_next, 2*cap, h->k_back, 2*cap, h->k_st, cap, h->k_st2, cap, h->k_keep, cap, h->k_err, cap, h->k_eig, 2*cap,
           h->k_age, cap, h->k_count, 2)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  if (!resident) {
    if (build_pyramid(h, 0, prev_gray, lmax, P->win, true)) return -3;      // both images with derivatives: each is "previous" once
    if (build_pyramid(h, 1, cur_gray, lmax, P->win, true)) return -3;
    h->have_pyr = h->have_pyr_cur = true;
  }
  FCK(cudaMemcpyAsync(h->k_prev, prev_pts, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->k_next, P->use_initial_flow ? next_pts : prev_pts, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
  if (P->check_static) FCK(cudaMemcpyAsync(h->k_age, prev_age, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemsetAsync(h->k_count, 0, 2*sizeof(int), h->s));
  const KltLevels LF = klt_levels(h, lf, 0), LB = klt_levels(h, lb, 1);
  const float min_eig = (float)P->min_eig_threshold;
  klt_launch(h, LF, n, h->k_prev, h->k_next, h->k_st, P->win, P->max_count, P->epsilon, P->use_initial_flow, min_eig, h->k_eig);
  if (P->use_initial_flow && n > 0) {
    // StaticFeatureTracker.cc:491-503: with OPTFLOW_USE_INITIAL_FLOW fewer than 10 successes -> track again from scratch
    int succ = 0;
    count_status_kernel<<<(n + 255)/256, 256, 0, h->s>>>(n, h->k_st, h->k_count);
    FCK(cudaMemcpyAsync(&succ, h->k_count, sizeof(int), cudaMemcpyDeviceToHost, h->s)); FCK(cudaStreamSynchronize(h->s));
    FCK(cudaMemsetAsync(h->k_count, 0, 2*sizeof(int), h->s));
    if (succ < 10) {
      FCK(cudaMemcpyAsync(h->k_next, h->k_prev, 2*(size_t)n*4, cudaMemcpyDeviceToDevice, h->s));
      klt_launch(h, LF, n, h->k_prev, h->k_next, h->k_st, P->win, P->max_count, P->epsilon, 0, min_eig, h->k_eig);
    }
  }
  FCK(cudaMemcpyAsync(h->k_back, h->k_next, 2*(size_t)n*4, cudaMemcpyDeviceToDevice, h->s));       // flags = 0: the backward search starts at the forward result
  klt_launch(h, LB, n, h->k_next, h->k_back, h->k_st2, P->win_back, P->max_count_back, P->epsilon_back, 0, min_eig, nullptr);
  if (n > 0) klt_fb_filter_kernel<<<(n + 255)/256, 256, 0, h->s>>>(n, h->k_prev, h->k_next, h->k_back, h->k_st, h->k_st2, (float)P->max_fb_distance, h->k_st,
                                                                  P->check_static, h->mask, h->W, h->H, P->track, h->k_age, P->max_feature_track_age, h->k_keep, h->k_count);
  return 0;
}

// ---- homography RANSAC
void dynofront_homography_default_params(dynofront_homography_params* p) {
  if (!p) return;
  p->threshold_px = 5.0; p->confidence = 0.995; p->max_iters = 2000; p->refine = 1;      // StaticFeatureTracker.cc:632, OpenCV defaults
}
static int hom_check_params(dynofront_ctx* h, const dynofront_homography_params& P) {
  if (!(P.threshold_px > 0) || !std::isfinite(P.threshold_px) || !(P.confidence > 0 && P.confidence < 1) || P.max_iters > (1 << 20)) {
    h->err = "homography params: threshold_px > 0, 0 < confidence < 1, max_iters <= 2^20"; return -1;
  }
  return 0;
}
// one CTA per problem over rows [off[p], off[p+1]) of src / dst (device), rows with sel == 0 left out when sel is given
static int hom_launch(dynofront_ctx* h, int np, const int* d_off, const float* src, const float* dst, const uint8_t* sel, size_t rows,
                      const dynofront_homography_params& P) {
  const int cap = h->hm_record > 0 ? std::min(h->hm_record, std::max(P.max_iters, 1)) : 0;
  const size_t nr = std::max(rows, (size_t)1);
  if (grow(h, h->hm_cidx, nr, h->hm_lidx, nr, h->hm_inl, nr, h->hm_mask, nr, h->hm_H, 9*(size_t)np, h->hm_stat, 6*(size_t)np)) return -3;
  if (cap && grow(h, h->hm_counts, (size_t)np*cap)) return -3;
  if (cap) FCK(cudaMemsetAsync(h->hm_counts, 0xff, 4*(size_t)np*cap, h->s));      // -1 past the last iteration
  HomBatch B{};
  B.off = d_off; B.src = src; B.dst = dst; B.sel = sel; B.cidx = h->hm_cidx; B.lidx = h->hm_lidx; B.inl = h->hm_inl;
  B.thr2 = (float)(P.threshold_px*P.threshold_px); B.conf = P.confidence; B.max_iters = P.max_iters; B.refine = P.refine != 0;
  B.H = h->hm_H; B.mask = h->hm_mask; int* st = h->hm_stat;
  B.n_inl = st; B.status = st + np; B.iters = st + 2*np; B.groups = st + 3*np; B.rejected = st + 4*np; B.best = st + 5*np;
  B.counts = cap ? (int*)h->hm_counts : nullptr; B.counts_cap = cap;
  for (int lg = -16; lg <= 16; lg++) B.lam[lg + 16] = std::exp(lg*std::log(10.));
  if (np > 0) hom_ransac_kernel<<<np, HOM_THREADS, 0, h->s>>>(B);
  h->hm_np = np; h->hm_cap = cap;
  return 0;
}
int dynofront_homography_record_counts(dynofront_handle h, int32_t counts_cap) {
  if (!h || counts_cap < 0) return -1;
  h->hm_record = counts_cap; return 0;
}
int dynofront_find_homography_batch(dynofront_handle h, int32_t n_problems, const int32_t* offsets, const float* src, const float* dst,
                                    const dynofront_homography_params* prm, double* H, uint8_t* mask, int32_t* n_inliers, int32_t* status,
                                    int32_t* iterations, float* ms_device) {
  if (!h || n_problems < 0 || !offsets || !H || !n_inliers || !status) return -1;
  dynofront_homography_params P; if (prm) P = *prm; else dynofront_homography_default_params(&P);
  if (hom_check_params(h, P)) return -1;
  if (offsets[0] != 0) { h->err = "offsets[0] must be 0"; return -1; }
  for (int p = 0; p < n_problems; p++) if (offsets[p + 1] < offsets[p]) { h->err = "offsets must not decrease"; return -1; }
  const size_t rows = (size_t)offsets[n_problems];
  if (rows > 0 && (!src || !dst || !mask)) return -1;
  for (size_t i = 0; i < 2*rows; i++) if (!std::isfinite(src[i]) || !std::isfinite(dst[i])) { h->err = "non-finite point"; return -1; }
  cudaSetDevice(h->dev);
  const size_t nr = std::max(rows, (size_t)1);
  if (grow(h, h->hm_off, (size_t)n_problems + 1, h->hm_src, 2*nr, h->hm_dst, 2*nr)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  FCK(cudaMemcpyAsync(h->hm_off, offsets, 4*((size_t)n_problems + 1), cudaMemcpyHostToDevice, h->s));
  if (rows) {
    FCK(cudaMemcpyAsync(h->hm_src, src, 8*rows, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->hm_dst, dst, 8*rows, cudaMemcpyHostToDevice, h->s));
  }
  if (int rc = hom_launch(h, n_problems, h->hm_off, h->hm_src, h->hm_dst, nullptr, rows, P)) return rc;
  const size_t np = (size_t)n_problems;
  if (np) {
    FCK(cudaMemcpyAsync(H, h->hm_H, 72*np, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(n_inliers, h->hm_stat, 4*np, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(status, h->hm_stat + np, 4*np, cudaMemcpyDeviceToHost, h->s));
    if (iterations) FCK(cudaMemcpyAsync(iterations, h->hm_stat + 2*np, 4*np, cudaMemcpyDeviceToHost, h->s));
  }
  if (rows) FCK(cudaMemcpyAsync(mask, h->hm_mask, rows, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}
int dynofront_homography_last_trace(dynofront_handle h, int32_t* status, int32_t* groups, int32_t* rejected, int32_t* best, int32_t counts_cap,
                                    int32_t* counts, int32_t* n_problems) {
  if (!h || !n_problems) return -1;
  cudaSetDevice(h->dev);
  const size_t np = (size_t)h->hm_np;
  *n_problems = h->hm_np;
  if (np == 0) return 0;
  if (status) FCK(cudaMemcpy(status, h->hm_stat + np, 4*np, cudaMemcpyDeviceToHost));
  if (groups) FCK(cudaMemcpy(groups, h->hm_stat + 3*np, 4*np, cudaMemcpyDeviceToHost));
  if (rejected) FCK(cudaMemcpy(rejected, h->hm_stat + 4*np, 4*np, cudaMemcpyDeviceToHost));
  if (best) FCK(cudaMemcpy(best, h->hm_stat + 5*np, 4*np, cudaMemcpyDeviceToHost));
  if (counts && counts_cap > 0) {
    std::fill(counts, counts + (size_t)counts_cap*np, -1);        // iterations that were not recorded
    const int w = std::min(counts_cap, h->hm_cap);
    if (w > 0)
    FCK(cudaMemcpy2D(counts, 4*(size_t)counts_cap, h->hm_counts, 4*(size_t)h->hm_cap, 4*(size_t)w, np, cudaMemcpyDeviceToHost));
  }
  return 0;
}
// ---- fundamental-matrix RANSAC
void dynofront_fundamental_default_params(dynofront_fundamental_params* p) {
  if (!p) return;
  p->threshold_px = 1.0; p->confidence = 0.99; p->max_iters = 1000;      // FeatureTracker.cc:280-281, the 6-argument overload
}
int dynofront_fundamental_record(dynofront_handle h, int32_t iters_cap) {
  if (!h || iters_cap < 0) return -1;
  h->fm_record = iters_cap; return 0;
}
static int fund_check_params(dynofront_ctx* h, const dynofront_fundamental_params& P) {
  if (!(P.threshold_px > 0) || !std::isfinite(P.threshold_px) || !(P.confidence > 0 && P.confidence < 1) || P.max_iters > (1 << 20)) {
    h->err = "fundamental params: threshold_px > 0, 0 < confidence < 1, max_iters <= 2^20"; return -1;
  }
  return 0;
}
// one CTA per problem over rows [off[p], off[p+1]) of src / dst (device; the offsets are read on the device, so a count computed
// there never visits the host); outputs in fm_F / fm_mask / fm_stat, the per-iteration record in fm_rec after dynofront_fundamental_record
static int fund_launch(dynofront_ctx* h, int np, const int* d_off, const float* src, const float* dst, size_t rows,
                       const dynofront_fundamental_params& P) {
  const size_t nr = std::max(rows, (size_t)1), npp = std::max((size_t)np, (size_t)1);
  const int cap = h->fm_record;
  if (grow(h, h->fm_mask, nr, h->fm_F, 27*npp, h->fm_stat, 9*npp)) return -3;
  if (cap && grow(h, h->fm_rec, 4*(size_t)np*cap + 1)) return -3;
  if (cap) FCK(cudaMemsetAsync(h->fm_rec, 0xff, 16*(size_t)np*cap, h->s));        // NaN: not recorded
  FundBatch B{};
  B.off = d_off; B.src = src; B.dst = dst; B.thr2 = (float)(P.threshold_px*P.threshold_px); B.conf = P.confidence;
  B.max_iters = P.max_iters; B.F = h->fm_F; B.mask = h->fm_mask; B.stat = h->fm_stat; B.rec = cap ? (float*)h->fm_rec : nullptr; B.rec_cap = cap;
  if (np) fund_ransac_kernel<<<(unsigned)np, FUND_THREADS, 0, h->s>>>(B);
  FCK(cudaGetLastError());
  h->fm_np = np; h->fm_cap = cap;
  return 0;
}
int dynofront_find_fundamental_batch(dynofront_handle h, int32_t n_problems, const int32_t* offsets, const float* p1, const float* p2,
                                     const dynofront_fundamental_params* prm, double* F, int32_t* n_models, uint8_t* mask, int32_t* n_inliers,
                                     int32_t* status, int32_t* iterations, float* ms_device) {
  if (!h || n_problems < 0 || !offsets || !F || !n_models || !n_inliers || !status) return -1;
  dynofront_fundamental_params P; if (prm) P = *prm; else dynofront_fundamental_default_params(&P);
  if (fund_check_params(h, P)) return -1;
  if (offsets[0] != 0) { h->err = "offsets[0] must be 0"; return -1; }
  for (int p = 0; p < n_problems; p++) if (offsets[p + 1] < offsets[p]) { h->err = "offsets must not decrease"; return -1; }
  const size_t rows = (size_t)offsets[n_problems];
  if (rows > 0 && (!p1 || !p2 || !mask)) return -1;
  for (size_t i = 0; i < 2*rows; i++) if (!std::isfinite(p1[i]) || !std::isfinite(p2[i])) { h->err = "non-finite point"; return -1; }
  cudaSetDevice(h->dev);
  const size_t nr = std::max(rows, (size_t)1), np = (size_t)n_problems;
  if (grow(h, h->fm_off, np + 1, h->fm_src, 2*nr, h->fm_dst, 2*nr)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  FCK(cudaMemcpyAsync(h->fm_off, offsets, 4*(np + 1), cudaMemcpyHostToDevice, h->s));
  if (rows) {
    FCK(cudaMemcpyAsync(h->fm_src, p1, 8*rows, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->fm_dst, p2, 8*rows, cudaMemcpyHostToDevice, h->s));
  }
  if (int rc = fund_launch(h, n_problems, h->fm_off, h->fm_src, h->fm_dst, rows, P)) return rc;
  if (np) {
    FCK(cudaMemcpyAsync(F, h->fm_F, 216*np, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(n_models, h->fm_stat, 4*np, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(n_inliers, h->fm_stat + np, 4*np, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(status, h->fm_stat + 2*np, 4*np, cudaMemcpyDeviceToHost, h->s));
    if (iterations) FCK(cudaMemcpyAsync(iterations, h->fm_stat + 3*np, 4*np, cudaMemcpyDeviceToHost, h->s));
  }
  if (rows) FCK(cudaMemcpyAsync(mask, h->fm_mask, rows, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}
int dynofront_fundamental_last_trace(dynofront_handle h, int32_t* groups, int32_t* rejected, int32_t* best, int32_t* best_root,
                                     int32_t* success, int32_t iters_cap, float* record, int32_t* n_problems) {
  if (!h || !n_problems) return -1;
  cudaSetDevice(h->dev);
  const size_t np = (size_t)h->fm_np;
  *n_problems = h->fm_np;
  if (np == 0) return 0;
  int32_t* outs[5] = {groups, rejected, best, best_root, success};
  for (int k = 0; k < 5; k++) if (outs[k]) FCK(cudaMemcpy(outs[k], h->fm_stat + (4 + k)*np, 4*np, cudaMemcpyDeviceToHost));
  if (record && iters_cap > 0) {
    std::fill(record, record + 4*(size_t)iters_cap*np, std::nanf(""));
    const int w = std::min(iters_cap, h->fm_cap);
    if (w > 0)
      FCK(cudaMemcpy2D(record, 16*(size_t)iters_cap, h->fm_rec, 16*(size_t)h->fm_cap, 16*(size_t)w, np, cudaMemcpyDeviceToHost));
  }
  return 0;
}
int dynofront_klt_track_points(dynofront_handle h, const uint8_t* prev_gray, const uint8_t* cur_gray, int32_t n, const float* prev_pts,
                               float* next_pts, uint8_t* status, const dynofront_klt_fb_params* fb, const dynofront_homography_params* hom,
                               const int32_t* prev_age, uint8_t* verified, uint8_t* keep, double* H, int32_t* hom_status, int32_t* n_status,
                               int32_t* n_verified, int32_t* n_keep, float* ms_device) {
  if (!h || n < 0 || !prev_pts || !next_pts || !status || !fb || !verified) return -1;
  const bool resident = !prev_gray && !cur_gray;
  if (!resident && (!prev_gray || !cur_gray)) { h->err = "pass both images, or none for the resident frames"; return -1; }
  if (resident && !(h->have_pyr && h->have_pyr_cur)) { h->err = "two frames are needed on the device"; return -2; }
  if (fb->win < 3 || fb->win > KLT_MAXWIN || fb->win_back < 3 || fb->win_back > KLT_MAXWIN || fb->max_level < 0 || fb->max_level_back < 0) { h->err = "win must be in [3,31]"; return -1; }
  if (fb->check_static && (!prev_age || !keep)) { h->err = "check_static needs prev_age and keep"; return -1; }
  if (klt_check_frame(h, std::max(fb->win, fb->win_back))) return -1;
  dynofront_homography_params P; if (hom) P = *hom; else dynofront_homography_default_params(&P);
  if (hom_check_params(h, P)) return -1;
  if (int rc = klt_fb_stages(h, resident, prev_gray, cur_gray, n, prev_pts, next_pts, fb, prev_age)) return rc;
  // one problem: the rows whose forward-backward status is set, in order -- trackPoints' good_previous / good_current
  const int off[2] = {0, n};
  if (grow(h, h->hm_off, 2)) return -3;
  FCK(cudaMemcpyAsync(h->hm_off, off, sizeof(off), cudaMemcpyHostToDevice, h->s));
  if (int rc = hom_launch(h, 1, h->hm_off, h->k_prev, h->k_next, h->k_st, (size_t)n, P)) return rc;
  FCK(cudaMemsetAsync(h->k_count, 0, 2*sizeof(int), h->s));       // (k_count[0] is reported from the status copy below)
  int counts[2] = {0, 0}, stat[2] = {0, 0};
  if (n > 0) ktp_post_kernel<<<(n + 255)/256, 256, 0, h->s>>>(n, h->hm_mask, h->k_keep, fb->check_static, h->k_count);
  FCK(cudaMemcpyAsync(next_pts, h->k_next, 2*(size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(status, h->k_st, n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(verified, h->hm_mask, n, cudaMemcpyDeviceToHost, h->s));
  if (fb->check_static) FCK(cudaMemcpyAsync(keep, h->k_keep, n, cudaMemcpyDeviceToHost, h->s));
  if (H) FCK(cudaMemcpyAsync(H, h->hm_H, 72, cudaMemcpyDeviceToHost, h->s));
  if (hom_status) FCK(cudaMemcpyAsync(hom_status, h->hm_stat + 1, 4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(counts, h->k_count, sizeof(counts), cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  for (int i = 0; i < n; i++) stat[0] += status[i] != 0;
  if (n_status) *n_status = stat[0]; if (n_verified) *n_verified = counts[0]; if (n_keep) *n_keep = counts[1];
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

// FeatureTracker::stereoTrack (FeatureTracker.cc:194-337): left -> right LK (21x21, 5 levels, OpenCV default criteria), then per
// matched point disparity = uL - uR, rejected when <= 1 px or uR < 0, depth = fx * baseline / disparity.  (The reference also
// runs the right -> left pass but its round-trip filter is commented out, :240-253, and a fundamental-matrix RANSAC sits between
// the LK status and the disparity test: dynofront_stereo_match below runs the whole chain in one call.)
// the per-point rule of FeatureTracker.cc:307-321: false when disparity = uL - uR (in double) <= 1 or uR < 0, else
// depth = fx * baseline / disparity
__device__ __forceinline__ bool stereo_disparity(float uLf, float uRf, double fx, double baseline, double* depth) {
  const double uL = (double)uLf, uR = (double)uRf;
  const double disparity = uL - uR;
  if (disparity <= 1.0 || uR < 0.0f) return false;
  *depth = fx*baseline/disparity;
  return true;
}
__global__ void stereo_post_kernel(int n, const float* __restrict__ left, const float* __restrict__ right, const uint8_t* __restrict__ st, double fx,
                                   double baseline, double* __restrict__ depth, uint8_t* __restrict__ valid) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  double d = 0.0;
  const bool ok = st[i] && stereo_disparity(left[2*i], right[2*i], fx, baseline, &d);
  valid[i] = ok ? 1 : 0;
  depth[i] = ok ? d : 0.0;
}
// dynofront_stereo_match, between the LK and the RANSAC (one CTA): the LK-good rows in input order -- stereoTrack's
// pts_left_tracked / pts_right_tracked -- as idx[rank] = row, rank[row] = rank, cl / cr = the rows' float points; off = {0, m}, or
// {0, 0} when m < 8 (the reference returns before its RANSAC), cnt = {m, 0, 0}
__global__ void __launch_bounds__(HOM_THREADS) stereo_compact_kernel(int n, const float* __restrict__ left, const float* __restrict__ right,
                                                                     const uint8_t* __restrict__ st, int* __restrict__ idx, int* __restrict__ rank,
                                                                     float* __restrict__ cl, float* __restrict__ cr, int* __restrict__ off,
                                                                     int* __restrict__ cnt) {
  __shared__ int sh_wcnt[HOM_WARPS];
  const int m = hom_compact(n, [&](int i) { return st[i] != 0; }, [](int i) { return i; }, idx, sh_wcnt);
  for (int k = threadIdx.x; k < m; k += HOM_THREADS) {
    const int i = idx[k];
    rank[i] = k;
    cl[2*k] = left[2*i]; cl[2*k + 1] = left[2*i + 1]; cr[2*k] = right[2*i]; cr[2*k + 1] = right[2*i + 1];
  }
  if (threadIdx.x == 0) { off[0] = 0; off[1] = m >= 8 ? m : 0; cnt[0] = m; cnt[1] = 0; cnt[2] = 0; }
}
// the per-feature loop of stereoTrack (FeatureTracker.cc:273-335) after the RANSAC: state, depth and uR per input row; cnt[1] / cnt[2]
// count the mask ones and the stereo features
__global__ void stereo_match_post_kernel(int n, const float* __restrict__ left, const float* __restrict__ right, const uint8_t* __restrict__ st,
                                         const int* __restrict__ rank, const uint8_t* __restrict__ mask, double fx, double baseline,
                                         uint8_t* __restrict__ state, double* __restrict__ depth, double* __restrict__ right_u, int* __restrict__ cnt) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t s = DYNOFRONT_STEREO_UNTOUCHED;
  double d = CUDART_NAN, u = CUDART_NAN;
  if (cnt[0] >= 8) {                                         // fewer than 8 tracked: the reference returns false, nothing marked
    if (!st[i]) s = DYNOFRONT_STEREO_LOST;
    else if (!mask[rank[i]]) s = DYNOFRONT_STEREO_EPIPOLAR;
    else {
      atomicAdd(cnt + 1, 1);
      double dd;
      if (stereo_disparity(left[2*i], right[2*i], fx, baseline, &dd)) { s = DYNOFRONT_STEREO_MATCHED; d = dd; u = (double)right[2*i]; atomicAdd(cnt + 2, 1); }
      else s = DYNOFRONT_STEREO_DISPARITY;
    }
  }
  state[i] = s; depth[i] = d; right_u[i] = u;
}
int dynofront_stereo_track(dynofront_handle h, const uint8_t* left_gray, const uint8_t* right_gray, int32_t n, const float* left_pts, float* right_pts,
                           uint8_t* status, double fx, double baseline, double* depth, uint8_t* valid, float* ms_device) {
  if (!h || !left_gray || !right_gray || n < 0 || !left_pts || !right_pts || !status || !depth || !valid) return -1;
  if (klt_check_frame(h, 21)) return -1;
  cudaSetDevice(h->dev);
  const int win = 21, levels = klt_top_level(h, 5, win);
  const size_t cap = feature_cap(n);
  if (grow(h, h->k_prev, 2*cap, h->k_next, 2*cap, h->k_st, cap, h->k_keep, cap, h->k_err, cap, h->k_eig, 2*cap, h->st_depth, cap)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  if (build_pyramid(h, 0, left_gray, levels, win, true)) return -3;
  if (build_pyramid(h, 1, right_gray, levels, win, false)) return -3;
  h->have_pyr = h->have_pyr_cur = false;
  FCK(cudaMemcpyAsync(h->k_prev, left_pts, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->k_next, left_pts, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
  klt_launch(h, klt_levels(h, levels, 0), n, h->k_prev, h->k_next, h->k_st, win, 30, 0.01, 0, 1e-4f, h->k_eig);
  if (n > 0) stereo_post_kernel<<<(n + 255)/256, 256, 0, h->s>>>(n, h->k_prev, h->k_next, h->k_st, fx, baseline, h->st_depth, h->k_keep);
  FCK(cudaMemcpyAsync(right_pts, h->k_next, 2*(size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(status, h->k_st, n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(depth, h->st_depth, (size_t)n*8, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(valid, h->k_keep, n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

// The right image's pyramid has no Scharr derivatives: LK reads derivatives of the image it tracks FROM only, and the reference's
// right -> left pass (FeatureTracker.cc:230-232) is computed but never used (its round-trip filter, :240-253, is commented out),
// so that pass does not run here.
int dynofront_set_right(dynofront_handle h, const uint8_t* right_gray) {
  if (!h || !right_gray) return -1;
  cudaSetDevice(h->dev);
  if (build_stereo_pyramid(h, 2, right_gray, klt_top_level(h, 5, 21), false)) return -3;
  h->has_right = true;
  return 0;                                                     // no synchronisation, as dynofront_next_frame
}
int dynofront_stereo_match(dynofront_handle h, const uint8_t* left_gray, const uint8_t* right_gray, int32_t n, const float* left_pts,
                           double fx, double baseline, const dynofront_fundamental_params* fund, int32_t* matched, uint8_t* state,
                           double* depth, double* right_u, float* right_pts, uint8_t* lk_status, double* F, int32_t* fund_status,
                           int32_t* n_tracked, int32_t* n_inliers, int32_t* n_stereo, float* ms_device) {
  if (!h || n < 0 || (n > 0 && !left_pts) || !matched || !state || !depth || !right_u) return -1;
  const bool resident = !left_gray && !right_gray;
  if (!resident && (!left_gray || !right_gray)) { h->err = "pass both images, or none for the resident frame and right image"; return -1; }
  dynofront_fundamental_params P; if (fund) P = *fund; else dynofront_fundamental_default_params(&P);
  if (fund_check_params(h, P)) return -1;
  if (klt_check_frame(h, 21)) return -1;
  for (size_t i = 0; i < 2*(size_t)n; i++) if (!std::isfinite(left_pts[i])) { h->err = "non-finite point"; return -1; }
  if (resident && !h->have_pyr_cur) { h->err = "no current frame on the device: call dynofront_next_frame first"; return -2; }
  if (resident && !h->has_right) { h->err = "no right image for the current frame: call dynofront_set_right after dynofront_next_frame"; return -2; }
  cudaSetDevice(h->dev);
  *matched = 0;
  if (n < 8) {                                                  // FeatureTracker.cc:205: nothing runs, nothing is marked
    for (int i = 0; i < n; i++) { state[i] = DYNOFRONT_STEREO_UNTOUCHED; depth[i] = right_u[i] = std::nan(""); }
    if (right_pts) std::copy(left_pts, left_pts + 2*(size_t)n, right_pts);
    if (lk_status) std::fill(lk_status, lk_status + n, 0);
    if (F) std::fill(F, F + 9, 0.0);
    if (fund_status) *fund_status = -1;
    if (n_tracked) *n_tracked = 0; if (n_inliers) *n_inliers = 0; if (n_stereo) *n_stereo = 0;
    h->fm_np = 0;                                               // the trace holds no problem
    if (ms_device) *ms_device = 0.f;
    return 0;
  }
  const int win = 21, levels = klt_top_level(h, 5, win);
  const size_t cap = feature_cap(n);
  if (grow(h, h->sm_left, 2*cap, h->sm_right, 2*cap, h->sm_cl, 2*cap, h->sm_cr, 2*cap, h->sm_st, cap, h->sm_state, cap, h->sm_idx, cap,
           h->sm_rank, cap, h->sm_off, 2, h->sm_cnt, 3, h->sm_depth, cap, h->sm_ru, cap, h->k_err, cap)) return -3;   // (klt_launch writes k_err)
  FCK(cudaEventRecord(h->e0, h->s));
  KltLevels L; L.nlev = levels + 1;
  if (!resident) {
    if (build_stereo_pyramid(h, 0, left_gray, levels, true)) return -3;
    if (build_stereo_pyramid(h, 1, right_gray, levels, false)) return -3;
  }
  for (int l = 0; l <= levels; l++) {                           // left: the current frame (pyramid 1, der2) or stereo slot 0
    L.I[l] = resident ? h->pyr[1][l] : h->st_pyr[0][l]; L.D[l] = resident ? h->der2[l] : h->st_der[l];
    L.J[l] = h->st_pyr[resident ? 2 : 1][l]; L.w[l] = h->lw[l]; L.h[l] = h->lh[l];
  }
  FCK(cudaMemcpyAsync(h->sm_left, left_pts, 8*(size_t)n, cudaMemcpyHostToDevice, h->s));
  FCK(cudaMemcpyAsync(h->sm_right, h->sm_left, 8*(size_t)n, cudaMemcpyDeviceToDevice, h->s));   // right_feature_points = left_feature_points
  klt_launch(h, L, n, h->sm_left, h->sm_right, h->sm_st, win, 30, 0.01, 0, 1e-4f, nullptr);
  stereo_compact_kernel<<<1, HOM_THREADS, 0, h->s>>>(n, h->sm_left, h->sm_right, h->sm_st, h->sm_idx, h->sm_rank, h->sm_cl, h->sm_cr, h->sm_off, h->sm_cnt);
  if (int rc = fund_launch(h, 1, h->sm_off, h->sm_cl, h->sm_cr, (size_t)n, P)) return rc;
  stereo_match_post_kernel<<<(n + 255)/256, 256, 0, h->s>>>(n, h->sm_left, h->sm_right, h->sm_st, h->sm_rank, h->fm_mask, fx, baseline, h->sm_state,
                                                            h->sm_depth, h->sm_ru, h->sm_cnt);
  int cnt[3] = {0, 0, 0}, fst = -1;
  FCK(cudaMemcpyAsync(state, h->sm_state, n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(depth, h->sm_depth, 8*(size_t)n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(right_u, h->sm_ru, 8*(size_t)n, cudaMemcpyDeviceToHost, h->s));
  if (right_pts) FCK(cudaMemcpyAsync(right_pts, h->sm_right, 8*(size_t)n, cudaMemcpyDeviceToHost, h->s));
  if (lk_status) FCK(cudaMemcpyAsync(lk_status, h->sm_st, n, cudaMemcpyDeviceToHost, h->s));
  if (F) FCK(cudaMemcpyAsync(F, h->fm_F, 72, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(&fst, h->fm_stat + 2, 4, cudaMemcpyDeviceToHost, h->s));       // status of problem 0 (9 arrays of 1)
  FCK(cudaMemcpyAsync(cnt, h->sm_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  *matched = cnt[0] >= 8;
  if (fund_status) *fund_status = cnt[0] >= 8 ? fst : -1;
  if (n_tracked) *n_tracked = cnt[0]; if (n_inliers) *n_inliers = cnt[1]; if (n_stereo) *n_stereo = cnt[2];
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

int dynofront_klt_last_min_eig(dynofront_handle h, int32_t n, float* out) {
  if (!h || !out || n < 0 || !h->k_eig.p || 2*(size_t)n > h->k_eig.cap) return -1;
  cudaSetDevice(h->dev);
  FCK(cudaMemcpy(out, h->k_eig, 2*(size_t)n*4, cudaMemcpyDeviceToHost));
  return 0;
}

int dynofront_track_static_flow(dynofront_handle h, int32_t n_prev, const double* prev_pred_kp, const int32_t* prev_age, const uint8_t* prev_usable,
                                int32_t n_det, const int32_t* det_xy, int32_t cell_size, int32_t max_features, int64_t* next_tracklet_id,
                                uint8_t* acc_prev, double* flow_prev, double* pred_prev, int32_t* age_out,
                                uint8_t* acc_det, double* flow_det, double* pred_det, int64_t* tracklet_det, int32_t* n_tracked, int32_t* n_detected) {
  if (!h || n_prev < 0 || n_det < 0 || cell_size <= 0 || !next_tracklet_id) return -1;
  if ((n_prev && (!prev_pred_kp || !prev_age || !prev_usable || !acc_prev || !flow_prev || !pred_prev || !age_out)) ||
      (n_det && (!det_xy || !acc_det || !flow_det || !pred_det || !tracklet_det))) { h->err = "null array"; return -1; }
  cudaSetDevice(h->dev);
  const int ncols = (int)std::ceil((double)h->W/cell_size), nrows = (int)std::ceil((double)h->H/cell_size), ncell = ncols*nrows;
  const size_t cap = feature_cap(std::max(n_prev, n_det));
  if (grow(h, h->sf_kp, 2*cap, h->sf_age, cap, h->sf_use, cap, h->sf_det, 2*cap, h->sf_cell, cap, h->sf_win, ncell, h->sf_win2, ncell, h->sf_cnt, 2,
           h->sf_pass, cap, h->sf_acc, cap, h->sf_flow, 2*cap, h->sf_pred, 2*cap, h->sf_oage, cap, h->sf_otid, cap)) return -3;
  fill_i32_kernel<<<(ncell + 255)/256, 256, 0, h->s>>>(h->sf_win, ncell, 0x7fffffff);
  fill_i32_kernel<<<(ncell + 255)/256, 256, 0, h->s>>>(h->sf_win2, ncell, 0x7fffffff);
  FCK(cudaMemsetAsync(h->sf_cnt, 0, 2*sizeof(int), h->s));
  int cnt[2] = {0, 0};
  if (n_prev) {          // (the copies out are ordered before the detections reuse sf_acc / sf_flow / sf_pred)
    FCK(cudaMemcpyAsync(h->sf_kp, prev_pred_kp, 2*(size_t)n_prev*8, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->sf_age, prev_age, (size_t)n_prev*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->sf_use, prev_usable, (size_t)n_prev, cudaMemcpyHostToDevice, h->s));
    sf_prev_kernel<<<(n_prev + 255)/256, 256, 0, h->s>>>(n_prev, h->sf_kp, h->sf_use, h->flow, h->mask, h->W, h->H, cell_size, ncols, h->sf_cell, h->sf_pass,
                                                         h->sf_flow, h->sf_pred, h->sf_win);
    sf_prev_resolve_kernel<<<(n_prev + 255)/256, 256, 0, h->s>>>(n_prev, h->sf_cell, h->sf_pass, h->sf_win, h->sf_age, h->sf_acc, h->sf_flow, h->sf_pred,
                                                                 h->sf_oage, h->sf_cnt);
    FCK(cudaMemcpyAsync(acc_prev, h->sf_acc, n_prev, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(flow_prev, h->sf_flow, 2*(size_t)n_prev*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(pred_prev, h->sf_pred, 2*(size_t)n_prev*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(age_out, h->sf_oage, (size_t)n_prev*4, cudaMemcpyDeviceToHost, h->s));
  }
  if (n_det) {
    FCK(cudaMemcpyAsync(h->sf_det, det_xy, 2*(size_t)n_det*4, cudaMemcpyHostToDevice, h->s));
    sf_det_kernel<<<(n_det + 255)/256, 256, 0, h->s>>>(n_det, h->sf_det, h->flow, h->mask, h->W, h->H, cell_size, ncols, h->sf_win, h->sf_cell, h->sf_pass,
                                                       h->sf_flow, h->sf_pred, h->sf_win2);
    sf_det_resolve_kernel<<<1, 1024, 0, h->s>>>(n_det, h->sf_cell, h->sf_pass, h->sf_win2, h->sf_cnt, max_features, (long long)*next_tracklet_id, h->sf_acc,
                                                h->sf_flow, h->sf_pred, h->sf_otid, h->sf_cnt + 1);
    FCK(cudaMemcpyAsync(acc_det, h->sf_acc, n_det, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(flow_det, h->sf_flow, 2*(size_t)n_det*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(pred_det, h->sf_pred, 2*(size_t)n_det*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(tracklet_det, h->sf_otid, (size_t)n_det*8, cudaMemcpyDeviceToHost, h->s));
  }
  FCK(cudaMemcpyAsync(cnt, h->sf_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, h->s)); FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  *next_tracklet_id += cnt[1];
  if (n_tracked) *n_tracked = cnt[0]; if (n_detected) *n_detected = cnt[1];
  return 0;
}

int dynofront_get_pyramid_level(dynofront_handle h, int32_t which, int32_t level, int32_t* w, int32_t* hgt, uint8_t* img, int16_t* deriv) {
  if (!h || which < 0 || which > 1 || level < 0 || level >= (int)h->lw.size()) return -1;
  cudaSetDevice(h->dev);
  if (w) *w = h->lw[level]; if (hgt) *hgt = h->lh[level];
  const size_t n = (size_t)h->lw[level]*h->lh[level];
  if (img) FCK(cudaMemcpy(img, h->pyr[which][level], n, cudaMemcpyDeviceToHost));
  if (deriv) FCK(cudaMemcpy(deriv, h->der[level], 2*n*sizeof(short), cudaMemcpyDeviceToHost));
  return 0;
}

// ---- depth and back-projection
int dynofront_set_depth(dynofront_handle h, const double* depth) {
  if (!h || !depth) return -1;
  if (!h->has_frame) { h->err = "no frame on the device: call dynofront_set_frame or dynofront_next_frame first"; return -1; }
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H;
  if (grow(h, h->depth, npx)) return -3;
  FCK(cudaMemcpyAsync(h->depth, depth, npx*sizeof(double), cudaMemcpyHostToDevice, h->s));
  h->has_depth = true;
  return 0;                                                     // no synchronisation, as dynofront_next_frame
}
static int depth_args(dynofront_ctx* h, double max_bg, double max_obj) {
  if (!(max_bg > 0.0) || !(max_obj > 0.0)) { h->err = "depth thresholds must be > 0 (Frame::setMaxBackgroundDepth / setMaxObjectDepth)"; return -1; }
  if (!h->has_depth) { h->err = "no depth for the current frame: call dynofront_set_depth after dynofront_set_frame / dynofront_next_frame"; return -1; }
  return 0;
}
static Calib5 calib_of(const double* c) { return Calib5{c[0], c[1], c[2], c[3], c[4]}; }

int dynofront_update_depths(dynofront_handle h, int32_t n, const double* kp, const int32_t* label, double max_background_depth,
                            double max_object_depth, double* depth_out, uint8_t* valid_out, int32_t* n_invalid, int32_t* n_outside, float* ms_device) {
  if (!h || n < 0 || (n && (!kp || !label || !depth_out || !valid_out))) return -1;
  if (depth_args(h, max_background_depth, max_object_depth)) return -1;
  cudaSetDevice(h->dev);
  const size_t cap = feature_cap(n);
  if (grow(h, h->dp_kp, 2*cap, h->dp_lab, cap, h->dp_depth, cap, h->dp_flag, cap, h->dp_cnt, 2)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  FCK(cudaMemsetAsync(h->dp_cnt, 0, 2*sizeof(int), h->s));
  int cnt[2] = {0, 0};
  if (n) {
    FCK(cudaMemcpyAsync(h->dp_kp, kp, 2*(size_t)n*8, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->dp_lab, label, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
    ud_kernel<<<(n + 255)/256, 256, 0, h->s>>>(n, h->dp_kp, h->dp_lab, h->depth, h->W, h->H, max_background_depth, max_object_depth, h->dp_depth,
                                               h->dp_flag, h->dp_cnt);
    FCK(cudaGetLastError());
    FCK(cudaMemcpyAsync(depth_out, h->dp_depth, (size_t)n*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(valid_out, h->dp_flag, (size_t)n, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(cnt, h->dp_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, h->s));
  }
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  if (n_invalid) *n_invalid = cnt[0];
  if (n_outside) *n_outside = cnt[1];
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

int dynofront_back_project(dynofront_handle h, int32_t n, const double* kp, const double* depth, const uint8_t* usable, const double* right_u,
                           const double* calib5, double baseline, int32_t rgbd, const double* X_world, int32_t capacity, int32_t* index,
                           double* point, double* stereo, uint8_t* outlier, int32_t* m, float* ms_device) {
  if (!h || n < 0 || capacity < 0 || !calib5 || !m || (n && (!kp || !depth || !usable))) return -1;
  if (capacity && (!index || !point || !stereo)) { h->err = "null measurement array"; return -1; }
  if (right_u)
    for (int i = 0; i < n; i++)
      if (usable[i] && !std::isnan(right_u[i]) && std::isnan(depth[i])) { h->err = "a usable feature has a right key-point but no depth"; return -1; }
  cudaSetDevice(h->dev);
  const size_t cap = feature_cap(n);
  if (grow(h, h->dp_kp, 2*cap, h->dp_depth, cap, h->dp_flag, cap, h->dp_right, cap, h->dp_out, cap, h->dp_index, cap, h->dp_point, 3*cap,
           h->dp_stereo, 3*cap, h->dp_cnt, 2)) return -3;
  Pose12 X{}; if (X_world) std::memcpy(X.m, X_world, sizeof(X.m));
  FCK(cudaEventRecord(h->e0, h->s));
  if (n) {
    FCK(cudaMemcpyAsync(h->dp_kp, kp, 2*(size_t)n*8, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->dp_depth, depth, (size_t)n*8, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->dp_flag, usable, (size_t)n, cudaMemcpyHostToDevice, h->s));
    if (right_u) FCK(cudaMemcpyAsync(h->dp_right, right_u, (size_t)n*8, cudaMemcpyHostToDevice, h->s));
  }
  const double fx_b = calib5[0]*baseline;                       // RGBDCamera::fx_b_
  bp_kernel<<<1, 1024, 0, h->s>>>(n, h->dp_kp, h->dp_depth, h->dp_flag, right_u ? h->dp_right.p : nullptr, calib_of(calib5), fx_b, rgbd ? 1 : 0, h->W, X,
                                  X_world ? 1 : 0, std::min(capacity, n), h->dp_index, h->dp_point, h->dp_stereo, h->dp_out, h->dp_cnt);
  FCK(cudaGetLastError());
  int total = 0;
  FCK(cudaMemcpyAsync(&total, h->dp_cnt, sizeof(int), cudaMemcpyDeviceToHost, h->s));
  if (n && outlier) FCK(cudaMemcpyAsync(outlier, h->dp_out, (size_t)n, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaStreamSynchronize(h->s));
  const int ncopy = std::min(total, capacity);
  if (ncopy) {
    FCK(cudaMemcpyAsync(index, h->dp_index, (size_t)ncopy*4, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(point, h->dp_point, 3*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(stereo, h->dp_stereo, 3*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
  }
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  *m = total;
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

int dynofront_dense_cloud(dynofront_handle h, const double* calib5, double max_background_depth, double max_object_depth, float* xyz, uint8_t* rgb,
                          uint32_t* label, uint8_t* valid, int32_t* n_valid, float* ms_device) {
  if (!h || !calib5) return -1;
  if (depth_args(h, max_background_depth, max_object_depth)) return -1;
  cudaSetDevice(h->dev);
  const size_t npx = (size_t)h->W*h->H;
  if (grow(h, h->dc_xyz, 3*npx, h->dc_rgb, 3*npx, h->dc_label, npx, h->dc_valid, npx, h->dp_cnt, 2)) return -3;
  FCK(cudaEventRecord(h->e0, h->s));
  FCK(cudaMemsetAsync(h->dp_cnt, 0, sizeof(int), h->s));
  dc_kernel<<<(unsigned)((npx + 255)/256), 256, 0, h->s>>>(npx, h->W, h->depth, h->mask, h->has_det ? h->det.p : nullptr, calib_of(calib5),
                                                           max_background_depth, max_object_depth, h->dc_xyz, h->dc_rgb, h->dc_label, h->dc_valid, h->dp_cnt);
  FCK(cudaGetLastError());
  int cnt = 0;
  FCK(cudaMemcpyAsync(&cnt, h->dp_cnt, sizeof(int), cudaMemcpyDeviceToHost, h->s));
  if (xyz) FCK(cudaMemcpyAsync(xyz, h->dc_xyz, 3*npx*4, cudaMemcpyDeviceToHost, h->s));
  if (rgb) FCK(cudaMemcpyAsync(rgb, h->dc_rgb, 3*npx, cudaMemcpyDeviceToHost, h->s));
  if (label) FCK(cudaMemcpyAsync(label, h->dc_label, npx*4, cudaMemcpyDeviceToHost, h->s));
  if (valid) FCK(cudaMemcpyAsync(valid, h->dc_valid, npx, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  if (n_valid) *n_valid = cnt;
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

// ---- trackDynamicKLT
void dynofront_klt_dynamic_default_params(dynofront_klt_dynamic_params* p) {
  if (!p) return;
  p->win = 21; p->max_level = 3; p->max_count = 30; p->epsilon = 0.03; p->min_eig_threshold = 1e-4;      // FeatureTracker.cc:625-639
  p->track.max_dynamic_feature_age = 20; p->track.min_distance = 2; p->track.shrink_row = 0; p->track.shrink_col = 0;
  p->max_features = 200; p->quality_level = 0.01; p->age_buffer = 3; p->min_tracks = 20; p->min_iou = 0.1;   // params/FrontendParams.yaml
}

int dynofront_track_dynamic_klt(dynofront_handle h, const uint8_t* prev_gray, const uint8_t* cur_gray, int32_t n, const float* prev_kp,
                                const int32_t* prev_label, const int32_t* prev_age, const int64_t* prev_tracklet, int32_t n_objects,
                                const int32_t* objects, const int32_t* inner_bb, const dynofront_klt_dynamic_params* prm, int64_t* next_tracklet_id,
                                float* lk_pts, uint8_t* lk_status, uint8_t* state, double* measured_flow, int32_t capacity, double* keypoint,
                                int32_t* age, int64_t* tracklet, int32_t* label, int32_t* source, int32_t* n_features,
                                dynofront_object_status* status, int32_t* n_outside_image, uint8_t* detection_mask_out, uint8_t* tracking_mask_out,
                                float* ms_device) {
  if (!h || !prm || !next_tracklet_id || !n_features || !status || n < 0 || capacity < 0 || n_objects < 0) return -1;
  if (n && (!prev_kp || !prev_label || !prev_age || !prev_tracklet)) { h->err = "null previous-feature array"; return -1; }
  if (n_objects && (!objects || !inner_bb)) { h->err = "null object array"; return -1; }
  if (capacity && (!keypoint || !age || !tracklet || !label || !source)) { h->err = "null feature array"; return -1; }
  if (check_objects(h, n_objects, objects)) return -1;
  for (int o = 0; o < n_objects; o++) {
    if (inner_bb[4*o + 2] < 0 || inner_bb[4*o + 3] < 0) { h->err = "bounding boxes must have width, height >= 0"; return -1; }
  }
  const dynofront_track_params& T = prm->track;
  if (T.min_distance < 0 || T.min_distance > 15) { h->err = "min_distance must be in [0,15]"; return -1; }
  if (prm->win < 3 || prm->win > KLT_MAXWIN || prm->max_level < 0) { h->err = "win must be in [3,31]"; return -1; }
  if (klt_check_frame(h, prm->win)) return -1;
  const int expiry = T.max_dynamic_feature_age - std::max(3, prm->age_buffer);
  if (expiry <= 0) { h->err = "max_dynamic_feature_age - max(3, age_buffer) must be > 0"; return -1; }
  if (prm->min_tracks < 0 || prm->max_features < 0) { h->err = "min_tracks and max_features must be >= 0"; return -1; }
  if (!(prm->quality_level > 0.0)) { h->err = "quality_level must be > 0"; return -1; }
  const int W = h->W, H = h->H; const size_t npx = (size_t)W*H;
  if (npx > ((size_t)1 << TK_ADDR_BITS)) { h->err = "image larger than 2^26 pixels"; return -1; }
  {
    const long long cmax = std::max(W, H) - 1;                   // no width of the search, for any K an object can need, may wrap
    bool wraps = cmax > 65535;
    for (int k = 2; k <= prm->max_features && !wraps; k++) wraps = anms_u16_wraps(cmax, k, W, H);
    if (wraps) { h->err = "image too large for the u16 range tree of the reference"; return -1; }
  }
  const bool resident = !prev_gray && !cur_gray;
  if (!resident && (!prev_gray || !cur_gray)) { h->err = "pass both images, or none for the resident frames"; return -1; }
  if (resident && !(h->have_pyr && h->have_pyr_cur)) { h->err = "two frames are needed on the device"; return -2; }
  if (!h->has_frame) { h->err = "no motion mask on the device"; return -2; }
  const int top = klt_top_level(h, prm->max_level, prm->win);
  if (resident && top > 5) { h->err = "the resident pyramids have 5 levels"; return -1; }
  cudaSetDevice(h->dev);
  const size_t cap = feature_cap(n), ocap = (size_t)n + (size_t)n_objects*std::max(prm->max_features, 1), tkeys = sort_cap(n), keycap = sort_cap(npx);
  if (grow(h, h->k_prev, 2*cap, h->k_next, 2*cap, h->k_st, cap, h->k_err, cap, h->k_eig, 2*cap, h->f_lab, cap, h->f_age, cap, h->f_tid, cap,
           h->f_x, cap, h->f_y, cap, h->f_state, cap, h->f_next, cap, h->f_flow, 2*cap, h->f_oage, cap, h->f_otid, cap, h->f_olab, cap, h->f_acc, cap,
           h->tk_rows, (ST_MAXOBJ + 1)*sizeof(TkRow), h->tk_cnt, sizeof(TkCounters), h->tk_int, 9*ST_MAXOBJ, h->tk_keys, tkeys, h->tk_eig, npx,
           h->tk_corners, 2*npx, h->dt_dx, npx, h->dt_dy, npx, h->dt_box, 3*npx, h->dt_keys, keycap, h->tk_kp, 2*ocap, h->tk_age, ocap,
           h->tk_tid, ocap, h->tk_lab, ocap, h->tk_src, ocap) || grow_resolver(h, npx)) return -3;
  TkRow* rows = reinterpret_cast<TkRow*>(h->tk_rows.p); TkCounters* cnt = reinterpret_cast<TkCounters*>(h->tk_cnt.p);
  int* const d_bb = h->tk_int; int* const d_K = d_bb + 4*ST_MAXOBJ; int* const d_cand = d_K + ST_MAXOBJ; int* const d_off = d_cand + ST_MAXOBJ;
  int* const d_ncorn = d_off + ST_MAXOBJ; int* const d_nsel = d_ncorn + ST_MAXOBJ;
  TkParams P; P.track = T; P.max_age = T.max_dynamic_feature_age; P.expiry = expiry; P.max_features = prm->max_features;
  P.min_tracks = prm->min_tracks; P.quality = prm->quality_level; P.min_iou = prm->min_iou;
  const Disc disc = make_disc(T.min_distance);
  FCK(cudaEventRecord(h->e0, h->s));
  if (!resident) {                                               // as dynofront_klt_track: the resident pyramids are overwritten
    if (build_pyramid(h, 0, prev_gray, top, prm->win, true)) return -3;
    if (build_pyramid(h, 1, cur_gray, top, prm->win, false)) return -3;
    h->have_pyr = h->have_pyr_cur = false;
  }
  if (n) {
    FCK(cudaMemcpyAsync(h->k_prev, prev_kp, 2*(size_t)n*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->k_next, h->k_prev, 2*(size_t)n*4, cudaMemcpyDeviceToDevice, h->s));
    FCK(cudaMemcpyAsync(h->f_lab, prev_label, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->f_age, prev_age, (size_t)n*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(h->f_tid, prev_tracklet, (size_t)n*8, cudaMemcpyHostToDevice, h->s));
  }
  if (n_objects) {
    FCK(cudaMemcpyAsync(h->d_objs, objects, (size_t)n_objects*4, cudaMemcpyHostToDevice, h->s));
    FCK(cudaMemcpyAsync(d_bb, inner_bb, (size_t)n_objects*16, cudaMemcpyHostToDevice, h->s));
  }
  prepare_det_work(h);                                          // detection_mask_impl starts as the boundary mask (255 without one)
  const unsigned gp = (unsigned)((npx + 255)/256);
  fill_i32_kernel<<<gp, 256, 0, h->s>>>(h->cell, npx, -1);
  fill_i32_kernel<<<gp, 256, 0, h->s>>>(h->trk_idx, npx, 0);
  tk_init_kernel<<<1, 128, 0, h->s>>>(n_objects + 1, rows, cnt, d_cand);
  // (1) forward LK on levels 0..top (flags 0)
  klt_launch(h, klt_levels(h, top, 0), n, h->k_prev, h->k_next, h->k_st, prm->win, prm->max_count, prm->epsilon, 0, (float)prm->min_eig_threshold, h->k_eig);
  // (2) per feature: gather, greedy disc resolution, counters, sort keys of the tracked features; the two masks
  if (n) {
    const int g = (n + 127)/128;
    tk_gather_kernel<<<g, 128, 0, h->s>>>(n, h->k_next, h->k_st, h->f_lab, h->f_age, h->mask, h->has_det ? h->det.p : nullptr, W, H, P, h->f_x, h->f_y,
                                          h->f_state, h->f_oage, h->f_olab);
    td_link_kernel<<<g, 128, 0, h->s>>>(n, h->f_x, h->f_y, h->f_state, W, h->cell, h->f_next);
    td_resolve_kernel<<<1, 1024, 0, h->s>>>(n, h->f_x, h->f_y, h->f_state, h->cell, h->f_next, W, H, disc, T.max_dynamic_feature_age, h->f_tid,
                                            h->f_oage, h->f_otid, h->f_acc, h->nextid, TK_MASKED);
    tk_count_kernel<<<g, 128, 0, h->s>>>(n, h->k_prev, h->k_next, h->f_x, h->f_y, h->f_state, h->cell, h->f_next, disc, W, H, h->f_lab, h->f_oage,
                                         h->f_olab, h->d_objs, n_objects, P, rows, cnt, h->tk_keys, h->f_flow);
    td_masks_kernel<<<g, 128, 0, h->s>>>(n, h->f_x, h->f_y, h->f_acc, W, H, disc, h->det_work, h->trk_idx);
    sort_keys_desc(h, h->tk_keys, &cnt->tracked, tkeys);
  }
  td_trk_final_kernel<<<gp, 256, 0, h->s>>>(npx, h->trk_idx, h->f_olab, h->trk);
  // (3) requiresSampling, (4) goodFeaturesToTrack per sampled object on the mono image, (5) range-tree ANMS
  if (n_objects) {
    const uint8_t* mono = h->pyr[1][0];
    const dim3 blk(32, 8), grd((W + 31)/32, (H + 7)/8);
    tk_decide_kernel<<<1, ST_MAXOBJ, 0, h->s>>>(n_objects, d_bb, P, rows, d_K);
    dt_sobel_kernel<<<grd, blk, 0, h->s>>>(mono, W, H, h->dt_dx, h->dt_dy);
    dt_box_kernel<<<(3*W + 31)/32, 32, 0, h->s>>>(h->dt_dx, h->dt_dy, W, H, h->dt_box);
    tk_eig_kernel<<<gp, 256, 0, h->s>>>(h->dt_box, npx, h->mask, h->det_work, h->d_objs, n_objects, rows, h->tk_eig);
    tk_cand_kernel<<<grd, blk, 0, h->s>>>(h->tk_eig, W, H, h->mask, h->det_work, h->d_objs, n_objects, rows, prm->quality_level, h->dt_keys, cnt, d_cand);
    sort_keys_desc(h, h->dt_keys, &cnt->cand, keycap);
    tk_offsets_kernel<<<1, 32, 0, h->s>>>(n_objects, d_cand, d_off);
    dt_gftt_select_kernel<<<n_objects, SEL_THREADS, 0, h->s>>>(h->dt_keys, d_off, d_cand, (1u << TK_ADDR_BITS) - 1u, W, H, T.min_distance, prm->max_features,
                                                                h->sel_px, h->sel_py, h->sel_next, h->sel_orig, h->tk_corners, d_ncorn, nullptr);
    anms_range_tree_kernel<<<n_objects, SEL_THREADS, 0, h->s>>>(d_off, d_ncorn, d_K, nullptr, 0.01f, nullptr, h->tk_corners, 0, W, H, h->sel_px, h->sel_py,
                                                                 h->sel_orig, h->sel_next, h->sel_out, d_nsel);
  }
  // (6) the output features
  const long long base_id = *next_tracklet_id;
  tk_construct_kernel<<<1, 1024, 0, h->s>>>(h->tk_keys, h->k_next, h->f_oage, h->f_olab, h->f_tid, h->d_objs, n_objects, d_off, d_nsel, h->sel_out,
                                            h->tk_corners, W, H, P, base_id, rows, cnt, h->tk_kp, h->tk_age, h->tk_tid, h->tk_lab, h->tk_src);
  FCK(cudaGetLastError());
  TkRow hr[ST_MAXOBJ + 1]; TkCounters hc;
  FCK(cudaMemcpyAsync(hr, rows, (size_t)(n_objects + 1)*sizeof(TkRow), cudaMemcpyDeviceToHost, h->s));
  FCK(cudaMemcpyAsync(&hc, cnt, sizeof(hc), cudaMemcpyDeviceToHost, h->s));
  if (n) {
    if (lk_pts) FCK(cudaMemcpyAsync(lk_pts, h->k_next, 2*(size_t)n*4, cudaMemcpyDeviceToHost, h->s));
    if (lk_status) FCK(cudaMemcpyAsync(lk_status, h->k_st, n, cudaMemcpyDeviceToHost, h->s));
    if (measured_flow) FCK(cudaMemcpyAsync(measured_flow, h->f_flow, 2*(size_t)n*8, cudaMemcpyDeviceToHost, h->s));
  }
  std::vector<int> st_host(state && n ? n : 0);
  if (state && n) FCK(cudaMemcpyAsync(st_host.data(), h->f_state, (size_t)n*4, cudaMemcpyDeviceToHost, h->s));
  if (detection_mask_out) FCK(cudaMemcpyAsync(detection_mask_out, h->det_work, npx, cudaMemcpyDeviceToHost, h->s));
  if (tracking_mask_out) FCK(cudaMemcpyAsync(tracking_mask_out, h->trk, npx, cudaMemcpyDeviceToHost, h->s));
  FCK(cudaStreamSynchronize(h->s));
  const int total = hc.features, ncopy = std::min(total, capacity);
  if (ncopy) {
    FCK(cudaMemcpyAsync(keypoint, h->tk_kp, 2*(size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(age, h->tk_age, (size_t)ncopy*4, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(tracklet, h->tk_tid, (size_t)ncopy*8, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(label, h->tk_lab, (size_t)ncopy*4, cudaMemcpyDeviceToHost, h->s));
    FCK(cudaMemcpyAsync(source, h->tk_src, (size_t)ncopy*4, cudaMemcpyDeviceToHost, h->s));
  }
  FCK(cudaEventRecord(h->e1, h->s));
  FCK(cudaStreamSynchronize(h->s));
  FCK(cudaGetLastError());
  for (int i = 0; i < (int)st_host.size(); i++) state[i] = (uint8_t)st_host[i];
  for (int r = 0; r <= n_objects; r++) {
    const TkRow& x = hr[r]; dynofront_object_status& s = status[r];
    s.object_id = r ? objects[r - 1] : 0; s.exists = x.exists; s.num_previous_track = x.prev; s.num_track = x.track;
    s.num_outside_shrunken_image = x.shrunk; s.num_tracked_with_different_label = x.diff; s.num_tracked_with_background_label = x.bg;
    s.object_new = x.is_new; s.object_resampled = x.resampled; s.sampled = x.sampled; s.num_sampled = x.num_sampled;
  }
  const int n_new = total - hc.tracked;
  *next_tracklet_id = base_id + n_new; *n_features = total;
  if (n_outside_image) *n_outside_image = hc.outside;
  if (ms_device) FCK(cudaEventElapsedTime(ms_device, h->e0, h->e1));
  return 0;
}

}  // extern "C"
