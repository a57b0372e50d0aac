// api.cu -- host side of libdynoba: C-ABI entry points (include/dynoba.h), symbolic phase (ordering, landmark
// grouping, band structure), device upload and the Levenberg-Marquardt control loop.
//
// The LM loop is a literal restatement of GTSAM 4.2.0's LevenbergMarquardtOptimizer::{iterate,tryLambda} and
// NonlinearOptimizer::defaultOptimize [GTSAM-ext] (SURVEY.md Appendix A.4), which is what the reference runs at
// dynosam/src/backend/RegularBackendModule.cc:405-428.  Control decisions need two scalars per trial step, so
// the loop lives on the host and everything else stays on the device.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <parallel/algorithm>
#include <omp.h>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <numeric>
#include <string>
#include <vector>
#include <map>

#include "../../include/dynoba.h"
#include "internal.cuh"
#include "var_layout.cuh"
#include "window_plan.cuh"

using namespace dynoba;

namespace {

struct HostBlock {
  int type = 0; int64_t n = 0;
  std::vector<int32_t, NoInitAlloc<int32_t>> idx, aux; std::vector<double, NoInitAlloc<double>> meas; std::vector<double> sigma;
  int sigma_dim = 1; bool bcast = true; double robust_k = 0; bool has_aux = false;
  // finalize products
  std::vector<int32_t, NoInitAlloc<int32_t>> perm;   // sorted position -> original factor index (filled in parallel, never value-initialised)
  DevBlock dev{};
  bool simple = false, pose_only = false;
  int part_off = 0, bs_off = 0;
  DevWindows win{}; bool use_window = false; bool all_window = false;   // all_window: no group left for the per-landmark atomics kernel
  int64_t win_ctas = 0, win_flushed = 0;   // accumulate-kernel CTAs and 6x6 blocks it flushes, per damped solve
};

struct HostPrior {      // gtsam::LinearContainerFactor(HessianFactor) over pose-like variables
  std::vector<int32_t> kind, idx; std::vector<double> lin, G, g; double f = 0;
  bool legacy = false;  // added through dynoba_add_linear_prior (pose-only graphs)
  DevPrior dev{}; int part_off = 0, bs_off = 0;
};

constexpr int LM_TRACE_COLS = 10;   // columns of a dynoba_get_lm_trace row
enum CovTiles { COV_NONE, COV_FACTOR, COV_SIGMA };   // what the covariance layout's tiles hold

}  // namespace

struct dynoba_solver {
  int device = 0; cudaStream_t stream = nullptr; cudaStream_t stream2 = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr; std::string err;
  // values [n][KINDS[kind].width] and keys of every variable kind, in caller order
  std::vector<double> vals[NUM_KINDS], aux; std::vector<uint64_t> keys[NUM_KINDS];
  double calib[6] = { 721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372 };
  std::vector<int32_t> hints[NUM_KINDS];   // order hints of the pose-like kinds
  int2* d_nav = nullptr; int n_nav = 0;   // device (position, dimension) of every velocity and bias
  std::vector<HostBlock> blocks;
  std::vector<HostPrior> priors;
  bool finalized = false, linearized = false, supported = true;
  VarLayout layout;      // where every variable sits, from finalize on
  DevVars cur{}, cand{}; BandPlan plan{}; DevBand& band = plan.band; int ncell_request = 0;
  double *dl_point = nullptr, *dl_flow = nullptr, *partials = nullptr, *scalars = nullptr;
  int* fail = nullptr; int n_partials = 0, n_lin_partials = 0, n_bs_partials = 0;
  int rank = 0, world = 1; dynoba_allreduce_fn allreduce = nullptr; void* ar_ctx = nullptr; int min_bw = 0;
  dynoba_reduce_fn reduce = nullptr; void* red_ctx = nullptr;
  int64_t launches = 0; int64_t jac_bytes = 0;
  GeneralGroups gen{}; int gen_bs_off = 0;
  std::vector<std::pair<void*, size_t>> allocs;   // device allocations (pointer, bytes)
  cudaEvent_t ev[8]{};
  // parity hooks: {oldLin, lin, fail} of the latest trial step, and one row per trial of the latest dynoba_optimize
  // (LM_TRACE_COLS doubles: iterations, inner, lambda, oldLin, lin, err, nerr, solved, success, stop)
  double last_model[3] = {0.0, 0.0, 0.0};
  std::vector<double> lm_trace;
  // dynoba_marginal_covariance / dynoba_joint_marginal_covariance: a plain layout of their own whose tiles hold nothing,
  // the factor L of the undamped reduced system or Sigma = S^-1 on its band (cov_tiles), and the landmark tables, kept
  // from the first call at a linearisation point until the values change
  BandPlan cov_plan{}; double* cov_stage = nullptr; double* cov_lmk = nullptr;
  bool cov_live = false, cov_lmk_ready = false; int cov_tiles = 0; float cov_ms[2] = {0.0f, 0.0f};
};

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return DYNOBA_ERR_CUDA; } } while (0)
#define ARG(cond, msg) do { if (!(cond)) { if (h) h->err = msg; return DYNOBA_ERR_BAD_ARG; } } while (0)

// Process-wide pinned staging arena for the SoA images of the factor blocks: host->device copies from it run at PCIe
// speed and asynchronously, so the upload of one block overlaps the host-side preparation of the next.  Grow-only.
#include <mutex>
namespace {
struct PinnedArena {
  char* base = nullptr; size_t cap = 0, off = 0; std::mutex mu;
  bool reserve(size_t bytes) {
    off = 0;
    if (bytes <= cap) return true;
    if (base) { cudaFreeHost(base); base = nullptr; cap = 0; }
    const size_t want = bytes + bytes/8 + (1 << 20);
    if (cudaHostAlloc((void**)&base, want, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); base = nullptr; return false; }
    cap = want; return true;
  }
  void* take(size_t bytes) { const size_t a = (off + 255) & ~(size_t)255; if (!base || a + bytes > cap) return nullptr; off = a + bytes; return base + a; }
};
PinnedArena g_arena;
// staging image of one SoA array: a slice of the arena, else plain new[] (no value-initialisation pass over ~1 GB)
template <class T> struct Staging {
  T* p; size_t n; std::unique_ptr<T[]> own;
  explicit Staging(size_t cnt) : p((T*)g_arena.take(cnt*sizeof(T))), n(cnt) { if (!p) { own.reset(new T[cnt]); p = own.get(); } }
  T* data() { return p; } size_t size() const { return n; } T& operator[](size_t i) { return p[i]; }
};
}  // namespace

// Process-wide cache of device allocations: a closed solver's blocks are kept and handed to the next one that asks for
// (about) the same size, because cudaMalloc / cudaFree of multi-GB blocks cost hundreds of milliseconds per optimize()
// call when the caller builds one solver per batch.  DYNOBA_NO_DEVCACHE=1 turns it off; the cache is trimmed when an
// allocation fails or when it holds more than DYNOBA_DEVCACHE_GB (default 48, 60 % of an 80 GB H100) gigabytes.
namespace {
struct DevCache {
  std::mutex mu; std::multimap<std::pair<int, size_t>, void*> blocks; size_t bytes = 0;   // keyed by (device, bytes)
  void* take(int dev, size_t need, size_t* got) {   // smallest cached block of this device with at least `need` bytes, if not much larger
    std::lock_guard<std::mutex> l(mu);
    auto it = blocks.lower_bound(std::make_pair(dev, need));
    if (it == blocks.end() || it->first.first != dev || it->first.second > need + need/4 + 4096) return nullptr;
    void* p = it->second; *got = it->first.second; bytes -= it->first.second; blocks.erase(it); return p;
  }
  void give(int dev, void* p, size_t n) {
    static const bool off = getenv("DYNOBA_NO_DEVCACHE") != nullptr;
    static const size_t cap = (size_t)(getenv("DYNOBA_DEVCACHE_GB") ? atof(getenv("DYNOBA_DEVCACHE_GB")) : 48.0)*(1ull << 30);
    std::lock_guard<std::mutex> l(mu);
    if (off || bytes + n > cap) { cudaFree(p); return; }
    blocks.emplace(std::make_pair(dev, n), p); bytes += n;
  }
  void trim() {       // (cudaFree takes the pointer's own device; the current device does not matter)
    std::lock_guard<std::mutex> l(mu); for (auto& b : blocks) cudaFree(b.second); blocks.clear(); bytes = 0;
  }
};
DevCache g_devcache;
}  // namespace

// clean = false: the caller overwrites every element it will ever read (band tiles: band_clear; Jacobian tiles: linearize;
// Schur slots: schur_stage) -- a recycled block then skips the multi-GB memset.
template <class T> static int dalloc(dynoba_solver* h, T** p, size_t count, bool clean = true) {
  *p = nullptr;
  if (count == 0) count = 1;
  const size_t bytes = (count*sizeof(T) + 255) & ~(size_t)255;
  size_t got = bytes;                        // a cached block may be larger than asked: its true size goes back with it
  void* q = g_devcache.take(h->device, bytes, &got);
  if (!q) {
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) { cudaGetLastError(); g_devcache.trim(); CK(cudaMalloc(&q, bytes)); }
  }
  if (clean) {
    // cudaMalloc does not zero and a recycled block holds the previous owner's data; several kernels leave entries they
    // own untouched (padding lanes, partial sums of early-exit CTAs) and read them back as zeros.  Ordered before any
    // later use: the solver's streams are non-blocking, so wait for the memset here.
    CK(cudaMemsetAsync(q, 0, bytes, h->stream)); CK(cudaStreamSynchronize(h->stream));
  }
  *p = (T*)q;
  h->allocs.emplace_back(q, got);
  return DYNOBA_OK;
}
// device copy of a host array: a clean dalloc (an empty array gets one zero element) and a copy on the handle's stream,
// waited for
template <class T> static int upload(dynoba_solver* h, T** p, const T* src, size_t count) {
  if (int rc = dalloc(h, p, count)) return rc;
  if (count) { CK(cudaMemcpyAsync(*p, src, count*sizeof(T), cudaMemcpyHostToDevice, h->stream)); CK(cudaStreamSynchronize(h->stream)); }
  return DYNOBA_OK;
}
template <class V> static int upload(dynoba_solver* h, typename V::value_type** p, const V& v) { return upload(h, p, v.data(), v.size()); }
static void free_device(dynoba_solver* h) {
  if (!h->allocs.empty()) cudaDeviceSynchronize();      // cudaFree used to imply this; cached blocks must be idle too
  for (auto& a : h->allocs) g_devcache.give(h->device, a.first, a.second);
  h->allocs.clear();
  h->finalized = false; h->linearized = false;
  h->cov_live = h->cov_lmk_ready = false; h->cov_tiles = COV_NONE; h->cov_stage = nullptr; h->cov_lmk = nullptr;
}
// hands one allocation of the handle back to the cache
static void release(dynoba_solver* h, void* q) {
  auto it = std::find_if(h->allocs.begin(), h->allocs.end(), [&](const std::pair<void*, size_t>& a) { return a.first == q; });
  if (it != h->allocs.end()) { g_devcache.give(h->device, it->first, it->second); h->allocs.erase(it); }
}
// One plain band problem (no cells) over the reduced system in buffers of its own, whatever partition the handle's solve
// uses: dynoba_marginal (factorisation stopped before column kend) and dynoba_marginal_covariance (kend < 0: every column)
static int plain_plan_create(dynoba_solver* h, BandPlan& mp, int kend) {
  mp = BandPlan{}; mp.outer_weight = 0;
  if (band_plan_layout(mp, h->band.n, h->band.bw, -1, 0, 1)) { h->err = "band layout failed"; return DYNOBA_ERR_BAD_ARG; }
  if (kend >= 0) mp.chains[0].Kend = kend;
  double* dbuf; int* ibuf; char* desc; int rc;
  if ((rc = dalloc(h, &dbuf, mp.n_doubles, false))) return rc;
  if ((rc = dalloc(h, &ibuf, mp.n_ints, false))) { release(h, dbuf); return rc; }
  if ((rc = dalloc(h, &desc, mp.n_desc_bytes))) { release(h, dbuf); release(h, ibuf); return rc; }
  band_plan_bind(mp, dbuf, ibuf, desc, nullptr);
  return DYNOBA_OK;
}
static void plain_plan_release(dynoba_solver* h, BandPlan& mp) {
  for (void* q : { (void*)mp.band.acc, (void*)mp.flags_base, (void*)mp.d_chains }) release(h, q);   // (d_chains: start of the descriptors)
}
// the values changed: the covariances of the old linearisation point go
static void cov_invalidate(dynoba_solver* h) {
  if (h->cov_live) { cudaStreamSynchronize(h->stream); plain_plan_release(h, h->cov_plan); release(h, h->cov_stage); }
  if (h->cov_lmk) release(h, h->cov_lmk);
  h->cov_live = h->cov_lmk_ready = false; h->cov_tiles = COV_NONE; h->cov_stage = nullptr; h->cov_lmk = nullptr;
}

// copy of a caller's array into the handle: parallel, so that the first touch of the fresh pages (the expensive part of a
// several-hundred-MB copy) is spread over the cores.  Runs on its own thread count: torchrun pins OMP_NUM_THREADS to 1.
template <class V, class T> static void par_assign(V& v, const T* src, size_t count) {
  v.resize(count);
  const size_t chunk = (size_t)1 << 18;
  const int64_t nchunk = (int64_t)((count + chunk - 1)/chunk);
  const int nt = (int)std::max<int64_t>(1, std::min<int64_t>(std::min(omp_get_num_procs(), 32), nchunk));
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int64_t c = 0; c < nchunk; c++) {
    const size_t a = (size_t)c*chunk, e = std::min(count, a + chunk);
    std::memcpy(v.data() + a, src + a, (e - a)*sizeof(T));
  }
}

extern "C" {

int dynoba_version(void) { return 100; }

const char* dynoba_status_string(int s) {
  switch (s) {
    case DYNOBA_OK: return "ok";
    case DYNOBA_ERR_BAD_ARG: return "bad argument";
    case DYNOBA_ERR_STATE: return "bad call order";
    case DYNOBA_ERR_CUDA: return "CUDA error / no usable device";
    case DYNOBA_ERR_INDETERMINATE: return "indeterminate linear system";
    case DYNOBA_ERR_UNSUPPORTED: return "unsupported topology";
    case DYNOBA_ERR_COMM: return "all-reduce callback failed";
    default: return "unknown";
  }
}
const char* dynoba_last_error(dynoba_handle h) { return h ? h->err.c_str() : "null handle"; }

void dynoba_lm_default_params(dynoba_lm_params* p) {
  p->lambda_initial = 1e-5; p->lambda_factor = 10.0; p->lambda_upper_bound = 1e5; p->lambda_lower_bound = 0.0;
  p->min_model_fidelity = 1e-3; p->relative_error_tol = 1e-5; p->absolute_error_tol = 1e-5; p->error_tol = 0.0;
  p->max_iterations = 100; p->verbosity = 0;
}

int dynoba_create(int device, dynoba_handle* out) {
  if (!out) return DYNOBA_ERR_BAD_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return DYNOBA_ERR_CUDA;  // no CPU fallback
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) return DYNOBA_ERR_CUDA;   // sm_90a code only
  dynoba_solver* h = new dynoba_solver();
  h->device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return DYNOBA_ERR_CUDA; }
  for (auto& e : h->ev) cudaEventCreate(&e);
  { int lo = 0, hi = 0; cudaDeviceGetStreamPriorityRange(&lo, &hi); cudaStreamCreateWithPriority(&h->stream2, cudaStreamNonBlocking, hi); }
  cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming); cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming);
  *out = h;
  return DYNOBA_OK;
}

int dynoba_destroy(dynoba_handle h) {
  if (!h) return DYNOBA_ERR_BAD_ARG;
  cudaSetDevice(h->device);
  free_device(h);
  for (auto& e : h->ev) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->stream2) cudaStreamDestroy(h->stream2);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork); if (h->ev_join) cudaEventDestroy(h->ev_join);
  delete h;
  return DYNOBA_OK;
}

static int64_t n_vars(const dynoba_solver* h, int kind) { return (int64_t)h->vals[kind].size()/KINDS[kind].width; }
static bool has_nav(const dynoba_solver* h) { return !h->vals[DYNOBA_VEL3].empty() || !h->vals[DYNOBA_BIAS6].empty(); }

int dynoba_set_variables(dynoba_handle h, int kind, int64_t n, const uint64_t* keys, const double* data) {
  ARG(h, "null handle"); ARG(n >= 0 && (n == 0 || data), "null data"); ARG(valid_kind(kind), "bad variable kind");
  std::vector<double>* dst = &h->vals[kind];
  const int w = KINDS[kind].width;
  const bool same_shape = dst->size() == (size_t)n*w;
  dst->assign(data, data + (size_t)n*w);
  if (keys) h->keys[kind].assign(keys, keys + n); else if (!same_shape) h->keys[kind].clear();   // a value refresh keeps the keys
  if (h->finalized && same_shape) {
    // refresh device values only (layout unchanged).  When the kind shares the pose SoA with other pose-like kinds, only
    // its columns are replaced in the current device image.
    cudaSetDevice(h->device);
    const VarLayout& L = h->layout;
    double* img_d = image_of(h->cur, kind);
    std::vector<double> img = L.blank_image(kind);
    if (KINDS[kind].poselike && L.NP() > L.count(kind)) { CK(cudaMemcpyAsync(img.data(), img_d, img.size()*8, cudaMemcpyDeviceToHost, h->stream)); CK(cudaStreamSynchronize(h->stream)); }
    L.scatter_values(kind, data, img.data());
    CK(cudaMemcpyAsync(img_d, img.data(), img.size()*8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->linearized = false; cov_invalidate(h);
  } else if (h->finalized) {
    free_device(h);
  }
  return DYNOBA_OK;
}

int dynoba_set_aux_poses(dynoba_handle h, int64_t n, const double* data) {
  ARG(h, "null handle"); ARG(n >= 0 && (n == 0 || data), "null data");
  h->aux.assign(data, data + (size_t)n*12);
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}
int dynoba_set_calibration(dynoba_handle h, const double calib[6]) {
  ARG(h, "null handle"); ARG(calib, "null calib");
  for (int i = 0; i < 6; i++) { h->calib[i] = calib[i]; h->cur.K[i] = calib[i]; h->cand.K[i] = calib[i]; }
  h->linearized = false; cov_invalidate(h);
  return DYNOBA_OK;
}

int dynoba_add_factors(dynoba_handle h, int type, int64_t n, const int32_t* idx, const double* meas, const double* sigma,
                       int sigma_dim, int64_t sigma_count, double robust_k, const int32_t* aux_idx) {
  ARG(h, "null handle"); ARG(type >= 0 && type < F_NUM_TYPES, "bad factor type");
  const TypeInfo ti = type_info(type);
  ARG(n >= 0 && (n == 0 || idx), "null idx"); ARG(ti.meas == 0 || n == 0 || meas, "factor type needs measurements");
  const bool imu = type == F_COMBINED_IMU15;
  // the reference never robustifies the visual-inertial factors (VisionImuBackendModule.hpp:114-243)
  if (is_nav_type(type) && robust_k > 0) { h->err = "the IMU factor and the velocity / bias priors take no robust kernel (robust_k must be <= 0)"; return DYNOBA_ERR_UNSUPPORTED; }
  if (imu) {
    ARG(sigma && sigma_dim == IMU_SQRT_INFO, "COMBINED_IMU15 takes its 15x15 square-root information: sigma_dim must be 225");
  } else {
    ARG(sigma && (sigma_dim == 1 || sigma_dim == ti.dim), "sigma_dim must be 1 or the residual dimension");
  }
  ARG(sigma_count == 1 || sigma_count == n, "sigma_count must be 1 or n"); ARG(!ti.needs_aux || n == 0 || aux_idx, "factor type needs aux_idx");
  HostBlock b; b.type = type; b.n = n;
  par_assign(b.idx, idx, (size_t)n*ti.arity);
  if (ti.meas) par_assign(b.meas, meas, (size_t)n*ti.meas);
  b.sigma_dim = sigma_dim; b.bcast = sigma_count == 1 && n != 1;
  b.sigma.assign(sigma, sigma + (size_t)sigma_count*sigma_dim);
  if (imu) {
    // noiseModel::Gaussian's R: finite, upper triangular Cholesky factor with a positive diagonal
    for (double s : b.sigma) ARG(std::isfinite(s), "square-root information must be finite");
    for (size_t o = 0; o < b.sigma.size(); o += IMU_SQRT_INFO) for (int k = 0; k < 15; k++) ARG(b.sigma[o + 16*k] > 0, "square-root information must have a positive diagonal");
  }
  else for (double s : b.sigma) ARG(s > 0, "sigma must be positive");
  if (is_linear_type(type)) {   // a linearised factor is already whitened: no noise model
    for (double s : b.sigma) ARG(s == 1.0, "LINEAR_PP3 / LINEAR_PPP3 take no noise model: sigma must be 1");
    ARG(robust_k == 0.0, "LINEAR_PP3 / LINEAR_PPP3 take no noise model: robust_k must be 0");
  }
  if (imu) for (size_t i = 0; i < b.meas.size(); i++) ARG(std::isfinite(b.meas[i]), "IMU measurement must be finite");
  b.robust_k = robust_k;
  if (aux_idx) { par_assign(b.aux, aux_idx, (size_t)n); b.has_aux = true; }
  h->blocks.push_back(std::move(b));
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

}  // extern "C"

// the one implementation behind dynoba_add_linear_prior and dynoba_add_linear_prior_vars (indices are checked at finalize,
// where the variable counts are known)
static int add_prior(dynoba_solver* h, int32_t n, const int32_t* kind, const int32_t* idx, const double* lin, const double* G,
                     const double* g, double f, bool legacy) {
  ARG(n > 0 && n <= 512 && kind && idx && lin && G && g, "bad prior");
  HostPrior P; P.kind.assign(kind, kind + n); P.idx.assign(idx, idx + n); P.f = f; P.legacy = legacy;
  size_t nlin = 0, dim = 0;
  for (int i = 0; i < n; i++) {
    ARG(poselike_kind(kind[i]), "a prior slot must be of kind DYNOBA_POSE6, DYNOBA_VEL3 or DYNOBA_BIAS6");
    dim += KINDS[kind[i]].tdim; nlin += KINDS[kind[i]].width;
  }
  P.lin.assign(lin, lin + nlin); P.G.assign(G, G + dim*dim); P.g.assign(g, g + dim);
  { std::vector<std::pair<int32_t, int32_t>> srt(n); for (int i = 0; i < n; i++) srt[i] = { kind[i], idx[i] };
    std::sort(srt.begin(), srt.end()); ARG(std::adjacent_find(srt.begin(), srt.end()) == srt.end(), "a prior lists a variable twice"); }
  for (size_t r = 0; r < dim; r++) for (size_t c = 0; c < r; c++)
    ARG(std::fabs(P.G[r*dim + c] - P.G[c*dim + r]) <= 1e-9*(std::fabs(P.G[r*dim + r]) + std::fabs(P.G[c*dim + c]) + 1e-300), "prior information matrix is not symmetric");
  h->priors.push_back(std::move(P));
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

extern "C" {

int dynoba_add_linear_prior(dynoba_handle h, int32_t n, const int32_t* pose_idx, const double* lin_poses, const double* G, const double* g, double f) {
  ARG(h, "null handle"); ARG(n > 0 && n <= 512 && pose_idx && lin_poses && G && g, "bad prior");
  if (has_nav(h)) { h->err = "dynoba_add_linear_prior is not available with velocity / bias variables"; return DYNOBA_ERR_UNSUPPORTED; }
  const std::vector<int32_t> kind(n, DYNOBA_POSE6);
  return add_prior(h, n, kind.data(), pose_idx, lin_poses, G, g, f, true);
}
int dynoba_add_linear_prior_vars(dynoba_handle h, int32_t n, const int32_t* kind, const int32_t* idx, const double* lin,
                                 const double* G, const double* g, double f) {
  ARG(h, "null handle");
  return add_prior(h, n, kind, idx, lin, G, g, f, false);
}

int dynoba_set_pose_order(dynoba_handle h, int64_t n, const int32_t* rank) {
  ARG(h, "null handle"); ARG(n >= 0 && (n == 0 || rank), "null rank");
  h->hints[DYNOBA_POSE6].assign(rank, rank + n);
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

int dynoba_set_variable_order(dynoba_handle h, int kind, int64_t n, const int32_t* rank) {
  ARG(h, "null handle"); ARG(kind == DYNOBA_VEL3 || kind == DYNOBA_BIAS6, "variable order hints are for DYNOBA_VEL3 / DYNOBA_BIAS6 (poses: dynoba_set_pose_order)");
  ARG(n >= 0 && (n == 0 || rank), "null rank");
  h->hints[kind].assign(rank, rank + n);
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

int dynoba_set_reduce(dynoba_handle h, dynoba_reduce_fn fn, void* ctx) {
  ARG(h, "null handle");
  if (fn && has_nav(h)) { h->err = "dynoba_set_reduce is not available with velocity / bias variables"; return DYNOBA_ERR_UNSUPPORTED; }
  h->reduce = fn; h->red_ctx = ctx;
  return DYNOBA_OK;
}
int dynoba_set_tuning(dynoba_handle h, const char* name, double value) {
  ARG(h, "null handle"); ARG(name, "null name");
  if (!std::strcmp(name, "outer_weight")) { h->plan.outer_weight = value; if (h->finalized) free_device(h); }
  else if (!std::strcmp(name, "band_ctas_per_chain")) band_set_tuning(std::max(0, (int)value));
  else if (!std::strcmp(name, "band_profile")) band_set_tuning(-1);
  else ARG(false, "unknown tuning parameter");
  return DYNOBA_OK;
}
int dynoba_plan_partition(int32_t n_poses, int32_t bandwidth, int32_t world, int32_t* first_position) {
  if (n_poses <= 0 || world < 1 || !first_position) return DYNOBA_ERR_BAD_ARG;
  std::vector<int> b(world + 1);
  if (band_plan_partition(6*n_poses, bandwidth, world, b.data()) < 0) return DYNOBA_ERR_BAD_ARG;
  for (int r = 0; r <= world; r++) first_position[r] = std::min(b[r]/6, n_poses);
  first_position[world] = n_poses;
  return DYNOBA_OK;
}
int dynoba_set_partition(dynoba_handle h, int ncells) {
  ARG(h, "null handle"); ARG(ncells >= -1 && ncells <= MAX_CELLS, "ncells out of range");
  h->ncell_request = ncells;
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

int dynoba_set_shard(dynoba_handle h, int rank, int world, dynoba_allreduce_fn fn, void* ctx, int min_bandwidth) {
  ARG(h, "null handle"); ARG(world >= 1 && rank >= 0 && rank < world, "bad rank/world"); ARG(world == 1 || fn, "world > 1 needs an all-reduce");
  if (world > 1 && has_nav(h)) { h->err = "dynoba_set_shard is not available with velocity / bias variables"; return DYNOBA_ERR_UNSUPPORTED; }
  h->rank = rank; h->world = world; h->allreduce = fn; h->ar_ctx = ctx; h->min_bw = min_bandwidth;
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ finalize
// algorithmic bytes of a block's linearize: factor record read once + whitened tiles written once (variable reads left out)
static int64_t block_bytes(const HostBlock& b) {
  const TypeInfo ti = type_info(b.type);
  return b.n*(4*ti.arity + 8*ti.meas + 8*b.sigma_dim + (b.has_aux ? 4 : 0) + 8*(ti.dim*ti.jcols + ti.dim));
}
static int uf_find(std::vector<int32_t>& p, int x) { while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; } return x; }
// x = v where better(v, x), atomically with relaxed ordering (a min / max the parallel loops over factors share)
template <class Better> static void atomic_keep(int32_t& x, int32_t v, Better better) {
  int32_t cur = __atomic_load_n(&x, __ATOMIC_RELAXED);
  while (better(v, cur) && !__atomic_compare_exchange_n(&x, &cur, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
}

static int finalize_impl(dynoba_solver* h) {
  if (h->finalized) return DYNOBA_OK;
  cudaSetDevice(h->device);
  // host-side symbolic phase runs on up to 32 threads regardless of OMP_NUM_THREADS (torchrun pins it to 1)
  struct OmpScope { int saved; OmpScope() : saved(omp_get_max_threads()) { int t = std::min(omp_get_num_procs(), 32); if (const char* e = getenv("DYNOBA_THREADS")) t = std::max(1, atoi(e)); omp_set_num_threads(t); } ~OmpScope() { omp_set_num_threads(saved); } } omp_scope;
  const bool timing = getenv("DYNOBA_TIMING") != nullptr;
  auto t_last = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) { if (!timing) return; auto t = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[dynoba finalize] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(t - t_last).count()); t_last = t; };
  h->layout = VarLayout{n_vars(h, DYNOBA_POSE6), n_vars(h, DYNOBA_POINT3), n_vars(h, DYNOBA_FLOW2), n_vars(h, DYNOBA_VEL3), n_vars(h, DYNOBA_BIAS6)};
  VarLayout& L = h->layout;
  const int64_t np = L.np, npt = L.npt, nfl = L.nfl, nv = L.nv, nb = L.nb, NP = L.NP();   // NP: pose-like variables
  const int64_t naux = (int64_t)h->aux.size()/KINDS[DYNOBA_POSE6].width;
  ARG(h->hints[DYNOBA_POSE6].empty() || (int64_t)h->hints[DYNOBA_POSE6].size() == np, "pose order hint length != number of poses");
  ARG(h->hints[DYNOBA_VEL3].empty() || (int64_t)h->hints[DYNOBA_VEL3].size() == nv, "velocity order hint length != number of velocities");
  ARG(h->hints[DYNOBA_BIAS6].empty() || (int64_t)h->hints[DYNOBA_BIAS6].size() == nb, "bias order hint length != number of biases");
  const bool legacy_prior = std::any_of(h->priors.begin(), h->priors.end(), [](const HostPrior& P) { return P.legacy; });
  if (NP > np && (legacy_prior || h->world > 1 || h->reduce)) {
    h->err = "velocity / bias variables cannot be combined with dynoba_add_linear_prior, dynoba_set_shard or dynoba_set_reduce";
    return DYNOBA_ERR_UNSUPPORTED;
  }
  // ---- validate indices
  for (auto& b : h->blocks) {
    const TypeInfo ti = type_info(b.type);
    int bad = 0;
    int64_t lim[6];
    for (int k = 0; k < ti.arity; k++) lim[k] = L.count(ti.cls[k]);
#pragma omp parallel for schedule(static) reduction(|:bad)
    for (int64_t i = 0; i < b.n; i++) {
      for (int k = 0; k < ti.arity; k++) {
        const int32_t ix = b.idx[i*ti.arity + k];
        if (!(ix >= 0 && ix < lim[k])) bad |= 1;
      }
      if (b.has_aux && !(b.aux[i] >= 0 && b.aux[i] < naux)) bad |= 2;
    }
    ARG(!(bad & 1), "factor index out of range"); ARG(!(bad & 2), "aux index out of range");
  }
  lap("validate");
  // ---- pose ordering
  L.pos = L.poselike_positions(h->hints);
  // ---- landmark groups (union-find across factors that touch two landmarks)
  const int64_t nl = npt + nfl;
  std::vector<int32_t> uf(nl); std::iota(uf.begin(), uf.end(), 0);
  auto lmk_id = [&](int cls, int ix) { return cls == VC_POINT ? ix : (int)npt + ix; };
  for (auto& b : h->blocks) {
    const TypeInfo ti = type_info(b.type);
    if (ti.nlmk < 2) continue;
    for (int64_t i = 0; i < b.n; i++) {
      int first = -1;
      for (int k = 0; k < ti.arity; k++) if (ti.cls[k] != VC_POSE) {
        const int l = lmk_id(ti.cls[k], b.idx[i*ti.arity + k]);
        if (first < 0) first = l; else { const int a = uf_find(uf, first), c = uf_find(uf, l); if (a != c) uf[c] = a; }
      }
    }
  }
  std::vector<int32_t, NoInitAlloc<int32_t>> root(nl);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < nl; i++) { int x = (int)i; while (uf[x] != x) x = uf[x]; root[i] = x; }      // read-only find
  std::vector<int32_t> gmin(nl, INT32_MAX), gmax(nl, -1), gblk(nl, -1), gcount(nl, 0), gsec(nl, INT32_MAX);
  for (int64_t i = 0; i < nl; i++) gcount[root[i]]++;
  int spread = 0, pos_lo = INT32_MAX, pos_hi = -1;     // pos_lo..pos_hi: pose positions this rank's factors touch
  for (size_t bi = 0; bi < h->blocks.size(); bi++) {
    auto& b = h->blocks[bi]; const TypeInfo ti = type_info(b.type);
    b.pose_only = ti.nlmk == 0;
    int lslot = -1; for (int k = 0; k < ti.arity; k++) if (!is_poselike(ti.cls[k])) { lslot = k; break; }
    int bspread = 0, blo = INT32_MAX, bhi = -1;
#pragma omp parallel for schedule(static) reduction(max:bspread) reduction(min:blo) reduction(max:bhi)
    for (int64_t i = 0; i < b.n; i++) {
      int lo = INT32_MAX, hi = -1;
      for (int k = 0; k < ti.arity; k++) if (is_poselike(ti.cls[k])) { const int p = L.column(ti.cls[k], b.idx[i*ti.arity + k]); lo = std::min(lo, p); hi = std::max(hi, p); }
      blo = std::min(blo, lo); bhi = std::max(bhi, hi);
      if (lslot < 0) { bspread = std::max(bspread, hi - lo); continue; }
      const int g = root[lmk_id(ti.cls[lslot], b.idx[i*ti.arity + lslot])];
      atomic_keep(gmin[g], lo, std::less<int32_t>()); atomic_keep(gmax[g], hi, std::greater<int32_t>());
      if (ti.npose >= 2) {   // secondary ordering key: user index of the last pose slot (object-major for DynOSAM's H keys)
        int last = -1; for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POSE) last = b.idx[i*ti.arity + k];
        atomic_keep(gsec[g], last, std::less<int32_t>());
      }
      int32_t gb = __atomic_load_n(&gblk[g], __ATOMIC_RELAXED);
      while (gb != (int)bi && gb != -2) {
        const int32_t want = gb == -1 ? (int32_t)bi : -2;
        if (__atomic_compare_exchange_n(&gblk[g], &gb, want, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) break;
      }
    }
    spread = std::max(spread, bspread); pos_lo = std::min(pos_lo, blo); pos_hi = std::max(pos_hi, bhi);
  }
  for (int64_t g = 0; g < nl; g++) if (gmax[g] >= 0) spread = std::max(spread, gmax[g] - gmin[g]);
  for (auto& P : h->priors) {       // a prior couples all of its variables
    int lo = INT32_MAX, hi = -1;
    for (size_t i = 0; i < P.idx.size(); i++) {
      const int p = L.column_checked(P.kind[i], P.idx[i]);
      ARG(p >= 0, "prior variable out of range"); lo = std::min(lo, p); hi = std::max(hi, p);
    }
    spread = std::max(spread, hi - lo); pos_lo = std::min(pos_lo, lo); pos_hi = std::max(pos_hi, hi);
  }
  // group rank: by first pose position, then root id
  std::vector<int32_t> gorder; gorder.reserve(nl);
  for (int64_t g = 0; g < nl; g++) if (root[g] == g) gorder.push_back((int32_t)g);
  // group order: by owning factor block (groups spanning blocks last), then by the secondary key (object-major for
  // two-pose factor types so that consecutive landmarks share their clique), else by the first pose position
  std::vector<int64_t> gkey(nl, 0);
#pragma omp parallel for schedule(static)
  for (int64_t g = 0; g < nl; g++) {
    const int64_t cls = gblk[g] >= 0 ? gblk[g] : (1 << 20);
    const int64_t sec = gsec[g] != INT32_MAX ? gsec[g] : (gmin[g] == INT32_MAX ? 0 : gmin[g]);
    gkey[g] = (cls << 40) | (sec & ((1LL << 40) - 1));
  }
  {
    bool sorted = true;
    for (size_t i = 1; i < gorder.size() && sorted; i++) sorted = gkey[gorder[i-1]] <= gkey[gorder[i]];
    if (!sorted) __gnu_parallel::stable_sort(gorder.begin(), gorder.end(), [&](int a, int b) { return gkey[a] < gkey[b]; });
  }
  std::vector<int32_t> grank(nl, 0);
  for (size_t r = 0; r < gorder.size(); r++) grank[gorder[r]] = (int32_t)r;
  std::vector<int32_t> lrank(nl);                       // group rank of every landmark (one gather per factor later)
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < nl; i++) lrank[i] = grank[root[i]];
  // landmark device indices: group order
  L.pt_new = positions_by(npt, [&](int32_t a, int32_t b) { return lrank[a] < lrank[b]; });
  L.fl_new = positions_by(nfl, [&](int32_t a, int32_t b) { return lrank[npt + a] < lrank[npt + b]; });
  lap("groups + landmark order");
  // ---- band structure: cell decomposition of the reduced system (kernels_band.cu)
  {
    int bw = 6*spread + 5; if (bw < h->min_bw) bw = h->min_bw;
    if (band_plan_layout(h->plan, (int)(6*NP), bw, h->ncell_request, h->rank, h->world)) { h->err = "band layout failed"; return DYNOBA_ERR_BAD_ARG; }
    double* dbuf; int* ibuf; char* desc; double* dp = nullptr; int rc;
    if ((rc = dalloc(h, &dbuf, h->plan.n_doubles, false))) return rc;     // accumulated part: band_clear; work buffers: written before read
    if ((rc = dalloc(h, &ibuf, h->plan.n_ints, false))) return rc;        // flags: cleared before every factorisation launch
    if ((rc = dalloc(h, &desc, h->plan.n_desc_bytes))) return rc;
    if (h->plan.band.ncell > 0) { if ((rc = dalloc(h, &dp, (size_t)h->plan.band.n_pad))) return rc; }
    band_plan_bind(h->plan, dbuf, ibuf, desc, dp);
    if (h->world > 1) {
      // every rank must have arrived at the same layout (the collectives exchange raw buffers): agree on n and bw.  The sums of
      // x and x^2 over the ranks equal world*x and world*x^2 only when all ranks hold the same x -- every rank sees the same sums,
      // so a disagreement is reported everywhere instead of hanging a collective.
      const double mine[4] = { (double)h->band.n, (double)h->band.n*(double)h->band.n, (double)h->band.bw, (double)h->band.bw*(double)h->band.bw };
      double got[4];
      CK(cudaMemcpyAsync(dbuf, mine, sizeof(mine), cudaMemcpyHostToDevice, h->stream));
      if (h->allreduce(h->ar_ctx, dbuf, 4, (void*)h->stream) != 0) { h->err = "all-reduce callback failed"; return DYNOBA_ERR_COMM; }
      CK(cudaMemcpyAsync(got, dbuf, sizeof(got), cudaMemcpyDeviceToHost, h->stream)); CK(cudaStreamSynchronize(h->stream));
      for (int k = 0; k < 4; k++) if (got[k] != h->world*mine[k]) {
        h->err = "ranks disagree on the reduced system's size or bandwidth: pass the bandwidth of the unsharded graph as min_bandwidth to dynoba_set_shard";
        return DYNOBA_ERR_BAD_ARG;
      }
      if (h->reduce && h->band.ncell > 0) {
        // which part of the reduced system does every rank touch?  All-gather [first, last] pose position (a sum over slots
        // that only their rank fills): the per-cell reduces then only move the part of a cell's tiles that a rank other than
        // its owner contributes to -- a halo of one co-visibility window when the landmarks are sharded in time.
        std::vector<double> rng((size_t)2*h->world, 0.0);
        rng[2*h->rank] = pos_hi >= 0 ? (double)pos_lo : 1.0; rng[2*h->rank + 1] = pos_hi >= 0 ? (double)pos_hi : 0.0;    // (empty: lo > hi)
        CK(cudaMemcpyAsync(dbuf, rng.data(), rng.size()*8, cudaMemcpyHostToDevice, h->stream));
        if (h->allreduce(h->ar_ctx, dbuf, rng.size(), (void*)h->stream) != 0) { h->err = "all-reduce callback failed"; return DYNOBA_ERR_COMM; }
        CK(cudaMemcpyAsync(rng.data(), dbuf, rng.size()*8, cudaMemcpyDeviceToHost, h->stream)); CK(cudaStreamSynchronize(h->stream));
        std::vector<int> lo(h->world), hi(h->world);
        for (int r = 0; r < h->world; r++) { lo[r] = 6*(int)rng[2*r]; hi[r] = 6*(int)rng[2*r + 1] + 5; }
        band_plan_trim(h->plan, lo.data(), hi.data());
      }
    }
  }
  DevBand& B = h->band;
  // ---- variables
  DevVars& V = h->cur;
  V.np = (int)NP; V.np_stride = L.stride(DYNOBA_POSE6); V.nl = (int)npt; V.nl_stride = L.stride(DYNOBA_POINT3); V.nf = (int)nfl; V.nf_stride = L.stride(DYNOBA_FLOW2);
  V.naux = (int)naux; V.naux_stride = pad32(naux);
  for (int i = 0; i < 6; i++) V.K[i] = h->calib[i];
  h->cand = V;
  {
    std::vector<double> soa = L.blank_image(DYNOBA_POSE6);
    for (int kind : {DYNOBA_POSE6, DYNOBA_VEL3, DYNOBA_BIAS6}) L.scatter_values(kind, h->vals[kind].data(), soa.data());
    int rc;
    if ((rc = upload(h, &h->cur.pose, soa)) || (rc = upload(h, &h->cand.pose, soa))) return rc;
    soa = L.blank_image(DYNOBA_POINT3); L.scatter_values(DYNOBA_POINT3, h->vals[DYNOBA_POINT3].data(), soa.data());
    if ((rc = upload(h, &h->cur.point, soa)) || (rc = dalloc(h, &h->cand.point, soa.size())) || (rc = dalloc(h, &h->dl_point, soa.size()))) return rc;
    soa = L.blank_image(DYNOBA_FLOW2); L.scatter_values(DYNOBA_FLOW2, h->vals[DYNOBA_FLOW2].data(), soa.data());
    if ((rc = upload(h, &h->cur.flow, soa)) || (rc = dalloc(h, &h->cand.flow, soa.size())) || (rc = dalloc(h, &h->dl_flow, soa.size()))) return rc;
    soa.assign((size_t)12*V.naux_stride, 0.0);
    for (int64_t i = 0; i < naux; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*V.naux_stride + i] = h->aux[i*12 + k];
    double* da; if ((rc = upload(h, &da, soa))) return rc;
    h->cur.aux = da; h->cand.aux = da;
  }
  lap("band + variables upload");
  // ---- factor blocks
  h->supported = true; h->jac_bytes = 96*(np + naux) + 24*npt + 16*nfl + 24*nv + 48*nb;
  int part = 0, bs = 0;
  struct GenRef { int32_t rank, blk, idx; };
  std::vector<GenRef> gen_refs;
  std::lock_guard<std::mutex> arena_lock(g_arena.mu);
  {
    size_t need = 0;
    for (auto& b : h->blocks) { const TypeInfo ti = type_info(b.type); const size_t st = pad32(b.n);
      need += ((size_t)ti.arity*4 + (size_t)std::max(ti.meas, 1)*8 + (size_t)b.sigma_dim*8 + 4)*st + 4*256; }
    g_arena.reserve(need);
  }
  for (size_t bi = 0; bi < h->blocks.size(); bi++) {
    auto& b = h->blocks[bi]; const TypeInfo ti = type_info(b.type);
    const int64_t n = b.n; const int stride = pad32(n);
    int lslot = -1, pslot = -1;
    for (int k = 0; k < ti.arity; k++) { if (!is_poselike(ti.cls[k]) && lslot < 0) lslot = k; if (ti.cls[k] == VC_POSE && pslot < 0) pslot = k; }
    // (serial value-initialisation of 10^7-element vectors costs tens of milliseconds each: first-touch them in parallel)
    b.perm.resize(n);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) b.perm[i] = (int32_t)i;
    std::unique_ptr<int32_t[]> frank_buf; int32_t* frank = nullptr;
    if (lslot >= 0) {
      frank_buf.reset(new int32_t[n]); frank = frank_buf.get();
      std::unique_ptr<int64_t[]> key_buf(new int64_t[n]); int64_t* key = key_buf.get();
#pragma omp parallel for schedule(static)
      for (int64_t i = 0; i < n; i++) {
        frank[i] = lrank[lmk_id(ti.cls[lslot], b.idx[i*ti.arity + lslot])];
        key[i] = ((int64_t)frank[i] << 32) | (uint32_t)L.column(VC_POSE, b.idx[i*ti.arity + pslot]);
      }
      order_block_factors(b.perm.data(), frank, key, n, gorder.size());
    }
    lap("  blk sort");
    // SoA host images, padding filled explicitly below
    Staging<int32_t> hidx((size_t)ti.arity*stride);
    Staging<double> hmeas((size_t)std::max(ti.meas, 1)*stride);
    Staging<double> hsig((size_t)b.sigma_dim*stride);
    Staging<int32_t> haux((size_t)stride);
    const bool pinned = !hidx.own && !hmeas.own && !hsig.own && !haux.own;
    auto h2d = [&](void* dst, const void* src, size_t bytes) { return pinned ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream2) : cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice); };
    for (int64_t s = n; s < stride; s++) {
      for (int k = 0; k < ti.arity; k++) hidx[(size_t)k*stride + s] = 0;
      for (int k = 0; k < std::max(ti.meas, 1); k++) hmeas[(size_t)k*stride + s] = 0.0;
      for (int k = 0; k < b.sigma_dim; k++) hsig[(size_t)k*stride + s] = 1.0;
      haux[s] = 0;
    }
    if (ti.meas == 0) {
#pragma omp parallel for schedule(static)
      for (int64_t s = 0; s < n; s++) hmeas[s] = 0.0;
    }
    if (!b.has_aux) {
#pragma omp parallel for schedule(static)
      for (int64_t s = 0; s < n; s++) haux[s] = 0;
    }
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < n; s++) {
      const int64_t o = b.perm[s];
      for (int k = 0; k < ti.arity; k++) {
        const int32_t ix = b.idx[o*ti.arity + k];
        hidx[(size_t)k*stride + s] = L.column(ti.cls[k], ix);
      }
      for (int k = 0; k < ti.meas; k++) hmeas[(size_t)k*stride + s] = b.meas[o*ti.meas + k];
      if (b.type == F_COMBINED_IMU15)   // square-root information, used as given
        for (int k = 0; k < b.sigma_dim; k++) hsig[(size_t)k*stride + s] = b.bcast ? b.sigma[k] : b.sigma[o*b.sigma_dim + k];
      else
        for (int k = 0; k < b.sigma_dim; k++) hsig[(size_t)k*stride + s] = 1.0/(b.bcast ? b.sigma[k] : b.sigma[o*b.sigma_dim + k]);
      if (b.has_aux) haux[s] = b.aux[o];
    }
    lap("  blk soa fill");
    DevBlock& d = b.dev; d = DevBlock{};
    d.type = b.type; d.n = (int)n; d.stride = stride; d.sigma_dim = b.sigma_dim; d.robust_k = b.robust_k;
    int* di; double* dm; double* ds; int* dax = nullptr; int rc;
    if ((rc = dalloc(h, &di, hidx.size(), false))) return rc; CK(h2d(di, hidx.data(), hidx.size()*4));
    if ((rc = dalloc(h, &dm, hmeas.size(), false))) return rc; CK(h2d(dm, hmeas.data(), hmeas.size()*8));
    if ((rc = dalloc(h, &ds, hsig.size(), false))) return rc; CK(h2d(ds, hsig.data(), hsig.size()*8));
    if (b.has_aux) { if ((rc = dalloc(h, &dax, haux.size(), false))) return rc; CK(h2d(dax, haux.data(), haux.size()*4)); }
    d.idx = di; d.meas = dm; d.isig = ds; d.aux = dax;
    if ((rc = dalloc(h, &d.J, (size_t)ti.dim*ti.jcols*stride, false))) return rc;
    if ((rc = dalloc(h, &d.b, (size_t)ti.dim*stride))) return rc;
    if (numeric_grid(b.type, (int)n) > 0) { if ((rc = dalloc(h, &d.num_scratch, (size_t)numeric_grid(b.type, (int)n)))) return rc; }
    lap("  blk upload+alloc");
    // groups: CSR over every landmark group that has factors in this block; groups this block cannot own alone
    // (several points, or factors in other blocks too) are marked -1 and collected for the general path
    b.simple = false;
    if (lslot >= 0) {
      std::vector<int32_t> gp, gl;
      {   // group boundaries of the sorted factor list, found in parallel segments and concatenated in order
        const int nseg = std::max(1, std::min<int>(omp_get_max_threads(), (int)(n/65536) + 1));
        std::vector<std::vector<int32_t>> sgp(nseg), sgl(nseg); std::vector<std::vector<GenRef>> sgen(nseg);
#pragma omp parallel for schedule(static, 1)
        for (int t = 0; t < nseg; t++) {
          const int64_t s0 = n*t/nseg, s1 = n*(t + 1)/nseg;
          for (int64_t s = s0; s < s1; s++) {
            const int64_t o = b.perm[s];
            const int l = lmk_id(ti.cls[lslot], b.idx[o*ti.arity + lslot]);
            const bool simple = ti.nlmk == 1 && gblk[root[l]] == (int)bi && gcount[root[l]] == 1;
            if (s == 0 || frank[o] != frank[b.perm[s-1]]) { sgp[t].push_back((int32_t)s); sgl[t].push_back(simple ? hidx[(size_t)lslot*stride + s] : -1); }
            if (!simple) sgen[t].push_back({ grank[root[l]], (int32_t)bi, (int32_t)s });
          }
        }
        for (int t = 0; t < nseg; t++) { gp.insert(gp.end(), sgp[t].begin(), sgp[t].end()); gl.insert(gl.end(), sgl[t].begin(), sgl[t].end());
                                         gen_refs.insert(gen_refs.end(), sgen[t].begin(), sgen[t].end()); }
      }
      gp.push_back((int32_t)n);
      int* dgp; int* dgl;
      if ((rc = upload(h, &dgp, gp)) || (rc = upload(h, &dgl, gl))) return rc;
      d.n_groups = (int)gl.size(); d.grp_ptr = dgp; d.grp_lmk = dgl;
      b.simple = true;
      // ---- window decomposition (kernels_window.cu) for the 3-dof landmark types
      const bool win_type = b.type == F_POSE2POINT3 || b.type == F_STEREO3 || b.type == F_HYBRID3 || b.type == F_HYBRID_STEREO3;
      b.use_window = false; b.all_window = false; b.win = DevWindows{}; b.win_ctas = 0; b.win_flushed = 0;
      if (win_type && !gl.empty()) {
        const int ng = (int)gl.size(), NPs = ti.npose;
        const int32_t* prow[2] = {nullptr, nullptr};
        { int c = 0; for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POSE && c < 2) prow[c++] = hidx.data() + (size_t)k*stride; }
        // window size: one 512-thread CTA holds 16 tiles of 8x4 blocks; NLOC 24 -> 12 tiles (one stripe), NLOC 40 -> 30 (two)
        int cap = NPs == 1 ? 24 : 40;
        const int nseg = std::max(1, std::min<int>(omp_get_max_threads(), ng/4096 + 1));
        const WindowPlan w = plan_windows(NPs, stride, NP, prow, gp.data(), gl.data(), ng, cap, nseg);
        int4* djobs; int4* dbat; int* dcb; int* dcv; unsigned char* dlv; unsigned char* dgw; double* dslots;
        if ((rc = upload(h, &djobs, w.jobs)) || (rc = upload(h, &dbat, w.batches)) || (rc = upload(h, &dcb, w.chunk_batch)) ||
            (rc = upload(h, &dcv, w.cvars)) || (rc = upload(h, &dlv, w.lvar)) || (rc = upload(h, &dgw, w.gwin))) return rc;
        if ((rc = dalloc(h, &dslots, (size_t)n*NPs*WIN_SLOT_DOUBLES, false))) return rc;
        b.win.n_jobs = (int)w.jobs.size(); b.win.jobs = djobs; b.win.batches = dbat; b.win.chunk_batch = dcb; b.win.cvars = dcv; b.win.lvar = dlv; b.win.grp_win = dgw; b.win.slots = dslots;
        b.use_window = true; b.all_window = w.all_window; b.win_ctas = w.win_ctas; b.win_flushed = w.win_flushed;
      }
    }
    lap("  blk groups+windows");
    b.part_off = part; part += is_nav_type(b.type) ? nav_grid(b.type, (int)n) : linearize_grid((int)n);
    b.bs_off = bs; bs += b.pose_only ? (int)((n + 127)/128) : backsub_grid(d.n_groups);
    h->jac_bytes += block_bytes(b);
  }
  lap("factor blocks");
  // ---- general landmark groups
  h->gen = GeneralGroups{};
  if (!gen_refs.empty()) {
    std::stable_sort(gen_refs.begin(), gen_refs.end(), [](const GenRef& a, const GenRef& c) { return a.rank < c.rank; });
    std::vector<int32_t> gptr, gl0, gnl; std::vector<int32_t> refs;
    for (size_t i = 0; i < gen_refs.size(); i++) {
      if (i == 0 || gen_refs[i].rank != gen_refs[i-1].rank) {
        gptr.push_back((int32_t)i);
        const int r = gorder[gen_refs[i].rank];           // root landmark id of the group
        // points of a group are contiguous in device order: count here, first device index filled in below
        gnl.push_back(gcount[r]);
        gl0.push_back(INT32_MAX);
        if (gcount[r] > 21 || r >= npt) h->supported = false;
      }
      refs.push_back(gen_refs[i].blk); refs.push_back(gen_refs[i].idx);
    }
    gptr.push_back((int32_t)gen_refs.size());
    // device index of the first point of each general group
    {
      std::vector<int32_t> rank2g(gorder.size(), -1);
      for (size_t g = 0; g + 1 < gptr.size(); g++) rank2g[gen_refs[gptr[g]].rank] = (int32_t)g;
      for (int64_t i = 0; i < nl; i++) { const int g = rank2g[grank[root[i]]]; if (g >= 0) { if (i >= npt) { h->supported = false; continue; } gl0[g] = std::min(gl0[g], L.column(DYNOBA_POINT3, i)); } }
    }
    std::vector<DevBlock> hb; for (auto& b : h->blocks) hb.push_back(b.dev);
    DevBlock* dblk; int* dgptr; int* drefs; int* dgl0; int* dgnl; int rc;
    if ((rc = upload(h, &dblk, hb)) || (rc = upload(h, &dgptr, gptr)) || (rc = upload(h, &drefs, refs)) || (rc = upload(h, &dgl0, gl0)) ||
        (rc = upload(h, &dgnl, gnl))) return rc;
    h->gen.n_groups = (int)gl0.size(); h->gen.blocks = dblk; h->gen.gptr = dgptr; h->gen.refs = drefs; h->gen.gl0 = dgl0; h->gen.gnl = dgnl;
  }
  for (auto& P : h->priors) {
    const int n = (int)P.idx.size(); std::vector<int4> slot; std::vector<int32_t> sidx;
    L.prior_table(n, P.kind.data(), P.idx.data(), slot, sidx);
    const int dim = (int)sidx.size();
    int4* dslot; int* dsidx; double *dlin, *dG, *dg, *dd, *dgc; int rc;
    if ((rc = upload(h, &dslot, slot)) || (rc = upload(h, &dsidx, sidx)) || (rc = upload(h, &dlin, P.lin)) || (rc = upload(h, &dG, P.G)) ||
        (rc = upload(h, &dg, P.g))) return rc;
    if ((rc = dalloc(h, &dd, (size_t)dim))) return rc; if ((rc = dalloc(h, &dgc, (size_t)dim))) return rc;
    P.dev = DevPrior{ n, dim, dslot, dsidx, dlin, dG, dg, P.f, dd, dgc };
    P.part_off = part; part += 1; P.bs_off = bs; bs += 1;
  }
  h->n_nav = 0; h->d_nav = nullptr;
  if (NP > np) {
    const std::vector<int2> nav = L.nav_table();
    if (int rc = upload(h, &h->d_nav, nav)) return rc;
    h->n_nav = (int)nav.size();
  }
  h->gen_bs_off = bs; bs += general_grid(h->gen.n_groups);
  h->n_lin_partials = part; h->n_bs_partials = bs + pose_norm_grid(B.n);
  h->n_partials = std::max(std::max(h->n_lin_partials, h->n_bs_partials), 1);
  { int rc; if ((rc = dalloc(h, &h->partials, (size_t)h->n_partials))) return rc; if ((rc = dalloc(h, &h->scalars, 8))) return rc; if ((rc = dalloc(h, &h->fail, 1))) return rc; }
  CK(cudaMemset(h->scalars, 0, 64)); CK(cudaMemset(h->fail, 0, 4)); CK(cudaMemset(h->partials, 0, (size_t)h->n_partials*8));
  CK(cudaDeviceSynchronize());
  lap("general groups + sync");
  h->finalized = true; h->linearized = false;
  return DYNOBA_OK;
}

// ------------------------------------------------------------------------------------------------ device steps
// fp64 peak of the device, the roofline denominator of the reduced solve: the best of plain FMAs (DFMA) and the fp64
// tensor-core shapes m8n8k4 (what the band kernel's tile updates use) and m16n8k16 (sm_90)
__global__ void fp64_rate_kernel(double* out, int iters) {
  double a[8];
#pragma unroll
  for (int k = 0; k < 8; k++) a[k] = 1.0 + 1e-3*(threadIdx.x + k);
  const double m = 1.0 - 1e-9, c = 1e-9;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = fma(a[k], m, c);
  }
  double s = 0; for (int k = 0; k < 8; k++) s += a[k];
  out[(size_t)blockIdx.x*blockDim.x + threadIdx.x] = s;
}
__global__ void fp64_dmma_k4_rate_kernel(double* out, int iters) {      // 8 independent m8n8k4 per step: 8*512 flops per warp
  const double a = 1.0 + 1e-3*(threadIdx.x & 31), b = 1.0 - 1e-9;
  double c[8][2];
#pragma unroll
  for (int k = 0; k < 8; k++) { c[k][0] = k; c[k][1] = -k; }
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 8; k++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c[k][0]), "+d"(c[k][1]) : "d"(a), "d"(b));
  }
  double s = 0; for (int k = 0; k < 8; k++) s += c[k][0] + c[k][1];
  out[(size_t)blockIdx.x*blockDim.x + threadIdx.x] = s;
}
__global__ void fp64_dmma_k16_rate_kernel(double* out, int iters) {     // 4 independent m16n8k16 per step: 4*4096 flops per warp
  const double a = 1e-3*(threadIdx.x & 31), b = 1e-3;
  double c[4][4];
#pragma unroll
  for (int k = 0; k < 4; k++) for (int j = 0; j < 4; j++) c[k][j] = k - j;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 4; k++)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %4, %4, %4, %4, %4, %4, %4}, {%5, %5, %5, %5}, "
                   "{%0, %1, %2, %3};" : "+d"(c[k][0]), "+d"(c[k][1]), "+d"(c[k][2]), "+d"(c[k][3]) : "d"(a), "d"(b));
  }
  double s = 0; for (int k = 0; k < 4; k++) for (int j = 0; j < 4; j++) s += c[k][j];
  out[(size_t)blockIdx.x*blockDim.x + threadIdx.x] = s;
}

__global__ void pack_fail_kernel(const int* fail, double* scalars) { scalars[3] = (double)(*fail); for (int i = 0; i < 4; i++) scalars[4 + i] = scalars[i]; }

static int allreduce_dev(dynoba_solver* h, double* p, size_t n) {
  if (h->world <= 1) return DYNOBA_OK;
  if (h->allreduce(h->ar_ctx, p, n, (void*)h->stream) != 0) { h->err = "all-reduce callback failed"; return DYNOBA_ERR_COMM; }
  return DYNOBA_OK;
}

// graph.error(values) on the given variable set -> scalars[slot]
static int eval_error(dynoba_solver* h, const DevVars& v, int slot) {
  for (auto& b : h->blocks) h->launches += launch_error(b.dev, v, h->partials + b.part_off, nullptr, h->stream);
  for (auto& P : h->priors) h->launches += launch_prior_eval(P.dev, v, h->partials + P.part_off, 0, h->stream);
  h->launches += launch_sum(h->partials, h->n_lin_partials, h->scalars + slot, h->stream);
  return DYNOBA_OK;
}
static int do_linearize(dynoba_solver* h) {
  // the compute-bound numeric-Jacobian blocks run on a side stream underneath the HBM-bound analytic ones
  bool side = false;
  for (auto& b : h->blocks) if (b.n && numeric_grid(b.type, (int)b.n) > 0) side = true;
  if (side) { cudaEventRecord(h->ev_fork, h->stream); cudaStreamWaitEvent(h->stream2, h->ev_fork, 0); }
  for (auto& b : h->blocks) if (numeric_grid(b.type, (int)b.n) > 0)      // compute-bound blocks first, high-priority stream
    h->launches += launch_linearize(b.dev, h->cur, h->partials + b.part_off, h->stream2);
  for (auto& b : h->blocks) if (numeric_grid(b.type, (int)b.n) == 0)
    h->launches += launch_linearize(b.dev, h->cur, h->partials + b.part_off, h->stream);
  for (auto& P : h->priors) h->launches += launch_prior_eval(P.dev, h->cur, h->partials + P.part_off, 1, h->stream);   // error(0) of the relinearised Hessian factor
  if (side) { cudaEventRecord(h->ev_join, h->stream2); cudaStreamWaitEvent(h->stream, h->ev_join, 0); }
  h->launches += launch_sum(h->partials, h->n_lin_partials, h->scalars + 0, h->stream);
  h->linearized = true;
  return DYNOBA_OK;
}
// S, g_S at the current linearization.  Multi-GPU: every rank accumulates the contribution of its landmarks into the full
// layout; the tiles of a cell are then summed at the rank that owns (factors) the cell -- a reduce per cell instead of an
// all-reduce of the whole band -- and the small right-hand-side region is all-reduced.  full_sum: all-reduce everything
// (parity hook dynoba_get_reduced_system; also the fallback when the host gave no reduce callback or there are no cells).
static int build_reduced(dynoba_solver* h, double lambda, bool full_sum = false) {
  CK(cudaMemsetAsync(h->fail, 0, 4, h->stream));
  h->launches += launch_band_clear(h->band, lambda, h->rank, (h->world > 1 && h->reduce && h->band.ncell > 0 && !full_sum) ? h->world : 1, h->stream);
  h->launches += launch_nav_inert(h->band, h->d_nav, h->n_nav, h->stream);
  for (auto& b : h->blocks) {
    if (b.pose_only) h->launches += launch_pose_factors(b.dev, h->band, h->stream);
    else {
      if (b.use_window) h->launches += launch_schur_window(b.dev, b.win, h->band, lambda, h->fail, h->stream);
      if (!b.all_window) h->launches += launch_schur_simple(b.dev, b.use_window ? b.win.grp_win : nullptr, h->band, lambda, h->fail, h->stream);
    }
  }
  h->launches += launch_schur_general(h->gen, h->band, lambda, h->fail, h->stream);
  for (auto& P : h->priors) h->launches += launch_prior_accum(P.dev, h->band, h->stream);
  if (h->world <= 1) return DYNOBA_OK;
  if (full_sum || !h->reduce || h->band.ncell == 0) return allreduce_dev(h, h->band.acc, h->band.acc_count);
  for (auto& r : h->plan.reduce_ranges)
    if (h->reduce(h->red_ctx, r.p, r.n, r.owner, (void*)h->stream) != 0) { h->err = "reduce callback failed"; return DYNOBA_ERR_COMM; }
  return allreduce_dev(h, h->plan.rhs_region, h->plan.rhs_count);
}
// factor + solve + back-substitute; scalars[1] = linearised cost decrease
static int solve_step(dynoba_solver* h, double lambda) {
  h->launches += launch_band_factor(h->plan, h->fail, h->stream);
  const bool dist = h->world > 1 && h->reduce && h->band.ncell > 0;      // cells are owned by ranks (else: replicated solve)
  if (dist && h->band.ncell >= 2) { int rc = allreduce_dev(h, h->plan.gq_base, h->plan.gq_count); if (rc) return rc; }
  h->launches += launch_band_top(h->plan, h->fail, h->stream);
  if (dist) { int rc = allreduce_dev(h, h->band.dp, (size_t)h->band.n_pad); if (rc) return rc; }
  int used = 0;
  for (auto& b : h->blocks) {
    if (b.pose_only) { h->launches += launch_pose_model(b.dev, h->band, h->partials + b.bs_off, h->stream); used = std::max(used, b.bs_off + (int)((b.n + 127)/128)); }
    else { h->launches += launch_backsub_simple(b.dev, h->band, lambda, h->dl_point, h->cur.nl_stride, h->dl_flow, h->cur.nf_stride, h->partials + b.bs_off, h->stream);
           used = std::max(used, b.bs_off + backsub_grid(b.dev.n_groups)); }
  }
  for (auto& P : h->priors) { h->launches += launch_prior_model(P.dev, h->band, h->partials + P.bs_off, h->stream); used = std::max(used, P.bs_off + 1); }
  if (h->gen.n_groups) {
    h->launches += launch_backsub_general(h->gen, h->band, lambda, h->dl_point, h->cur.nl_stride, h->partials + h->gen_bs_off, h->stream);
    used = std::max(used, h->gen_bs_off + general_grid(h->gen.n_groups));
  }
  if (h->rank == 0) { h->launches += launch_pose_delta_norm(h->band, lambda, h->partials + used, h->stream); used += pose_norm_grid(h->band.n); }
  h->launches += launch_sum(h->partials, used, h->scalars + 1, h->stream);
  return DYNOBA_OK;
}

static int check_ready(dynoba_solver* h, bool need_supported) {
  if (!h) return DYNOBA_ERR_BAD_ARG;
  int rc = finalize_impl(h); if (rc) return rc;
  cudaSetDevice(h->device);
  if (need_supported && !h->supported) { h->err = "graph has a landmark group with more than 21 chained points or a chained optical-flow variable"; return DYNOBA_ERR_UNSUPPORTED; }
  return DYNOBA_OK;
}

static int read_scalars(dynoba_solver* h, double* out4, bool reduce) {
  // the rank-local sums stay in scalars[0..3]; the all-reduce runs on a scratch copy (scalars[4..7]) so that a value
  // written once per outer iteration (scalars[0], the linearised error at delta = 0) is not summed again on every trial
  pack_fail_kernel<<<1, 1, 0, h->stream>>>(h->fail, h->scalars); h->launches++;
  if (reduce) { int rc = allreduce_dev(h, h->scalars + 4, 4); if (rc) return rc; }
  CK(cudaMemcpyAsync(out4, h->scalars + 4, 32, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DYNOBA_OK;
}

extern "C" {

int dynoba_fp64_rate(dynoba_handle h, double* tflops) {
  ARG(h && tflops, "null");
  cudaSetDevice(h->device);
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
  const int grid = sms*8, block = 256, iters = 1 << 15;
  double* d; int rc = dalloc(h, &d, (size_t)grid*block, false); if (rc) return rc;
  void (*kern[3])(double*, int) = { fp64_rate_kernel, fp64_dmma_k4_rate_kernel, fp64_dmma_k16_rate_kernel };
  const double flops_per_thread_step[3] = { 2.0*8, 8*512.0/32, 4*4096.0/32 };
  const int kiters[3] = { iters, iters/2, iters/8 };
  double peak = 0;
  for (int k = 0; k < 3; k++) {
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
      CK(cudaEventRecord(h->ev[0], h->stream));
      kern[k]<<<grid, block, 0, h->stream>>>(d, kiters[k]);
      CK(cudaEventRecord(h->ev[1], h->stream)); CK(cudaStreamSynchronize(h->stream));
      float ms; CK(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1])); if (rep && ms < best) best = ms;
    }
    peak = std::max(peak, flops_per_thread_step[k]*kiters[k]*(double)grid*block/(best*1e-3)/1e12);
  }
  *tflops = peak;
  return DYNOBA_OK;
}

int dynoba_finalize(dynoba_handle h) { if (!h) return DYNOBA_ERR_BAD_ARG; return finalize_impl(h); }

int dynoba_num_variables(dynoba_handle h, int kind, int64_t* out) {
  ARG(h && out, "null");
  ARG(valid_kind(kind), "bad variable kind");
  *out = n_vars(h, kind);
  return DYNOBA_OK;
}
int dynoba_get_keys(dynoba_handle h, int kind, int64_t n, uint64_t* out) {
  ARG(h && out, "null");
  ARG(valid_kind(kind), "bad variable kind");
  const auto& k = h->keys[kind];
  ARG((int64_t)k.size() == n, "no keys stored / size mismatch");
  std::copy(k.begin(), k.end(), out);
  return DYNOBA_OK;
}
int dynoba_problem_info(dynoba_handle h, int32_t* reduced_dim, int32_t* bandwidth, int64_t* jacobian_bytes) {
  int rc = check_ready(h, false); if (rc) return rc;
  if (reduced_dim) *reduced_dim = h->band.n; if (bandwidth) *bandwidth = h->band.bw; if (jacobian_bytes) *jacobian_bytes = h->jac_bytes;
  return DYNOBA_OK;
}

int dynoba_window_census(dynoba_handle h, int64_t* accum_ctas, int64_t* blocks_flushed) {
  int rc = check_ready(h, false); if (rc) return rc;
  for (int k = 0; k < 2; k++) { if (accum_ctas) accum_ctas[k] = 0; if (blocks_flushed) blocks_flushed[k] = 0; }
  for (const HostBlock& b : h->blocks) if (b.use_window) {
    const int k = (b.type == F_HYBRID3 || b.type == F_HYBRID_STEREO3) ? 1 : 0;
    if (accum_ctas) accum_ctas[k] += b.win_ctas;
    if (blocks_flushed) blocks_flushed[k] += b.win_flushed;
  }
  return DYNOBA_OK;
}

int dynoba_error(dynoba_handle h, double* out) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(out, "null out");
  eval_error(h, h->cur, 2);
  double s[4]; rc = read_scalars(h, s, true); if (rc) return rc;
  *out = s[2];
  return DYNOBA_OK;
}

int dynoba_linearize(dynoba_handle h, float* ms) {
  int rc = check_ready(h, false); if (rc) return rc;
  CK(cudaEventRecord(h->ev[0], h->stream));
  do_linearize(h);
  CK(cudaEventRecord(h->ev[1], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (ms) CK(cudaEventElapsedTime(ms, h->ev[0], h->ev[1]));
  CK(cudaGetLastError());
  return DYNOBA_OK;
}

int dynoba_linearize_block(dynoba_handle h, int bi, float* ms, int64_t* bytes) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(bi >= 0 && bi < (int)h->blocks.size(), "bad block index");
  auto& b = h->blocks[bi];
  CK(cudaEventRecord(h->ev[0], h->stream));
  h->launches += launch_linearize(b.dev, h->cur, h->partials + b.part_off, h->stream);
  CK(cudaEventRecord(h->ev[1], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (ms) CK(cudaEventElapsedTime(ms, h->ev[0], h->ev[1]));
  if (bytes) *bytes = block_bytes(b);
  CK(cudaGetLastError());
  return DYNOBA_OK;
}

int dynoba_get_linearization(dynoba_handle h, int bi, double* A, double* bv) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(bi >= 0 && bi < (int)h->blocks.size(), "bad block index");
  if (!h->linearized) { h->err = "call dynoba_linearize first"; return DYNOBA_ERR_STATE; }
  auto& b = h->blocks[bi]; const TypeInfo ti = type_info(b.type); const int ne = ti.dim*ti.jcols, st = b.dev.stride;
  std::vector<double> hj((size_t)ne*st), hb((size_t)ti.dim*st);
  CK(cudaMemcpy(hj.data(), b.dev.J, hj.size()*8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hb.data(), b.dev.b, hb.size()*8, cudaMemcpyDeviceToHost));
  for (int64_t s = 0; s < b.n; s++) {
    const int64_t o = b.perm[s];
    if (A) for (int e = 0; e < ne; e++) A[o*ne + e] = hj[(size_t)e*st + s];
    if (bv) for (int r = 0; r < ti.dim; r++) bv[o*ti.dim + r] = hb[(size_t)r*st + s];
  }
  return DYNOBA_OK;
}

int dynoba_get_factor_errors(dynoba_handle h, int bi, double* err) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(bi >= 0 && bi < (int)h->blocks.size() && err, "bad block index");
  auto& b = h->blocks[bi];
  double* d; rc = dalloc(h, &d, (size_t)b.dev.stride); if (rc) return rc;
  h->launches += launch_error(b.dev, h->cur, h->partials + b.part_off, d, h->stream);
  std::vector<double> he(b.dev.stride);
  CK(cudaMemcpyAsync(he.data(), d, he.size()*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int64_t s = 0; s < b.n; s++) err[b.perm[s]] = he[s];
  release(h, d);
  return DYNOBA_OK;
}

int dynoba_get_reduced_system(dynoba_handle h, double lambda, double* S, double* g) {
  int rc = check_ready(h, true); if (rc) return rc;
  if (!h->linearized) do_linearize(h);
  rc = build_reduced(h, lambda, true); if (rc) return rc;
  const DevBand& B = h->band;
  std::vector<double> hacc(B.acc_count);
  CK(cudaMemcpyAsync(hacc.data(), B.acc, hacc.size()*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  std::vector<BandProb> hch = h->plan.chains;            // host view of the same layout
  for (auto& p : hch) {
    p.tiles = hacc.data() + (p.tiles - B.acc); p.rhs = hacc.data() + (p.rhs - B.acc);
    if (p.ff) p.ff = hacc.data() + (p.ff - B.acc); if (p.gf) p.gf = hacc.data() + (p.gf - B.acc);
  }
  DevBand HB = B; HB.chains = hch.data(); HB.cells = h->plan.cells.data();
  const std::vector<int32_t> usr = h->layout.reduced_map();
  const int n = (int)h->layout.reduced_dim();
  if (S) {
    std::fill(S, S + (size_t)n*n, 0.0);
    for (int j = 0; j < B.n; j++) for (int i = j; i < B.n && i <= j + B.bw; i++) {
      if (usr[i] < 0 || usr[j] < 0) continue;
      const double v = *band_at(HB, i, j);
      S[(size_t)usr[i]*n + usr[j]] = v; S[(size_t)usr[j]*n + usr[i]] = v;
    }
  }
  if (g) for (int i = 0; i < B.n; i++) if (usr[i] >= 0) g[usr[i]] = *rhs_at(HB, i);
  return DYNOBA_OK;
}

int dynoba_solve(dynoba_handle h, double lambda, double* delta) {
  int rc = check_ready(h, true); if (rc) return rc;
  ARG(delta, "null delta");
  if (!h->linearized) do_linearize(h);
  rc = build_reduced(h, lambda); if (rc) return rc;
  rc = solve_step(h, lambda); if (rc) return rc;
  double s[4]; rc = read_scalars(h, s, true); if (rc) return rc;
  h->last_model[0] = s[0]; h->last_model[1] = s[1]; h->last_model[2] = s[3];
  CK(cudaGetLastError());
  if (s[3] != 0.0) { h->err = "reduced system not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  const VarLayout& L = h->layout;
  std::vector<double> hr(h->band.n_pad), hp(L.image_size(DYNOBA_POINT3)), hf(L.image_size(DYNOBA_FLOW2));
  CK(cudaMemcpyAsync(hr.data(), h->band.dp, hr.size()*8, cudaMemcpyDeviceToHost, h->stream));
  if (L.npt) CK(cudaMemcpyAsync(hp.data(), h->dl_point, hp.size()*8, cudaMemcpyDeviceToHost, h->stream));
  if (L.nfl) CK(cudaMemcpyAsync(hf.data(), h->dl_flow, hf.size()*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  L.walk_delta(hr.data(), hp.data(), hf.data(), [&](size_t u, double& v) { delta[u] = v; });
  return DYNOBA_OK;
}

int dynoba_retract(dynoba_handle h, const double* delta) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(delta, "null delta");
  const VarLayout& L = h->layout;
  std::vector<double> hr(h->band.n_pad, 0.0), hp(L.image_size(DYNOBA_POINT3), 0.0), hf(L.image_size(DYNOBA_FLOW2), 0.0);
  L.walk_delta(hr.data(), hp.data(), hf.data(), [&](size_t u, double& v) { v = delta[u]; });
  CK(cudaMemcpyAsync(h->band.dp, hr.data(), hr.size()*8, cudaMemcpyHostToDevice, h->stream));
  if (L.npt) CK(cudaMemcpyAsync(h->dl_point, hp.data(), hp.size()*8, cudaMemcpyHostToDevice, h->stream));
  if (L.nfl) CK(cudaMemcpyAsync(h->dl_flow, hf.data(), hf.size()*8, cudaMemcpyHostToDevice, h->stream));
  h->launches += launch_retract(h->cur, h->cand, h->band, h->dl_point, h->dl_flow, h->stream);
  h->launches += launch_nav_retract(h->cur, h->cand, h->band, h->d_nav, h->n_nav, h->stream);
  CK(cudaStreamSynchronize(h->stream));
  std::swap(h->cur, h->cand);
  h->linearized = false; cov_invalidate(h);
  return DYNOBA_OK;
}

}  // extern "C"

// Marginal information of the LAST n_keep pose-like variables (solver order) at the current values: every landmark and
// every other pose-like variable eliminated.  The band Cholesky already leaves a Schur complement in the columns it does
// not factor, so this is one plain band factorisation that stops at the tile holding the first kept variable; the few
// scalars of that tile that precede the kept block are eliminated on the host.  The one implementation behind
// dynoba_marginal and dynoba_marginal_vars; f == nullptr skips the constant (and the full solve it takes).
static int marginal_impl(dynoba_solver* h, int32_t n_keep, const int32_t* kind, const int32_t* idx, double* G, double* g, double* f) {
  const int64_t NP = h->cur.np;
  ARG(n_keep <= NP, "more variables than there are");
  if (h->world > 1) { h->err = "dynoba_marginal is a single-GPU entry point"; return DYNOBA_ERR_UNSUPPORTED; }
  std::vector<int> slot(n_keep, -1), off(n_keep + 1, 0);   // kept variable k sits at solver position NP - n_keep + slot
  for (int k = 0; k < n_keep; k++) {
    ARG(poselike_kind(kind[k]), "a kept variable must be of kind DYNOBA_POSE6, DYNOBA_VEL3 or DYNOBA_BIAS6");
    const int32_t c = h->layout.column_checked(kind[k], idx[k]);
    ARG(c >= 0, "variable out of range");
    const int p = c - (int)(NP - n_keep);
    if (p < 0) { h->err = "the kept variables must be the last ones of the elimination order (most recent frames)"; return DYNOBA_ERR_UNSUPPORTED; }
    slot[k] = p; off[k + 1] = off[k] + KINDS[kind[k]].tdim;
  }
  { std::vector<int> srt = slot; std::sort(srt.begin(), srt.end()); ARG(std::adjacent_find(srt.begin(), srt.end()) == srt.end(), "a variable is listed twice"); }
  int rc;
  if (!h->linearized) do_linearize(h);
  double lin_s[4] = {0, 0, 0, 0};
  if (f) {   // undamped solve of the whole system: scalars[0] = 1/2 sum |b_w|^2, scalars[1] = 1/2 g^T H^-1 g
    if ((rc = build_reduced(h, 0.0)) || (rc = solve_step(h, 0.0)) || (rc = read_scalars(h, lin_s, true))) return rc;
    if (lin_s[3] != 0.0) { h->err = "the reduced system is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  }
  // a second, plain layout whose factorisation stops before the kept block
  const int p0 = 6*(int)(NP - n_keep), K0 = p0/TILE;
  BandPlan mp;
  if ((rc = plain_plan_create(h, mp, K0))) return rc;
  const int NT = mp.band.NT, WBm = mp.band.WB;
  if (NT - K0 > WBm + 1) { plain_plan_release(h, mp); h->err = "the kept block is wider than the band of the reduced system"; return DYNOBA_ERR_UNSUPPORTED; }
  std::swap(h->plan, mp);                               // (h->band refers to h->plan.band)
  rc = build_reduced(h, 0.0);
  if (!rc) h->launches += launch_band_factor(h->plan, h->fail, h->stream);
  const BandProb ch = h->plan.chains[0];
  const int m = (NT - K0)*TILE, W1 = WBm + 1;
  std::vector<double> tiles((size_t)(NT - K0)*W1*TILE2), rhs((size_t)m);
  int failed = 0;
  if (!rc) {
    CK(cudaMemcpyAsync(tiles.data(), ch.tiles + (size_t)K0*W1*TILE2, tiles.size()*8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(rhs.data(), ch.rhs + (size_t)K0*TILE, rhs.size()*8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&failed, h->fail, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  std::swap(h->plan, mp);
  plain_plan_release(h, mp);
  if (rc) return rc;
  if (failed) { h->err = "the eliminated block is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  // dense symmetric copy of the trailing block: local scalar q <-> solver position K0*32 + q
  std::vector<double> M((size_t)m*m, 0.0);
  for (int j = 0; j < m; j++) for (int i = j; i < m; i++) {
    const int I = i >> 5, J = j >> 5; if (I - J > WBm) continue;
    const double v = tiles[((size_t)J*W1 + (I - J))*TILE2 + (size_t)(j & 31)*TILE + (i & 31)];
    M[(size_t)i*m + j] = v; M[(size_t)j*m + i] = v;
  }
  // eliminate the e = p0 - K0*32 scalars in front of the kept block (symmetric Gaussian elimination, e < 32)
  const int e = p0 - K0*TILE;
  for (int k = 0; k < e; k++) {
    const double piv = M[(size_t)k*m + k];
    if (!(piv > 0.0)) { h->err = "the eliminated block is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
    for (int i = k + 1; i < m; i++) {
      const double l = M[(size_t)i*m + k]/piv;
      if (l == 0.0) continue;
      for (int j = k + 1; j < m; j++) M[(size_t)i*m + j] -= l*M[(size_t)k*m + j];
      rhs[i] -= l*rhs[k];
    }
  }
  // caller's slot order and tangent layout; the inert scalars of a kept velocity are left out
  const int dim = off[n_keep];
  for (int a = 0; a < n_keep; a++) for (int r = 0; r < off[a + 1] - off[a]; r++) {
    const int qi = e + 6*slot[a] + r;
    g[off[a] + r] = rhs[qi];
    for (int b = 0; b < n_keep; b++) for (int c = 0; c < off[b + 1] - off[b]; c++) G[(size_t)(off[a] + r)*dim + off[b] + c] = M[(size_t)qi*m + e + 6*slot[b] + c];
  }
  if (f) {
    // f = sum |b_w|^2 - g_e^T H_ee^-1 g_e, and g_e^T H_ee^-1 g_e = g^T H^-1 g - g_m^T G_m^-1 g_m (block elimination of H):
    // the last term by a dense Cholesky of the kept block
    std::vector<double> L(G, G + (size_t)dim*dim), y(g, g + dim);
    for (int j = 0; j < dim; j++) {
      double d = L[(size_t)j*dim + j];
      for (int k = 0; k < j; k++) d -= L[(size_t)j*dim + k]*L[(size_t)j*dim + k];
      if (!(d > 0.0)) { h->err = "the marginal information is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
      L[(size_t)j*dim + j] = std::sqrt(d);
      for (int i = j + 1; i < dim; i++) {
        double v = L[(size_t)i*dim + j];
        for (int k = 0; k < j; k++) v -= L[(size_t)i*dim + k]*L[(size_t)j*dim + k];
        L[(size_t)i*dim + j] = v/L[(size_t)j*dim + j];
      }
    }
    double gGg = 0.0;
    for (int i = 0; i < dim; i++) {
      for (int k = 0; k < i; k++) y[i] -= L[(size_t)i*dim + k]*y[k];
      y[i] /= L[(size_t)i*dim + i]; gGg += y[i]*y[i];
    }
    *f = 2.0*lin_s[0] - (2.0*lin_s[1] - gGg);
  }
  return DYNOBA_OK;
}

extern "C" {

int dynoba_marginal(dynoba_handle h, int32_t n_keep, const int32_t* keep_pose_idx, double* G, double* g) {
  int rc = check_ready(h, true); if (rc) return rc;
  ARG(n_keep > 0 && keep_pose_idx && G && g, "bad arguments");
  if (has_nav(h)) { h->err = "dynoba_marginal is not available with velocity / bias variables"; return DYNOBA_ERR_UNSUPPORTED; }
  const std::vector<int32_t> kind(n_keep, DYNOBA_POSE6);
  return marginal_impl(h, n_keep, kind.data(), keep_pose_idx, G, g, nullptr);
}
int dynoba_marginal_vars(dynoba_handle h, int32_t n_keep, const int32_t* kind, const int32_t* idx, double* G, double* g, double* f) {
  int rc = check_ready(h, true); if (rc) return rc;
  ARG(n_keep > 0 && kind && idx && G && g, "bad arguments");
  return marginal_impl(h, n_keep, kind, idx, G, g, f);
}

// The host finds the factors of the kept points and checks them against the kept pose-like set.  The device then copies
// their linearisation out (linear_gather_kernel) and zeroes their pose columns and rhs (linear_mask_kernel), so that they
// add exactly 0 to S, g_S and g_l in the one marginal_impl call that follows.  Linearising again afterwards restores every
// Jacobian and rhs bit for bit.  The constant f of marginal_impl counts 1/2 |b|^2 from the linearize pass, which still
// holds the kept factors: their sum |b|^2 is taken off on the host.
int dynoba_marginal_keep_points(dynoba_handle h, int32_t n_keep, const int32_t* kind, const int32_t* idx, int32_t n_pts,
                                const int32_t* pt_kind, const int32_t* pt_idx, double* G, double* g, double* f,
                                int64_t capacity, int64_t* n_out, int32_t* out_type, int32_t* out_idx, double* out_Ab) {
  int rc = check_ready(h, true); if (rc) return rc;
  ARG(n_keep > 0 && kind && idx && G && g && n_out, "bad arguments");
  ARG(n_pts >= 0 && (n_pts == 0 || pt_idx), "bad kept points");
  *n_out = 0;
  if (n_pts == 0) return marginal_impl(h, n_keep, kind, idx, G, g, f);
  if (h->world > 1) { h->err = "dynoba_marginal_keep_points is a single-GPU entry point"; return DYNOBA_ERR_UNSUPPORTED; }
  const VarLayout& L = h->layout;
  std::vector<char> kept_pt(L.npt, 0), kept_pose(L.np, 0);
  for (int32_t i = 0; i < n_pts; i++) {
    ARG(!pt_kind || pt_kind[i] == DYNOBA_POINT3, "only POINT3 landmarks can be kept: a flow variable is always eliminated");
    ARG(pt_idx[i] >= 0 && pt_idx[i] < L.npt, "kept point out of range");
    ARG(!kept_pt[pt_idx[i]], "a point is listed twice"); kept_pt[pt_idx[i]] = 1;
  }
  for (int32_t k = 0; k < n_keep; k++) {
    ARG(poselike_kind(kind[k]) && L.column_checked(kind[k], idx[k]) >= 0, "a kept variable must be a pose-like variable in range");
    if (kind[k] == DYNOBA_POSE6) kept_pose[idx[k]] = 1;
  }
  // the kept points' factors, block by block in caller order
  struct Export { int bi; std::vector<int32_t> orig; };
  std::vector<Export> ex; int64_t count = 0;
  for (size_t bi = 0; bi < h->blocks.size(); bi++) {
    const HostBlock& b = h->blocks[bi]; const TypeInfo ti = type_info(b.type);
    if (ti.nlmk == 0) continue;
    std::vector<int32_t> orig;
    for (int64_t i = 0; i < b.n; i++) {
      const int32_t* ix = b.idx.data() + i*ti.arity;
      bool touches = false;
      for (int k = 0; k < ti.arity; k++) touches |= ti.cls[k] == VC_POINT && kept_pt[ix[k]];
      if (!touches) continue;
      if (ti.nlmk > 1) { h->err = "a kept point belongs to a group of more than one point (a WCME / WCPE chain)"; return DYNOBA_ERR_UNSUPPORTED; }
      if (!(b.type == F_POSE2POINT3 || b.type == F_STEREO3 || b.type == F_HYBRID3 || b.type == F_HYBRID_STEREO3 || is_linear_type(b.type))) {
        h->err = "a kept point has a factor of a type that is not kept (POSE2POINT3, STEREO3, HYBRID3, HYBRID_STEREO3, LINEAR_PP3, LINEAR_PPP3)";
        return DYNOBA_ERR_UNSUPPORTED;
      }
      for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POSE && !kept_pose[ix[k]]) {
        h->err = "a kept point has a factor on a pose that is not kept (a backtracked tracklet would couple the kept landmarks densely)";
        return DYNOBA_ERR_UNSUPPORTED;
      }
      orig.push_back((int32_t)i);
    }
    if (!orig.empty()) { count += (int64_t)orig.size(); ex.push_back({ (int)bi, std::move(orig) }); }
  }
  *n_out = count;
  ARG(capacity >= count, "capacity is smaller than the number of exported factors (*n_out)");
  ARG(count == 0 || (out_type && out_idx && out_Ab), "null output array");
  if (count == 0) return marginal_impl(h, n_keep, kind, idx, G, g, f);
  std::vector<int32_t> pos; pos.reserve(count);
  {
    int64_t k = 0;
    for (const Export& e : ex) {
      const HostBlock& b = h->blocks[e.bi]; const TypeInfo ti = type_info(b.type);
      std::vector<int32_t> sorted_of(b.n);
      for (int64_t s = 0; s < b.n; s++) sorted_of[b.perm[s]] = (int32_t)s;
      for (int32_t o : e.orig) {
        pos.push_back(sorted_of[o]);
        out_type[k] = ti.npose == 1 ? DYNOBA_LINEAR_PP3 : DYNOBA_LINEAR_PPP3;
        for (int c = 0; c < 3; c++) out_idx[3*k + c] = c < ti.arity ? b.idx[(int64_t)o*ti.arity + c] : -1;
        k++;
      }
    }
  }
  int* dpos; double* dout;
  if ((rc = upload(h, &dpos, pos))) return rc;
  if ((rc = dalloc(h, &dout, (size_t)count*3*LINEAR_EXPORT_COLS, false))) { release(h, dpos); return rc; }
  if (!h->linearized) do_linearize(h);
  {
    int64_t off = 0;
    for (const Export& e : ex) {
      h->launches += launch_linear_export(h->blocks[e.bi].dev, dpos + off, (int)e.orig.size(), dout + off*3*LINEAR_EXPORT_COLS, h->stream);
      off += (int64_t)e.orig.size();
    }
  }
  CK(cudaMemcpyAsync(out_Ab, dout, (size_t)count*3*LINEAR_EXPORT_COLS*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  release(h, dpos); release(h, dout);
  rc = marginal_impl(h, n_keep, kind, idx, G, g, f);
  do_linearize(h);                                      // the masked factors get their Jacobians and rhs back
  CK(cudaStreamSynchronize(h->stream)); CK(cudaGetLastError());
  if (rc) return rc;
  if (f) {
    double sb2 = 0.0;
    for (int64_t k = 0; k < count*3; k++) { const double bk = out_Ab[k*LINEAR_EXPORT_COLS + LINEAR_EXPORT_COLS - 1]; sb2 += bk*bk; }
    *f -= sb2;
  }
  return DYNOBA_OK;
}

}  // extern "C"

// The factor L of S, the undamped reduced system at the current values, in the covariance layout's tiles: build and
// factor (over whatever the tiles held).  The stage times are kept for the DYNOBA_TIMING lines.
static int cov_factor(dynoba_solver* h) {
  int rc;
  if (!h->linearized) do_linearize(h);
  if (!h->cov_live) {
    if ((rc = plain_plan_create(h, h->cov_plan, -1))) return rc;
    if ((rc = dalloc(h, &h->cov_stage, selinv_stage_count(h->cov_plan.band.WB), false))) { plain_plan_release(h, h->cov_plan); return rc; }
    h->cov_live = true;
  }
  h->cov_tiles = COV_NONE;
  std::swap(h->plan, h->cov_plan);                      // (h->band refers to h->plan.band)
  cudaEventRecord(h->ev[0], h->stream);
  rc = build_reduced(h, 0.0);
  cudaEventRecord(h->ev[1], h->stream);
  if (!rc) h->launches += launch_band_factor(h->plan, h->fail, h->stream);
  cudaEventRecord(h->ev[2], h->stream);
  std::swap(h->plan, h->cov_plan);
  if (rc) return rc;
  int failed = 0;
  CK(cudaMemcpyAsync(&failed, h->fail, 4, cudaMemcpyDeviceToHost, h->stream)); CK(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < 2; k++) cudaEventElapsedTime(&h->cov_ms[k], h->ev[k], h->ev[k + 1]);
  if (failed) { h->err = "the reduced system is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  h->cov_tiles = COV_FACTOR;
  return DYNOBA_OK;
}
// Sigma = S^-1 on the band, over L in place (selected inversion).  DYNOBA_TIMING=1 prints the CUDA-event times of the
// stages, build and factor from the call that factored.
static int cov_selinv(dynoba_solver* h) {
  cudaEventRecord(h->ev[2], h->stream);
  h->launches += launch_band_selinv(h->cov_plan.chains[0], h->cov_plan.band.WB, h->cov_stage, h->stream);
  cudaEventRecord(h->ev[3], h->stream);
  CK(cudaStreamSynchronize(h->stream)); CK(cudaGetLastError());
  if (getenv("DYNOBA_TIMING")) {
    float t; cudaEventElapsedTime(&t, h->ev[2], h->ev[3]);
    std::fprintf(stderr, "[dynoba covariance] reduced system %.3f ms  factor %.3f ms  selected inversion %.3f ms  (n %d, WB %d)\n",
                 h->cov_ms[0], h->cov_ms[1], t, h->cov_plan.band.n, h->cov_plan.band.WB);
  }
  h->cov_tiles = COV_SIGMA;
  return DYNOBA_OK;
}
// covariances of every point ([npt][9]) and flow ([nfl][4]) in device order, from Sigma on the band.  A landmark that no
// factor touches keeps NaN.
static int cov_landmarks(dynoba_solver* h) {
  int rc;
  const int64_t npt = h->cur.nl, nfl = h->cur.nf;
  if (!h->cov_lmk && (rc = dalloc(h, &h->cov_lmk, (size_t)9*npt + 4*nfl, false))) return rc;
  CK(cudaMemsetAsync(h->cov_lmk, 0xff, ((size_t)9*npt + 4*nfl)*8, h->stream));    // all-ones bits: NaN
  CK(cudaMemsetAsync(h->fail, 0, 4, h->stream));
  const BandProb& ch = h->cov_plan.chains[0];
  cudaEventRecord(h->ev[0], h->stream);
  for (auto& b : h->blocks) if (!b.pose_only) h->launches += launch_cov_simple(b.dev, ch.tiles, ch.TPC, h->cov_lmk, h->cov_lmk + 9*npt, h->fail, h->stream);
  h->launches += launch_cov_general(h->gen, ch.tiles, ch.TPC, h->cov_lmk, h->fail, h->stream);
  cudaEventRecord(h->ev[1], h->stream);
  int failed = 0;
  CK(cudaMemcpyAsync(&failed, h->fail, 4, cudaMemcpyDeviceToHost, h->stream)); CK(cudaStreamSynchronize(h->stream)); CK(cudaGetLastError());
  if (getenv("DYNOBA_TIMING")) { float t; cudaEventElapsedTime(&t, h->ev[0], h->ev[1]); std::fprintf(stderr, "[dynoba covariance] landmarks %.3f ms (%lld points, %lld flows)\n", t, (long long)npt, (long long)nfl); }
  if (failed) { h->err = "a landmark's information block is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  h->cov_lmk_ready = true;
  return DYNOBA_OK;
}

extern "C" {

int dynoba_marginal_covariance(dynoba_handle h, int kind, int64_t n, const int32_t* idx, double* cov) {
  int rc = check_ready(h, true); if (rc) return rc;
  if (h->world > 1) { h->err = "dynoba_marginal_covariance is a single-GPU entry point"; return DYNOBA_ERR_UNSUPPORTED; }
  ARG(valid_kind(kind), "bad variable kind");
  const VarLayout& L = h->layout;
  const int64_t nk = L.count(kind);
  ARG(idx ? n >= 0 : n == nk, "idx == NULL asks for every variable of the kind: n must be their number");
  ARG(n == 0 || cov, "null cov");
  for (int64_t i = 0; idx && i < n; i++) ARG(idx[i] >= 0 && idx[i] < nk, "variable out of range");
  if (n == 0) return DYNOBA_OK;
  if (h->cov_tiles != COV_SIGMA) {
    if (h->cov_tiles != COV_FACTOR && (rc = cov_factor(h))) return rc;
    if ((rc = cov_selinv(h))) return rc;
  }
  const bool poselike = KINDS[kind].poselike;
  if (!poselike && !h->cov_lmk_ready && (rc = cov_landmarks(h))) return rc;
  const int d = KINDS[kind].tdim;
  // caller order -> scalar position of the block (pose-like) / device landmark index
  std::vector<int32_t> at(n);
  for (int64_t i = 0; i < n; i++) at[i] = (poselike ? 6 : 1)*L.column(kind, idx ? idx[i] : i);
  int* dat; double* dout;
  if ((rc = dalloc(h, &dat, (size_t)n, false))) return rc;
  if ((rc = dalloc(h, &dout, (size_t)n*d*d, false))) { release(h, dat); return rc; }
  CK(cudaMemcpyAsync(dat, at.data(), (size_t)n*4, cudaMemcpyHostToDevice, h->stream));
  const BandProb& ch = h->cov_plan.chains[0];
  if (poselike) h->launches += launch_cov_pose_gather(ch.tiles, ch.TPC, dat, (int)n, d, dout, h->stream);
  else h->launches += launch_cov_rows_gather(h->cov_lmk + (kind == DYNOBA_FLOW2 ? 9*h->cur.nl : 0), dat, (int)n, d*d, dout, h->stream);
  CK(cudaMemcpyAsync(cov, dout, (size_t)n*d*d*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  release(h, dat); release(h, dout);
  for (int64_t e = 0; e < n*d*d; e++)
    if (std::isnan(cov[e])) { h->err = "a requested landmark is not touched by any factor"; return DYNOBA_ERR_INDETERMINATE; }
  return DYNOBA_OK;
}

}  // extern "C"

// Joint marginal covariance of n variables (DESIGN.md §4 "Joint marginal covariances").  C = the requested pose-like
// variables and every pose a factor of a requested landmark's group touches; X = S^-1 E_C by the span-restricted band
// sweeps over L; the requested landmark groups' strips from X[C, C]; the D x D result assembled here.
static int joint_impl(dynoba_solver* h, int32_t n, const int32_t* kind, const int32_t* idx, double* cov) {
  const VarLayout& L = h->layout;
  const int64_t NP = L.NP();
  // ---- requested landmark groups: points chained by a factor with several landmarks form one group
  std::vector<int32_t> uf;                              // union-find over points (empty: every point alone)
  auto root = [&](int32_t a) { if (uf.empty()) return a; while (uf[a] != a) a = uf[a] = uf[uf[a]]; return a; };
  bool any_lmk = false;
  for (int32_t i = 0; i < n; i++) any_lmk |= !KINDS[kind[i]].poselike;
  if (any_lmk)
    for (const HostBlock& b : h->blocks) {
      const TypeInfo ti = type_info(b.type);
      if (ti.nlmk < 2) continue;
      if (uf.empty()) { uf.resize(L.npt); std::iota(uf.begin(), uf.end(), 0); }
      for (int64_t o = 0; o < b.n; o++) {
        int32_t r0 = -1;
        for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POINT) {
          const int32_t r = root(b.idx[o*ti.arity + k]);
          if (r0 < 0) r0 = r; else if (r != r0) uf[r] = r0;
        }
      }
    }
  // group of every requested landmark, in order of first request; key: root point, or npt + flow index
  std::vector<int32_t> gkey_of((size_t)(L.npt + L.nfl), -1), gkey;
  struct Req { int i, g; };
  std::vector<Req> req;
  for (int32_t i = 0; i < n; i++) {
    if (KINDS[kind[i]].poselike) continue;
    const int64_t key = kind[i] == DYNOBA_POINT3 ? root(idx[i]) : L.npt + idx[i];
    if (gkey_of[key] < 0) { gkey_of[key] = (int32_t)gkey.size(); gkey.push_back((int32_t)key); }
    req.push_back({ i, gkey_of[key] });
  }
  const int ng = (int)gkey.size();
  // every factor of a requested group (block, sorted position), and the poses they touch
  std::vector<std::vector<int32_t>> grefs(ng);
  std::vector<char> in_c((size_t)NP, 0);
  for (int32_t i = 0; i < n; i++) if (KINDS[kind[i]].poselike) in_c[L.column(kind[i], idx[i])] = 1;
  for (size_t bi = 0; ng && bi < h->blocks.size(); bi++) {
    const HostBlock& b = h->blocks[bi]; const TypeInfo ti = type_info(b.type);
    if (ti.nlmk == 0) continue;
    std::vector<std::pair<int32_t, int32_t>> hit;       // (original index, group)
    for (int64_t o = 0; o < b.n; o++) {
      const int32_t* ix = b.idx.data() + o*ti.arity;
      for (int k = 0; k < ti.arity; k++) {
        if (is_poselike(ti.cls[k])) continue;
        const int32_t g = gkey_of[ti.cls[k] == VC_POINT ? root(ix[k]) : L.npt + ix[k]];
        if (g >= 0) { hit.push_back({ (int32_t)o, g }); break; }
      }
    }
    if (hit.empty()) continue;
    std::vector<int32_t> sorted_of(b.n);
    for (int64_t s = 0; s < b.n; s++) sorted_of[b.perm[s]] = (int32_t)s;
    for (const auto& e : hit) {
      grefs[e.second].push_back((int32_t)bi); grefs[e.second].push_back(sorted_of[e.first]);
      for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POSE) in_c[L.column(VC_POSE, b.idx[(int64_t)e.first*ti.arity + k])] = 1;
    }
  }
  for (int g = 0; g < ng; g++) if (grefs[g].empty()) { h->err = "a requested landmark is not touched by any factor"; return DYNOBA_ERR_INDETERMINATE; }
  // first device index and size of every group (a chain's points are contiguous in device order)
  std::vector<int4> groups(ng);
  {
    std::vector<int32_t> lo(ng, INT32_MAX), hi(ng, -1), cnt(ng, 0);
    auto add = [&](int g, int32_t d) { lo[g] = std::min(lo[g], d); hi[g] = std::max(hi[g], d); cnt[g]++; };
    if (!uf.empty()) { for (int64_t p = 0; p < L.npt; p++) { const int32_t g = gkey_of[root((int32_t)p)]; if (g >= 0) add(g, L.pt_new[p]); } }
    for (int g = 0; g < ng; g++) {
      if (gkey[g] >= L.npt) { lo[g] = L.fl_new[gkey[g] - L.npt]; cnt[g] = 0; continue; }
      if (uf.empty()) { lo[g] = hi[g] = L.pt_new[gkey[g]]; cnt[g] = 1; }
      if (3*cnt[g] > STRIP_LD || hi[g] - lo[g] + 1 != cnt[g]) { h->err = "a requested landmark belongs to a group of more than 21 chained points"; return DYNOBA_ERR_UNSUPPORTED; }
    }
    int32_t r = 0;
    for (int g = 0; g < ng; g++) { groups[g] = make_int4(r, r + (int)grefs[g].size()/2, lo[g], cnt[g]); r = groups[g].y; }
  }
  // C: ascending solver positions, the live scalars of each (a velocity's 3)
  std::vector<char> is_vel((size_t)NP, 0);
  for (int64_t i = 0; i < L.nv; i++) is_vel[L.column(DYNOBA_VEL3, i)] = 1;
  std::vector<int32_t> cmap((size_t)NP, -1), cs;
  for (int64_t p = 0; p < NP; p++) if (in_c[p]) { cmap[p] = (int32_t)cs.size(); for (int c = 0; c < (is_vel[p] ? 3 : 6); c++) cs.push_back((int32_t)(6*p + c)); }
  const int nc = (int)cs.size(), J0 = cs[0]/TILE;
  // requested landmarks grouped: rptr / rl, and each one's slot there
  std::vector<int32_t> rptr(ng + 1, 0), rl(req.size()), rslot(req.size());
  for (const Req& q : req) rptr[q.g + 1]++;
  for (int g = 0; g < ng; g++) rptr[g + 1] += rptr[g];
  {
    std::vector<int32_t> fill(rptr.begin(), rptr.end() - 1);
    for (size_t k = 0; k < req.size(); k++) {
      const int s = fill[req[k].g]++;
      rslot[k] = s; rl[s] = L.column(kind[req[k].i], idx[req[k].i]);
    }
  }
  // ---- device: L, sweeps, X[C, C], strips
  int rc;
  const bool fresh = h->cov_tiles != COV_FACTOR;        // L is built here (else an earlier call left it)
  if (fresh && (rc = cov_factor(h))) return rc;
  const BandProb& ch = h->cov_plan.chains[0];
  const size_t nreq = req.size();
  std::vector<void*> owned;
  auto done = [&](int r) { for (void* q : owned) release(h, q); return r; };
  int* dcs; double *dpanel, *dxcc;
  if ((rc = upload(h, &dcs, cs))) return rc;
  owned.push_back(dcs);
  if ((rc = dalloc(h, &dpanel, joint_panel_count(ch.NT, J0, nc), false))) return done(rc);
  owned.push_back(dpanel);
  if ((rc = dalloc(h, &dxcc, (size_t)nc*nc, false))) return done(rc);
  owned.push_back(dxcc);
  cudaEventRecord(h->ev[3], h->stream);
  h->launches += launch_band_sweeps(ch, h->cov_plan.band.WB, dcs, nc, J0, dpanel, h->stream);
  cudaEventRecord(h->ev[4], h->stream);
  h->launches += launch_joint_gather(dpanel, J0, dcs, nc, dxcc, h->stream);
  std::vector<double> xcc((size_t)nc*nc), m(nreq*nc*3), z(nreq*3*nc), vinv((size_t)ng*STRIP_LD*STRIP_LD);
  if (ng) {
    StripJob j{};
    std::vector<DevBlock> hb; for (const HostBlock& b : h->blocks) hb.push_back(b.dev);
    std::vector<int32_t> refs; for (const auto& r : grefs) refs.insert(refs.end(), r.begin(), r.end());
    DevBlock* dblk; int32_t *drefs, *drptr, *drl, *dcmap; int4* dgroups; double *dm, *dz, *dvinv;
    if ((rc = upload(h, &dblk, hb))) return done(rc);
    owned.push_back(dblk);
    if ((rc = upload(h, &drefs, refs))) return done(rc);
    owned.push_back(drefs);
    if ((rc = upload(h, &dgroups, groups))) return done(rc);
    owned.push_back(dgroups);
    if ((rc = upload(h, &drptr, rptr))) return done(rc);
    owned.push_back(drptr);
    if ((rc = upload(h, &drl, rl))) return done(rc);
    owned.push_back(drl);
    if ((rc = upload(h, &dcmap, cmap))) return done(rc);
    owned.push_back(dcmap);
    if ((rc = dalloc(h, &dm, m.size()))) return done(rc);        // zeroed: the strips add into it
    owned.push_back(dm);
    if ((rc = dalloc(h, &dz, z.size(), false))) return done(rc);
    owned.push_back(dz);
    if ((rc = dalloc(h, &dvinv, vinv.size(), false))) return done(rc);
    owned.push_back(dvinv);
    j.blocks = dblk; j.refs = drefs; j.groups = dgroups; j.rptr = drptr; j.rl = drl; j.cmap = dcmap; j.xcc = dxcc; j.nc = nc;
    j.m = dm; j.z = dz; j.vinv = dvinv; j.ng = ng; j.fail = h->fail;
    if (cudaMemsetAsync(h->fail, 0, 4, h->stream) != cudaSuccess) return done(DYNOBA_ERR_CUDA);
    h->launches += launch_cov_strips(j, h->stream);
    cudaEventRecord(h->ev[5], h->stream);
    cudaMemcpyAsync(m.data(), dm, m.size()*8, cudaMemcpyDeviceToHost, h->stream);
    cudaMemcpyAsync(z.data(), dz, z.size()*8, cudaMemcpyDeviceToHost, h->stream);
    cudaMemcpyAsync(vinv.data(), dvinv, vinv.size()*8, cudaMemcpyDeviceToHost, h->stream);
  } else {
    cudaEventRecord(h->ev[5], h->stream);
  }
  int failed = 0;
  cudaMemcpyAsync(xcc.data(), dxcc, xcc.size()*8, cudaMemcpyDeviceToHost, h->stream);
  if (ng) cudaMemcpyAsync(&failed, h->fail, 4, cudaMemcpyDeviceToHost, h->stream);
  const cudaError_t e = cudaStreamSynchronize(h->stream);
  rc = done(DYNOBA_OK);
  if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) { h->err = std::string("joint covariance: ") + cudaGetErrorString(e); return DYNOBA_ERR_CUDA; }
  if (getenv("DYNOBA_TIMING")) {
    float t[2]; cudaEventElapsedTime(&t[0], h->ev[3], h->ev[4]); cudaEventElapsedTime(&t[1], h->ev[4], h->ev[5]);
    std::fprintf(stderr, "[dynoba joint covariance] reduced system %.3f ms  factor %.3f ms%s  sweeps %.3f ms  strips %.3f ms  (span %d tiles, |C| %d, %d landmark groups, n %d, WB %d)\n",
                 h->cov_ms[0], h->cov_ms[1], fresh ? "" : " (earlier call)", t[0], t[1], ch.NT - J0, nc, ng, h->cov_plan.band.n, h->cov_plan.band.WB);
  }
  if (failed) { h->err = "a requested landmark's information block is not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  // ---- assembly: scalar a of the result = (variable, tangent index); the lower triangle, mirrored
  std::vector<int32_t> var_of, sub_of, slot_of(n, -1);
  for (size_t k = 0; k < req.size(); k++) slot_of[req[k].i] = rslot[k];
  std::vector<int32_t> grp_of(n, -1);
  for (const Req& q : req) grp_of[q.i] = q.g;
  for (int32_t i = 0; i < n; i++) for (int c = 0; c < KINDS[kind[i]].tdim; c++) { var_of.push_back(i); sub_of.push_back(c); }
  const int64_t D = (int64_t)var_of.size();
  auto cidx = [&](int32_t i, int c) { return (size_t)cmap[L.column(kind[i], idx[i])] + c; };
  auto loff = [&](int32_t i) { const int g = grp_of[i]; return (groups[g].w ? 3 : 2)*(L.column(kind[i], idx[i]) - groups[g].z); };
  for (int64_t a = 0; a < D; a++) for (int64_t b = 0; b <= a; b++) {
    const int32_t i = var_of[a], k = var_of[b]; const int r = sub_of[a], c = sub_of[b];
    const bool pi = KINDS[kind[i]].poselike, pk = KINDS[kind[k]].poselike;
    double v;
    if (pi && pk) v = xcc[cidx(i, r)*nc + cidx(k, c)];
    else if (!pi && pk) v = z[((size_t)slot_of[i]*3 + r)*nc + cidx(k, c)];
    else if (pi && !pk) v = z[((size_t)slot_of[k]*3 + c)*nc + cidx(i, r)];
    else {
      v = grp_of[i] == grp_of[k] ? vinv[(size_t)grp_of[i]*STRIP_LD*STRIP_LD + (size_t)(loff(i) + r)*STRIP_LD + loff(k) + c] : 0.0;
      const double* zi = z.data() + ((size_t)slot_of[i]*3 + r)*nc; const double* mk = m.data() + (size_t)slot_of[k]*nc*3 + c;
      for (int q = 0; q < nc; q++) v -= zi[q]*mk[(size_t)q*3];
    }
    cov[a*D + b] = v; cov[b*D + a] = v;
  }
  return rc;
}

extern "C" {

int dynoba_joint_marginal_covariance(dynoba_handle h, int32_t n, const int32_t* kind, const int32_t* idx, double* cov) {
  int rc = check_ready(h, true); if (rc) return rc;
  if (h->world > 1) { h->err = "dynoba_joint_marginal_covariance is a single-GPU entry point"; return DYNOBA_ERR_UNSUPPORTED; }
  ARG(n > 0, "n must be positive"); ARG(kind && idx, "null kind or idx"); ARG(cov, "null cov");
  std::vector<std::pair<int32_t, int32_t>> seen(n);
  for (int32_t i = 0; i < n; i++) {
    ARG(valid_kind(kind[i]), "bad variable kind");
    ARG(h->layout.column_checked(kind[i], idx[i]) >= 0, "variable out of range");
    seen[i] = { kind[i], idx[i] };
  }
  std::sort(seen.begin(), seen.end());
  ARG(std::adjacent_find(seen.begin(), seen.end()) == seen.end(), "a variable is listed twice");
  return joint_impl(h, n, kind, idx, cov);
}

int dynoba_get_variables(dynoba_handle h, int kind, int64_t n, double* out) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(out, "null out"); ARG(valid_kind(kind), "bad kind");
  const VarLayout& L = h->layout;
  ARG(n == L.count(kind), "size mismatch");
  std::vector<double> img(L.image_size(kind));
  CK(cudaMemcpyAsync(img.data(), image_of(h->cur, kind), img.size()*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  L.gather_values(kind, img.data(), out);
  return DYNOBA_OK;
}

// LevenbergMarquardtOptimizer::optimize()  [GTSAM-ext nonlinear/{NonlinearOptimizer,LevenbergMarquardtOptimizer}.cpp]
int dynoba_optimize(dynoba_handle h, const dynoba_lm_params* prm, dynoba_lm_stats* st) {
  if (!h) return DYNOBA_ERR_BAD_ARG;
  dynoba_lm_params P; if (prm) P = *prm; else dynoba_lm_default_params(&P);
  h->lm_trace.clear();
  if (!lm_params_usable(P)) { h->err = "LM parameters under which the LM loop need not end (see dynoba_lm_params)"; return DYNOBA_ERR_BAD_ARG; }
  int rc = check_ready(h, true); if (rc) return rc;
  dynoba_lm_stats S; std::memset(&S, 0, sizeof(S));
  const int64_t launches0 = h->launches;
  cudaEvent_t* ev = h->ev;
  float ms;
  auto tick = [&](int i) { cudaEventRecord(ev[i], h->stream); };
  auto tock = [&](int a, int b, double& acc) { cudaEventElapsedTime(&ms, ev[a], ev[b]); acc += ms; };
  double sc[4];
  tick(6);
  tick(0); eval_error(h, h->cur, 2); tick(1);
  rc = read_scalars(h, sc, true); if (rc) return rc;
  tock(0, 1, S.ms_error);
  double err = sc[2], lambda = P.lambda_initial;
  S.error_initial = err; S.reduced_dim = h->band.n; S.bandwidth = h->band.bw;
  int iterations = 0, inner = 0;
  if (lm_starts(err, P)) {
    double newError = err, currentError;
    do {
      currentError = newError;
      tick(0); do_linearize(h); tick(1);
      for (;;) {   // tryLambda
        tick(2); rc = build_reduced(h, lambda); if (rc) return rc;
        tick(3); rc = solve_step(h, lambda); if (rc) return rc;
        tick(4);
        h->launches += launch_retract(h->cur, h->cand, h->band, h->dl_point, h->dl_flow, h->stream);
        h->launches += launch_nav_retract(h->cur, h->cand, h->band, h->d_nav, h->n_nav, h->stream);
        eval_error(h, h->cand, 2);
        tick(5);
        rc = read_scalars(h, sc, true); if (rc) return rc;
        if (iterations + inner >= 0) { tock(2, 3, S.ms_schur); tock(3, 4, S.ms_factor); tock(4, 5, S.ms_error); }
        const bool solved = sc[3] == 0.0;
        const double oldLin = sc[0], lin = sc[1], nerr = sc[2];
        const LmDecision d = lm_decide(solved, oldLin, lin, err, nerr, P);
        h->last_model[0] = oldLin; h->last_model[1] = lin; h->last_model[2] = sc[3];
        const double row[LM_TRACE_COLS] = {(double)iterations, (double)inner, lambda, oldLin, lin, err, nerr, (double)solved, (double)d.success, (double)d.stop};
        h->lm_trace.insert(h->lm_trace.end(), row, row + LM_TRACE_COLS);
        if (P.verbosity > 0) {
          if (solved && std::isfinite(lin)) std::fprintf(stderr, "[dynoba-lm] it %d inner %d lambda %.3e err %.12e -> %.12e lin %.6e %s\n", iterations, inner, lambda, err, nerr, lin, d.success ? "ok" : "rej");
          else std::fprintf(stderr, "[dynoba-lm] it %d inner %d lambda %.3e solve failed (flag %.0f)\n", iterations, inner, lambda, sc[3]);
        }
        if (d.success) { std::swap(h->cur, h->cand); h->linearized = false; }
        if (lm_update(d, nerr, P, lambda, err, iterations, inner)) break;
      }
      { float m2; cudaEventElapsedTime(&m2, ev[0], ev[1]); S.ms_linearize += m2; }
      newError = err;
    } while (lm_continues(iterations, currentError, newError, P));
  }
  tick(7); cudaEventSynchronize(ev[7]); cudaEventElapsedTime(&ms, ev[6], ev[7]); S.ms_total = ms;
  S.iterations = iterations; S.inner_iterations = inner; S.error_final = err; S.lambda_final = lambda;
  S.kernel_launches = h->launches - launches0;
  if (st) *st = S;
  if (iterations) cov_invalidate(h);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return DYNOBA_ERR_CUDA; }
  return DYNOBA_OK;
}

int dynoba_last_model(dynoba_handle h, double out[3]) {
  ARG(h && out, "null argument");
  for (int i = 0; i < 3; i++) out[i] = h->last_model[i];
  return DYNOBA_OK;
}

int dynoba_get_lm_trace(dynoba_handle h, int64_t capacity, double* rows, int64_t* n) {
  ARG(h && n && capacity >= 0 && (rows || capacity == 0), "null argument");
  const int64_t have = (int64_t)h->lm_trace.size()/LM_TRACE_COLS;
  std::copy(h->lm_trace.begin(), h->lm_trace.begin() + std::min(have, capacity)*LM_TRACE_COLS, rows);
  *n = have;
  return DYNOBA_OK;
}

}  // extern "C"
