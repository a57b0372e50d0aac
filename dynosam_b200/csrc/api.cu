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
#include <memory>
#include <numeric>
#include <string>
#include <vector>
#include <map>

#include "../../include/dynoba.h"
#include "internal.cuh"

using namespace dynoba;

namespace {

// std::vector without the serial value-initialisation pass (the elements are written in parallel right after resize)
template <class T> struct NoInitAlloc : std::allocator<T> {
  template <class U> struct rebind { using other = NoInitAlloc<U>; };
  template <class U, class... A> void construct(U* p, A&&... a) {
    if constexpr (sizeof...(A) == 0) ::new ((void*)p) U; else ::new ((void*)p) U(std::forward<A>(a)...);
  }
};

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
};

struct HostPrior {      // gtsam::LinearContainerFactor(HessianFactor) over pose-like variables
  std::vector<int32_t> idx; std::vector<double> lin, G, g; double f = 0;
  DevPrior dev{}; int part_off = 0, bs_off = 0;
};

}  // namespace

struct dynoba_solver {
  int device = 0; cudaStream_t stream = nullptr; cudaStream_t stream2 = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr; std::string err;
  std::vector<double> pose, point, flow, aux; std::vector<uint64_t> kpose, kpoint, kflow;
  double calib[6] = { 721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372 };
  std::vector<int32_t> hint;
  // navigation variables (DYNOBA_VEL3 / DYNOBA_BIAS6): pose-like, solver positions pos[np + i] / pos[np + nv + i]
  std::vector<double> vel, bias; std::vector<uint64_t> kvel, kbias; std::vector<int32_t> vhint, bhint;
  int2* d_nav = nullptr; int n_nav = 0;   // device (position, dimension) of every velocity and bias
  std::vector<HostBlock> blocks;
  std::vector<HostPrior> priors;
  bool finalized = false, linearized = false, supported = true;
  std::vector<int32_t> pos, pt_new, fl_new;
  DevVars cur{}, cand{}; BandPlan plan{}; DevBand& band = plan.band; int ncell_request = 0;
  double *dl_point = nullptr, *dl_flow = nullptr, *partials = nullptr, *scalars = nullptr;
  int* fail = nullptr; int n_partials = 0, n_lin_partials = 0, n_bs_partials = 0;
  int rank = 0, world = 1; dynoba_allreduce_fn allreduce = nullptr; void* ar_ctx = nullptr; int min_bw = 0;
  dynoba_reduce_fn reduce = nullptr; void* red_ctx = nullptr;
  int64_t launches = 0; int64_t jac_bytes = 0;
  GeneralGroups gen{}; int gen_bs_off = 0;
  std::vector<std::pair<void*, size_t>> allocs;   // device allocations (pointer, bytes)
  cudaEvent_t ev[8]{};
};

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return DYNOBA_ERR_CUDA; } } while (0)
#define ARG(cond, msg) do { if (!(cond)) { if (h) h->err = msg; return DYNOBA_ERR_BAD_ARG; } } while (0)

static int pad32(int64_t n) { return (int)((n + 31)/32*32); }

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
static void free_device(dynoba_solver* h) {
  if (!h->allocs.empty()) cudaDeviceSynchronize();      // cudaFree used to imply this; cached blocks must be idle too
  for (auto& a : h->allocs) g_devcache.give(h->device, a.first, a.second);
  h->allocs.clear();
  h->finalized = false; h->linearized = false;
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

static std::vector<double>* var_store(dynoba_solver* h, int kind) {
  switch (kind) {
    case DYNOBA_POSE6: return &h->pose; case DYNOBA_POINT3: return &h->point; case DYNOBA_FLOW2: return &h->flow;
    case DYNOBA_VEL3: return &h->vel; case DYNOBA_BIAS6: return &h->bias; default: return nullptr;
  }
}
static std::vector<uint64_t>* key_store(dynoba_solver* h, int kind) {
  switch (kind) {
    case DYNOBA_POSE6: return &h->kpose; case DYNOBA_POINT3: return &h->kpoint; case DYNOBA_FLOW2: return &h->kflow;
    case DYNOBA_VEL3: return &h->kvel; case DYNOBA_BIAS6: return &h->kbias; default: return nullptr;
  }
}
static int kind_width(int kind) { return kind == DYNOBA_POSE6 ? 12 : (kind == DYNOBA_POINT3 || kind == DYNOBA_VEL3 ? 3 : (kind == DYNOBA_BIAS6 ? 6 : 2)); }
static bool has_nav(const dynoba_solver* h) { return !h->vel.empty() || !h->bias.empty(); }

int dynoba_set_variables(dynoba_handle h, int kind, int64_t n, const uint64_t* keys, const double* data) {
  ARG(h, "null handle"); ARG(n >= 0 && (n == 0 || data), "null data");
  const int w = kind_width(kind);
  std::vector<double>* dst = var_store(h, kind);
  std::vector<uint64_t>* kd = key_store(h, kind);
  ARG(dst, "bad variable kind");
  const bool same_shape = dst->size() == (size_t)n*w;
  dst->assign(data, data + (size_t)n*w);
  if (keys) kd->assign(keys, keys + n); else if (!same_shape) kd->clear();   // a value refresh keeps the keys
  if (h->finalized && same_shape && (has_nav(h) || kind == DYNOBA_VEL3 || kind == DYNOBA_BIAS6)) {
    // pose-like values of a visual-inertial graph: the pose SoA holds poses, velocities and biases, so only the rows of
    // the refreshed kind are replaced in the current device image
    const int64_t np = (int64_t)h->pose.size()/12, nv = (int64_t)h->vel.size()/3;
    const int64_t base = kind == DYNOBA_POSE6 ? 0 : (kind == DYNOBA_VEL3 ? np : np + nv);
    const int st = h->cur.np_stride;
    if (kind == DYNOBA_POSE6 || kind == DYNOBA_VEL3 || kind == DYNOBA_BIAS6) {
      if (n == 0) return DYNOBA_OK;
      cudaSetDevice(h->device);
      std::vector<double> soa((size_t)12*st);
      CK(cudaMemcpy(soa.data(), h->cur.pose, soa.size()*8, cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < n; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*st + h->pos[base + i]] = k < w ? data[i*w + k] : 0.0;
      CK(cudaMemcpy(h->cur.pose, soa.data(), soa.size()*8, cudaMemcpyHostToDevice));
      h->linearized = false;
      return DYNOBA_OK;
    }
  }
  if (h->finalized && same_shape) {
    // refresh device values only (layout unchanged)
    cudaSetDevice(h->device);
    std::vector<double> soa;
    if (kind == DYNOBA_POSE6) {
      soa.assign((size_t)12*h->cur.np_stride, 0.0);
      for (int64_t i = 0; i < n; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*h->cur.np_stride + h->pos[i]] = data[i*12 + k];
      for (int p = (int)n; p < h->cur.np_stride; p++) { soa[(size_t)0*h->cur.np_stride + p] = soa[(size_t)4*h->cur.np_stride + p] = soa[(size_t)8*h->cur.np_stride + p] = 1.0; }
      CK(cudaMemcpyAsync(h->cur.pose, soa.data(), soa.size()*8, cudaMemcpyHostToDevice, h->stream));
    } else if (kind == DYNOBA_POINT3) {
      soa.assign((size_t)3*h->cur.nl_stride, 0.0);
      for (int64_t i = 0; i < n; i++) for (int k = 0; k < 3; k++) soa[(size_t)k*h->cur.nl_stride + h->pt_new[i]] = data[i*3 + k];
      CK(cudaMemcpyAsync(h->cur.point, soa.data(), soa.size()*8, cudaMemcpyHostToDevice, h->stream));
    } else {
      soa.assign((size_t)2*h->cur.nf_stride, 0.0);
      for (int64_t i = 0; i < n; i++) for (int k = 0; k < 2; k++) soa[(size_t)k*h->cur.nf_stride + h->fl_new[i]] = data[i*2 + k];
      CK(cudaMemcpyAsync(h->cur.flow, soa.data(), soa.size()*8, cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaStreamSynchronize(h->stream));
    h->linearized = false;
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
  h->linearized = false;
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
  if (imu) for (size_t i = 0; i < b.meas.size(); i++) ARG(std::isfinite(b.meas[i]), "IMU measurement must be finite");
  b.robust_k = robust_k;
  if (aux_idx) { par_assign(b.aux, aux_idx, (size_t)n); b.has_aux = true; }
  h->blocks.push_back(std::move(b));
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

int dynoba_add_linear_prior(dynoba_handle h, int32_t n, const int32_t* pose_idx, const double* lin_poses, const double* G, const double* g, double f) {
  ARG(h, "null handle"); ARG(n > 0 && n <= 512 && pose_idx && lin_poses && G && g, "bad prior");
  if (has_nav(h)) { h->err = "dynoba_add_linear_prior is not available with velocity / bias variables"; return DYNOBA_ERR_UNSUPPORTED; }
  HostPrior P; P.idx.assign(pose_idx, pose_idx + n); P.lin.assign(lin_poses, lin_poses + (size_t)12*n);
  P.G.assign(G, G + (size_t)36*n*n); P.g.assign(g, g + (size_t)6*n); P.f = f;
  { std::vector<int32_t> srt = P.idx; std::sort(srt.begin(), srt.end()); ARG(std::adjacent_find(srt.begin(), srt.end()) == srt.end(), "a prior lists a variable twice"); }
  for (int r = 0; r < 6*n; r++) for (int c = 0; c < r; c++)
    ARG(std::fabs(P.G[(size_t)r*6*n + c] - P.G[(size_t)c*6*n + r]) <= 1e-9*(std::fabs(P.G[(size_t)r*6*n + r]) + std::fabs(P.G[(size_t)c*6*n + c]) + 1e-300), "prior information matrix is not symmetric");
  h->priors.push_back(std::move(P));
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

int dynoba_set_pose_order(dynoba_handle h, int64_t n, const int32_t* rank) {
  ARG(h, "null handle"); ARG(n >= 0 && (n == 0 || rank), "null rank");
  h->hint.assign(rank, rank + n);
  if (h->finalized) free_device(h);
  return DYNOBA_OK;
}

int dynoba_set_variable_order(dynoba_handle h, int kind, int64_t n, const int32_t* rank) {
  ARG(h, "null handle"); ARG(kind == DYNOBA_VEL3 || kind == DYNOBA_BIAS6, "variable order hints are for DYNOBA_VEL3 / DYNOBA_BIAS6 (poses: dynoba_set_pose_order)");
  ARG(n >= 0 && (n == 0 || rank), "null rank");
  (kind == DYNOBA_VEL3 ? h->vhint : h->bhint).assign(rank, rank + n);
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
static int uf_find(std::vector<int32_t>& p, int x) { while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; } return x; }

static int finalize_impl(dynoba_solver* h) {
  if (h->finalized) return DYNOBA_OK;
  cudaSetDevice(h->device);
  // host-side symbolic phase runs on up to 32 threads regardless of OMP_NUM_THREADS (torchrun pins it to 1)
  struct OmpScope { int saved; OmpScope() : saved(omp_get_max_threads()) { int t = std::min(omp_get_num_procs(), 32); if (const char* e = getenv("DYNOBA_THREADS")) t = std::max(1, atoi(e)); omp_set_num_threads(t); } ~OmpScope() { omp_set_num_threads(saved); } } omp_scope;
  const bool timing = getenv("DYNOBA_TIMING") != nullptr;
  auto t_last = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) { if (!timing) return; auto t = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[dynoba finalize] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(t - t_last).count()); t_last = t; };
  const int64_t np = (int64_t)h->pose.size()/12, npt = (int64_t)h->point.size()/3, nfl = (int64_t)h->flow.size()/2, naux = (int64_t)h->aux.size()/12;
  const int64_t nv = (int64_t)h->vel.size()/3, nb = (int64_t)h->bias.size()/6, NP = np + nv + nb;   // NP: pose-like variables
  ARG(h->hint.empty() || (int64_t)h->hint.size() == np, "pose order hint length != number of poses");
  ARG(h->vhint.empty() || (int64_t)h->vhint.size() == nv, "velocity order hint length != number of velocities");
  ARG(h->bhint.empty() || (int64_t)h->bhint.size() == nb, "bias order hint length != number of biases");
  if (NP > np && (!h->priors.empty() || h->world > 1 || h->reduce)) {
    h->err = "velocity / bias variables cannot be combined with dynoba_add_linear_prior, dynoba_set_shard or dynoba_set_reduce";
    return DYNOBA_ERR_UNSUPPORTED;
  }
  // pose-like index of a key slot: poses [0, np), velocities [np, np + nv), biases [np + nv, NP)
  auto plx = [&](int cls, int32_t ix) -> int64_t { return cls == VC_POSE ? ix : (cls == VC_VEL ? np + ix : np + nv + ix); };
  // ---- validate indices
  for (auto& b : h->blocks) {
    const TypeInfo ti = type_info(b.type);
    int bad = 0;
#pragma omp parallel for schedule(static) reduction(|:bad)
    for (int64_t i = 0; i < b.n; i++) {
      for (int k = 0; k < ti.arity; k++) {
        const int32_t ix = b.idx[i*ti.arity + k];
        const int c = ti.cls[k];
        const int64_t lim = c == VC_POSE ? np : (c == VC_POINT ? npt : (c == VC_FLOW ? nfl : (c == VC_VEL ? nv : nb)));
        if (!(ix >= 0 && ix < lim)) bad |= 1;
      }
      if (b.has_aux && !(b.aux[i] >= 0 && b.aux[i] < naux)) bad |= 2;
    }
    ARG(!(bad & 1), "factor index out of range"); ARG(!(bad & 2), "aux index out of range");
  }
  lap("validate");
  // ---- pose ordering
  h->pos.resize(NP);
  if (NP == np) {
    std::vector<int32_t> ord(np); std::iota(ord.begin(), ord.end(), 0);
    if (!h->hint.empty()) std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return h->hint[a] < h->hint[b]; });
    for (int64_t i = 0; i < np; i++) h->pos[ord[i]] = (int32_t)i;
  } else {
    // visual-inertial graph: ordered by (rank, kind: pose < velocity < bias, index); a kind without a hint ranks by index,
    // so X_k, V_k, b_k with the frame as rank sit next to each other and the system stays banded
    std::vector<int32_t> ord(NP), rk(NP);
    std::iota(ord.begin(), ord.end(), 0);
    for (int64_t i = 0; i < np; i++) rk[i] = h->hint.empty() ? (int32_t)i : h->hint[i];
    for (int64_t i = 0; i < nv; i++) rk[np + i] = h->vhint.empty() ? (int32_t)i : h->vhint[i];
    for (int64_t i = 0; i < nb; i++) rk[np + nv + i] = h->bhint.empty() ? (int32_t)i : h->bhint[i];
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return rk[a] < rk[b]; });
    for (int64_t i = 0; i < NP; i++) h->pos[ord[i]] = (int32_t)i;
  }
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
      for (int k = 0; k < ti.arity; k++) if (is_poselike(ti.cls[k])) { const int p = h->pos[plx(ti.cls[k], b.idx[i*ti.arity + k])]; lo = std::min(lo, p); hi = std::max(hi, p); }
      blo = std::min(blo, lo); bhi = std::max(bhi, hi);
      if (lslot < 0) { bspread = std::max(bspread, hi - lo); continue; }
      const int g = root[lmk_id(ti.cls[lslot], b.idx[i*ti.arity + lslot])];
      int32_t cur = __atomic_load_n(&gmin[g], __ATOMIC_RELAXED);
      while (lo < cur && !__atomic_compare_exchange_n(&gmin[g], &cur, lo, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
      cur = __atomic_load_n(&gmax[g], __ATOMIC_RELAXED);
      while (hi > cur && !__atomic_compare_exchange_n(&gmax[g], &cur, hi, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
      if (ti.npose >= 2) {   // secondary ordering key: user index of the last pose slot (object-major for DynOSAM's H keys)
        int last = -1; for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POSE) last = b.idx[i*ti.arity + k];
        cur = __atomic_load_n(&gsec[g], __ATOMIC_RELAXED);
        while (last < cur && !__atomic_compare_exchange_n(&gsec[g], &cur, last, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
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
    for (int32_t ix : P.idx) { ARG(ix >= 0 && ix < np, "prior variable out of range"); lo = std::min(lo, h->pos[ix]); hi = std::max(hi, h->pos[ix]); }
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
  // landmark device indices
  h->pt_new.assign(npt, 0); h->fl_new.assign(nfl, 0);
  {
    std::vector<int32_t> ord(npt); std::iota(ord.begin(), ord.end(), 0);
    int unsorted = 0;
#pragma omp parallel for schedule(static) reduction(|:unsorted)
    for (int64_t i = 1; i < npt; i++) unsorted |= grank[root[i-1]] > grank[root[i]];
    if (unsorted) __gnu_parallel::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return grank[root[a]] < grank[root[b]]; });
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < npt; i++) h->pt_new[ord[i]] = (int32_t)i;
    std::vector<int32_t> of(nfl); std::iota(of.begin(), of.end(), 0);
    std::stable_sort(of.begin(), of.end(), [&](int a, int b) { return grank[root[npt + a]] < grank[root[npt + b]]; });
    for (int64_t i = 0; i < nfl; i++) h->fl_new[of[i]] = (int32_t)i;
  }
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
  V.np = (int)NP; V.np_stride = pad32(NP); V.nl = (int)npt; V.nl_stride = pad32(npt); V.nf = (int)nfl; V.nf_stride = pad32(nfl);
  V.naux = (int)naux; V.naux_stride = pad32(naux);
  for (int i = 0; i < 6; i++) V.K[i] = h->calib[i];
  h->cand = V;
  {
    std::vector<double> soa((size_t)12*V.np_stride, 0.0);
    for (int p = 0; p < V.np_stride; p++) soa[(size_t)0*V.np_stride + p] = soa[(size_t)4*V.np_stride + p] = soa[(size_t)8*V.np_stride + p] = 1.0;
    for (int64_t i = 0; i < np; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*V.np_stride + h->pos[i]] = h->pose[i*12 + k];
    for (int64_t i = 0; i < nv; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*V.np_stride + h->pos[np + i]] = k < 3 ? h->vel[i*3 + k] : 0.0;
    for (int64_t i = 0; i < nb; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*V.np_stride + h->pos[np + nv + i]] = k < 6 ? h->bias[i*6 + k] : 0.0;
    int rc = dalloc(h, &h->cur.pose, soa.size()); if (rc) return rc; rc = dalloc(h, &h->cand.pose, soa.size()); if (rc) return rc;
    CK(cudaMemcpy(h->cur.pose, soa.data(), soa.size()*8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->cand.pose, soa.data(), soa.size()*8, cudaMemcpyHostToDevice));
    soa.assign((size_t)3*V.nl_stride, 0.0);
    for (int64_t i = 0; i < npt; i++) for (int k = 0; k < 3; k++) soa[(size_t)k*V.nl_stride + h->pt_new[i]] = h->point[i*3 + k];
    rc = dalloc(h, &h->cur.point, soa.size()); if (rc) return rc; rc = dalloc(h, &h->cand.point, soa.size()); if (rc) return rc;
    rc = dalloc(h, &h->dl_point, soa.size()); if (rc) return rc;
    CK(cudaMemcpy(h->cur.point, soa.data(), soa.size()*8, cudaMemcpyHostToDevice));
    CK(cudaMemset(h->dl_point, 0, std::max<size_t>(soa.size(), 1)*8));
    soa.assign((size_t)2*V.nf_stride, 0.0);
    for (int64_t i = 0; i < nfl; i++) for (int k = 0; k < 2; k++) soa[(size_t)k*V.nf_stride + h->fl_new[i]] = h->flow[i*2 + k];
    rc = dalloc(h, &h->cur.flow, soa.size()); if (rc) return rc; rc = dalloc(h, &h->cand.flow, soa.size()); if (rc) return rc;
    rc = dalloc(h, &h->dl_flow, soa.size()); if (rc) return rc;
    CK(cudaMemcpy(h->cur.flow, soa.data(), soa.size()*8, cudaMemcpyHostToDevice));
    CK(cudaMemset(h->dl_flow, 0, std::max<size_t>(soa.size(), 1)*8));
    soa.assign((size_t)12*V.naux_stride, 0.0);
    for (int64_t i = 0; i < naux; i++) for (int k = 0; k < 12; k++) soa[(size_t)k*V.naux_stride + i] = h->aux[i*12 + k];
    double* da; rc = dalloc(h, &da, soa.size()); if (rc) return rc;
    CK(cudaMemcpy(da, soa.data(), soa.size()*8, cudaMemcpyHostToDevice));
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
        key[i] = ((int64_t)frank[i] << 32) | (uint32_t)h->pos[b.idx[i*ti.arity + pslot]];
      }
      int unsorted = 0;
#pragma omp parallel for schedule(static) reduction(|:unsorted)
      for (int64_t i = 1; i < n; i++) unsorted |= key[i-1] > key[i];
      if (unsorted) {
        // Fast path: the caller lists each landmark's factors contiguously with ascending poses (how DynOSAM's
        // formulations add them) and only the ORDER OF THE LANDMARKS differs from ours -- then sorting the runs (one per
        // landmark) replaces sorting the factors.  Anything else falls back to the general stable sort.
        std::vector<int64_t> run0;                                 // first factor of each run of equal group rank
        {
          const int nseg = std::max(1, std::min<int>(omp_get_max_threads(), (int)(n/65536) + 1));
          std::vector<std::vector<int64_t>> seg(nseg);
#pragma omp parallel for schedule(static, 1)
          for (int t = 0; t < nseg; t++) {
            const int64_t s0 = n*t/nseg, s1 = n*(t + 1)/nseg;
            for (int64_t i = s0; i < s1; i++) if (i == 0 || frank[i] != frank[i-1]) seg[t].push_back(i);
          }
          for (auto& v : seg) run0.insert(run0.end(), v.begin(), v.end());
        }
        const int64_t nrun = (int64_t)run0.size();
        int bad = 0;                                               // a rank in two runs, or poses not ascending inside a run
        std::vector<int64_t> order(nrun);
        if (nrun <= (int64_t)gorder.size()) {
#pragma omp parallel for schedule(static) reduction(|:bad)
          for (int64_t r = 0; r < nrun; r++) {
            order[r] = r;
            const int64_t e = r + 1 < nrun ? run0[r + 1] : n;
            for (int64_t i = run0[r] + 1; i < e; i++) bad |= key[i-1] > key[i];
          }
          if (!bad) {
            __gnu_parallel::sort(order.begin(), order.end(), [&](int64_t a, int64_t c) { return frank[run0[a]] < frank[run0[c]]; });
#pragma omp parallel for schedule(static) reduction(|:bad)
            for (int64_t r = 1; r < nrun; r++) bad |= frank[run0[order[r-1]]] == frank[run0[order[r]]];
          }
        } else bad = 1;
        if (!bad) {
          std::vector<int64_t> dst(nrun + 1, 0);
          for (int64_t r = 0; r < nrun; r++) { const int64_t a = order[r]; dst[r + 1] = dst[r] + ((a + 1 < nrun ? run0[a + 1] : n) - run0[a]); }
#pragma omp parallel for schedule(static)
          for (int64_t r = 0; r < nrun; r++) {
            const int64_t a = order[r], len = dst[r + 1] - dst[r];
            for (int64_t k = 0; k < len; k++) b.perm[dst[r] + k] = (int32_t)(run0[a] + k);
          }
        } else {
          __gnu_parallel::stable_sort(b.perm.begin(), b.perm.end(), [&](int a, int c) { return key[a] < key[c]; });
        }
      }
    }
    lap("  blk sort");
    // SoA host images
    // staging images: plain new[] (no value-initialisation pass over ~1 GB), padding filled explicitly below
    struct Buf32 { std::unique_ptr<int32_t[]> p; size_t n; int32_t* data() { return p.get(); } size_t size() const { return n; } int32_t& operator[](size_t i) { return p[i]; } };
    struct Buf64 { std::unique_ptr<double[]> p; size_t n; double* data() { return p.get(); } size_t size() const { return n; } double& operator[](size_t i) { return p[i]; } };
    struct View32 { int32_t* p; size_t n; std::unique_ptr<int32_t[]> own; int32_t* data() { return p; } size_t size() const { return n; } int32_t& operator[](size_t i) { return p[i]; } };
    struct View64 { double* p; size_t n; std::unique_ptr<double[]> own; double* data() { return p; } size_t size() const { return n; } double& operator[](size_t i) { return p[i]; } };
    auto mk32 = [&](size_t cnt) { View32 v; v.n = cnt; v.p = (int32_t*)g_arena.take(cnt*4); if (!v.p) { v.own.reset(new int32_t[cnt]); v.p = v.own.get(); } return v; };
    auto mk64 = [&](size_t cnt) { View64 v; v.n = cnt; v.p = (double*)g_arena.take(cnt*8); if (!v.p) { v.own.reset(new double[cnt]); v.p = v.own.get(); } return v; };
    View32 hidx = mk32((size_t)ti.arity*stride);
    View64 hmeas = mk64((size_t)std::max(ti.meas, 1)*stride);
    View64 hsig = mk64((size_t)b.sigma_dim*stride);
    View32 haux = mk32((size_t)stride);
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
        hidx[(size_t)k*stride + s] = is_poselike(ti.cls[k]) ? h->pos[plx(ti.cls[k], ix)] : (ti.cls[k] == VC_POINT ? h->pt_new[ix] : h->fl_new[ix]);
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
      if ((rc = dalloc(h, &dgp, gp.size()))) return rc; CK(cudaMemcpy(dgp, gp.data(), gp.size()*4, cudaMemcpyHostToDevice));
      if ((rc = dalloc(h, &dgl, gl.size()))) return rc; if (!gl.empty()) CK(cudaMemcpy(dgl, gl.data(), gl.size()*4, cudaMemcpyHostToDevice));
      d.n_groups = (int)gl.size(); d.grp_ptr = dgp; d.grp_lmk = dgl;
      b.simple = true;
      // ---- window decomposition (kernels_window.cu) for the 3-dof landmark types
      const bool win_type = b.type == F_POSE2POINT3 || b.type == F_STEREO3 || b.type == F_HYBRID3 || b.type == F_HYBRID_STEREO3;
      b.use_window = false; b.all_window = false; b.win = DevWindows{};
      if (win_type && !gl.empty()) {
        const int ng = (int)gl.size(), NPs = ti.npose;
        std::vector<unsigned char> gwin(ng, 0);
        std::vector<unsigned char, NoInitAlloc<unsigned char>> lvar((size_t)NPs*stride);   // only read for window-path factors
        std::vector<int32_t> chunk_nloc, cvars; std::vector<int4> jobs, batches;
        int pose_slot[2] = {0, 0}; { int c = 0; for (int k = 0; k < ti.arity; k++) if (ti.cls[k] == VC_POSE && c < 2) pose_slot[c++] = k; }
        // window size: one 512-thread CTA holds 16 tiles of 8x4 blocks; NLOC 24 -> 12 tiles (one stripe), NLOC 40 -> 30 (two)
        int cap = NPs == 1 ? 24 : 40;
        // greedy chunking, independently inside parallel segments of the group list (a chunk never crosses a segment)
        const int nseg = std::max(1, std::min<int>(omp_get_max_threads(), ng/4096 + 1));
        struct SegOut { std::vector<int32_t> g0, nloc, cv, b0; std::vector<int4> bat; };   // b0: first batch of each chunk (+ end)
        std::vector<SegOut> seg(nseg);
#pragma omp parallel for schedule(static, 1)
        for (int t = 0; t < nseg; t++) {
          const int ga = (int)((int64_t)ng*t/nseg), gb_ = (int)((int64_t)ng*(t + 1)/nseg);
          std::vector<int32_t> stamp(NP, -1), gstamp(NP, -1), inchunk(NP, -1), cur;   // indexed by solver position
          int cur_g0 = ga, chunk_id = 0; SegOut& out = seg[t];
          auto close_chunk = [&](int g_end) {
            std::vector<int32_t> sorted = cur; std::sort(sorted.begin(), sorted.end());
            for (size_t i = 0; i < sorted.size(); i++) stamp[sorted[i]] = (int32_t)i;       // position -> local index
            for (int g = cur_g0; g < g_end; g++) if (gwin[g] == 1)
              for (int s_ = gp[g]; s_ < gp[g+1]; s_++) for (int k = 0; k < NPs; k++)
                lvar[(size_t)k*stride + s_] = (unsigned char)stamp[hidx[(size_t)pose_slot[k]*stride + s_]];
            for (size_t i = 0; i < sorted.size(); i++) stamp[sorted[i]] = -1;
            out.g0.push_back(cur_g0); out.nloc.push_back((int32_t)sorted.size());
            sorted.resize(WIN_NLOC_MAX, 0); out.cv.insert(out.cv.end(), sorted.begin(), sorted.end());
            // batches of the chunk: runs of window-path landmarks (other groups end a run), bounded in landmarks and slots
            out.b0.push_back((int32_t)out.bat.size());
            int rg0 = -1, rslots = 0;
            auto close_batch = [&](int ge) { if (rg0 >= 0) out.bat.push_back(make_int4(rg0, ge, gp[rg0], gp[ge])); rg0 = -1; rslots = 0; };
            for (int g = cur_g0; g < g_end; g++) {
              if (gwin[g] != 1) { close_batch(g); continue; }
              const int ns_ = (gp[g+1] - gp[g])*NPs;
              if (rg0 >= 0 && (rslots + ns_ > WIN_BATCH_SLOTS || g - rg0 >= WIN_BATCH_LMK)) close_batch(g);
              if (rg0 < 0) rg0 = g;
              rslots += ns_;
            }
            close_batch(g_end);
            chunk_id++; cur.clear(); cur_g0 = g_end;
          };
          for (int g = ga; g < gb_; g++) {
            if (gl[g] < 0) continue;
            const int T = gp[g+1] - gp[g];
            bool dup = false; int fresh = 0;
            if (T > WIN_TMAX) { gwin[g] = 2; continue; }
            for (int s_ = gp[g]; s_ < gp[g+1] && !dup; s_++) for (int k = 0; k < NPs; k++) {
              const int p_ = hidx[(size_t)pose_slot[k]*stride + s_];
              if (gstamp[p_] == g) { dup = true; break; }
              gstamp[p_] = g;
              if (inchunk[p_] != chunk_id) fresh++;
            }
            if (dup) { gwin[g] = 2; continue; }
            if (!cur.empty() && (int)cur.size() + fresh > cap) {      // a landmark wider than cap gets a chunk of its own
              close_chunk(g);
            }
            for (int s_ = gp[g]; s_ < gp[g+1]; s_++) for (int k = 0; k < NPs; k++) {
              const int p_ = hidx[(size_t)pose_slot[k]*stride + s_];
              if (inchunk[p_] != chunk_id) { inchunk[p_] = chunk_id; cur.push_back(p_); }
            }
            gwin[g] = 1;
          }
          close_chunk(gb_);
        }
        for (int t = 0; t < nseg; t++) for (size_t c = 0; c < seg[t].g0.size(); c++) {
          const int chunk_id = (int)chunk_nloc.size();
          chunk_nloc.push_back(seg[t].nloc[c]);
          cvars.insert(cvars.end(), seg[t].cv.begin() + c*WIN_NLOC_MAX, seg[t].cv.begin() + (c + 1)*WIN_NLOC_MAX);
          const int nl_ = seg[t].nloc[c]; const int ntile = win_ntiles(nl_);
          const size_t sb0 = seg[t].b0[c], sb1 = c + 1 < seg[t].b0.size() ? seg[t].b0[c + 1] : seg[t].bat.size();
          const int b0 = (int)batches.size();
          batches.insert(batches.end(), seg[t].bat.begin() + sb0, seg[t].bat.begin() + sb1);
          const int b1 = (int)batches.size();
          if (b1 > b0) for (int st = 0; st*WIN_ACC_WARPS < ntile; st++) jobs.push_back(make_int4(chunk_id, st, b0, b1));
        }
        int4* djobs; int4* dbat; int* dnl; int* dcv; unsigned char* dlv; unsigned char* dgw; double* dslots;
        if ((rc = dalloc(h, &djobs, jobs.size()))) return rc; if (!jobs.empty()) CK(cudaMemcpy(djobs, jobs.data(), jobs.size()*sizeof(int4), cudaMemcpyHostToDevice));
        if ((rc = dalloc(h, &dbat, batches.size()))) return rc; if (!batches.empty()) CK(cudaMemcpy(dbat, batches.data(), batches.size()*sizeof(int4), cudaMemcpyHostToDevice));
        if ((rc = dalloc(h, &dnl, chunk_nloc.size()))) return rc; CK(cudaMemcpy(dnl, chunk_nloc.data(), chunk_nloc.size()*4, cudaMemcpyHostToDevice));
        if ((rc = dalloc(h, &dcv, cvars.size()))) return rc; CK(cudaMemcpy(dcv, cvars.data(), cvars.size()*4, cudaMemcpyHostToDevice));
        if ((rc = dalloc(h, &dlv, lvar.size()))) return rc; CK(cudaMemcpy(dlv, lvar.data(), lvar.size(), cudaMemcpyHostToDevice));
        if ((rc = dalloc(h, &dgw, gwin.size()))) return rc; CK(cudaMemcpy(dgw, gwin.data(), gwin.size(), cudaMemcpyHostToDevice));
        if ((rc = dalloc(h, &dslots, (size_t)n*NPs*WIN_SLOT_DOUBLES, false))) return rc;
        b.win.n_jobs = (int)jobs.size(); b.win.jobs = djobs; b.win.batches = dbat; b.win.chunk_nloc = dnl; b.win.cvars = dcv; b.win.lvar = dlv; b.win.grp_win = dgw; b.win.slots = dslots;
        b.use_window = true;
        { size_t nw = 0; for (int g = 0; g < ng; g++) nw += gwin[g] == 1 || gl[g] < 0; b.all_window = nw == (size_t)ng; }
      }
    }
    lap("  blk groups+windows");
    b.part_off = part; part += is_nav_type(b.type) ? nav_grid(b.type, (int)n) : linearize_grid((int)n);
    b.bs_off = bs; bs += b.pose_only ? (int)((n + 127)/128) : backsub_grid(d.n_groups);
    const int64_t rd = 4*ti.arity + 8*ti.meas + 8*b.sigma_dim + (b.has_aux ? 4 : 0), wr = 8*(ti.dim*ti.jcols + ti.dim);
    h->jac_bytes += n*(rd + wr);
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
      for (int64_t i = 0; i < nl; i++) { const int g = rank2g[grank[root[i]]]; if (g >= 0) { if (i >= npt) { h->supported = false; continue; } gl0[g] = std::min(gl0[g], h->pt_new[i]); } }
    }
    std::vector<DevBlock> hb; for (auto& b : h->blocks) hb.push_back(b.dev);
    DevBlock* dblk; int* dgptr; int* drefs; int* dgl0; int* dgnl; int rc;
    if ((rc = dalloc(h, &dblk, hb.size()))) return rc; CK(cudaMemcpy(dblk, hb.data(), hb.size()*sizeof(DevBlock), cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dgptr, gptr.size()))) return rc; CK(cudaMemcpy(dgptr, gptr.data(), gptr.size()*4, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &drefs, refs.size()))) return rc; CK(cudaMemcpy(drefs, refs.data(), refs.size()*4, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dgl0, gl0.size()))) return rc; CK(cudaMemcpy(dgl0, gl0.data(), gl0.size()*4, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dgnl, gnl.size()))) return rc; CK(cudaMemcpy(dgnl, gnl.data(), gnl.size()*4, cudaMemcpyHostToDevice));
    h->gen.n_groups = (int)gl0.size(); h->gen.blocks = dblk; h->gen.gptr = dgptr; h->gen.refs = drefs; h->gen.gl0 = dgl0; h->gen.gnl = dgnl;
  }
  for (auto& P : h->priors) {
    const int n = (int)P.idx.size(); std::vector<int32_t> ppos(n);
    for (int i = 0; i < n; i++) ppos[i] = h->pos[P.idx[i]];
    int* dpos; double *dlin, *dG, *dg, *dd, *dgc; int rc;
    if ((rc = dalloc(h, &dpos, (size_t)n, false))) return rc; CK(cudaMemcpy(dpos, ppos.data(), (size_t)n*4, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dlin, (size_t)12*n, false))) return rc; CK(cudaMemcpy(dlin, P.lin.data(), (size_t)12*n*8, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dG, (size_t)36*n*n, false))) return rc; CK(cudaMemcpy(dG, P.G.data(), (size_t)36*n*n*8, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dg, (size_t)6*n, false))) return rc; CK(cudaMemcpy(dg, P.g.data(), (size_t)6*n*8, cudaMemcpyHostToDevice));
    if ((rc = dalloc(h, &dd, (size_t)6*n))) return rc; if ((rc = dalloc(h, &dgc, (size_t)6*n))) return rc;
    P.dev = DevPrior{ n, dpos, dlin, dG, dg, P.f, dd, dgc };
    P.part_off = part; part += 1; P.bs_off = bs; bs += 1;
  }
  h->n_nav = 0; h->d_nav = nullptr;
  if (NP > np) {
    std::vector<int2> nav(nv + nb);
    for (int64_t i = 0; i < nv; i++) nav[i] = make_int2(h->pos[np + i], 3);
    for (int64_t i = 0; i < nb; i++) nav[nv + i] = make_int2(h->pos[np + nv + i], 6);
    int rc; if ((rc = dalloc(h, &h->d_nav, nav.size(), false))) return rc;
    CK(cudaMemcpy(h->d_nav, nav.data(), nav.size()*sizeof(int2), cudaMemcpyHostToDevice));
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
  const std::vector<double>* v = var_store(h, kind);
  ARG(v, "bad variable kind");
  *out = (int64_t)v->size()/kind_width(kind);
  return DYNOBA_OK;
}
int dynoba_get_keys(dynoba_handle h, int kind, int64_t n, uint64_t* out) {
  ARG(h && out, "null");
  const std::vector<uint64_t>* kp = key_store(h, kind);
  ARG(kp, "bad variable kind");
  const auto& k = *kp;
  ARG((int64_t)k.size() == n, "no keys stored / size mismatch");
  std::copy(k.begin(), k.end(), out);
  return DYNOBA_OK;
}
int dynoba_problem_info(dynoba_handle h, int32_t* reduced_dim, int32_t* bandwidth, int64_t* jacobian_bytes) {
  int rc = check_ready(h, false); if (rc) return rc;
  if (reduced_dim) *reduced_dim = h->band.n; if (bandwidth) *bandwidth = h->band.bw; if (jacobian_bytes) *jacobian_bytes = h->jac_bytes;
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
  auto& b = h->blocks[bi]; const TypeInfo ti = type_info(b.type);
  CK(cudaEventRecord(h->ev[0], h->stream));
  h->launches += launch_linearize(b.dev, h->cur, h->partials + b.part_off, h->stream);
  CK(cudaEventRecord(h->ev[1], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (ms) CK(cudaEventElapsedTime(ms, h->ev[0], h->ev[1]));
  if (bytes) {   // factor record read once + whitened tiles written once (variable reads left out: conservative)
    const int64_t rd = 4*ti.arity + 8*ti.meas + 8*b.sigma_dim + (b.has_aux ? 4 : 0), wr = 8*(ti.dim*ti.jcols + ti.dim);
    *bytes = b.n*(rd + wr);
  }
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
  { auto it = std::find_if(h->allocs.begin(), h->allocs.end(), [&](const std::pair<void*, size_t>& a) { return a.first == (void*)d; });
    g_devcache.give(h->device, it->first, it->second); h->allocs.erase(it); }
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
  // caller layout [poses 6 | velocities 3 | biases 6]; the inert scalars of the velocity blocks are left out
  const int nb_ = B.n; const int64_t NP = nb_/6, np = (int64_t)h->pose.size()/12, nv = (int64_t)h->vel.size()/3;
  std::vector<int32_t> usr(nb_, -1);
  for (int64_t i = 0; i < NP; i++) {
    const int64_t off = i < np ? 6*i : (i < np + nv ? 6*np + 3*(i - np) : 6*np + 3*nv + 6*(i - np - nv));
    const int d = i >= np && i < np + nv ? 3 : 6;
    for (int c = 0; c < d; c++) usr[6*(size_t)h->pos[i] + c] = (int32_t)(off + c);
  }
  const int n = (int)(nb_ - 3*nv);
  if (S) {
    std::fill(S, S + (size_t)n*n, 0.0);
    for (int j = 0; j < nb_; j++) for (int i = j; i < nb_ && i <= j + B.bw; i++) {
      if (usr[i] < 0 || usr[j] < 0) continue;
      const double v = *band_at(HB, i, j);
      S[(size_t)usr[i]*n + usr[j]] = v; S[(size_t)usr[j]*n + usr[i]] = v;
    }
  }
  if (g) for (int i = 0; i < nb_; i++) if (usr[i] >= 0) g[usr[i]] = *rhs_at(HB, i);
  return DYNOBA_OK;
}

static int download_delta(dynoba_solver* h, double* delta) {
  const DevBand& B = h->band; const int64_t np = (int64_t)h->pose.size()/12, npt = h->cur.nl, nfl = h->cur.nf;
  std::vector<double> hr(B.n_pad), hp((size_t)3*h->cur.nl_stride), hf((size_t)2*h->cur.nf_stride);
  CK(cudaMemcpyAsync(hr.data(), B.dp, hr.size()*8, cudaMemcpyDeviceToHost, h->stream));
  if (npt) CK(cudaMemcpyAsync(hp.data(), h->dl_point, hp.size()*8, cudaMemcpyDeviceToHost, h->stream));
  if (nfl) CK(cudaMemcpyAsync(hf.data(), h->dl_flow, hf.size()*8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int64_t i = 0; i < np; i++) for (int c = 0; c < 6; c++) delta[6*i + c] = hr[6*(size_t)h->pos[i] + c];
  double* dp = delta + 6*np;
  for (int64_t i = 0; i < npt; i++) for (int c = 0; c < 3; c++) dp[3*i + c] = hp[(size_t)c*h->cur.nl_stride + h->pt_new[i]];
  double* df = dp + 3*npt;
  for (int64_t i = 0; i < nfl; i++) for (int c = 0; c < 2; c++) df[2*i + c] = hf[(size_t)c*h->cur.nf_stride + h->fl_new[i]];
  double* dn = df + 2*nfl;          // velocities (3), then biases (6)
  for (int64_t i = np; i < (int64_t)h->pos.size(); i++) {
    const int d = i < np + (int64_t)h->vel.size()/3 ? 3 : 6;
    for (int c = 0; c < d; c++) *dn++ = hr[6*(size_t)h->pos[i] + c];
  }
  return DYNOBA_OK;
}

int dynoba_solve(dynoba_handle h, double lambda, double* delta) {
  int rc = check_ready(h, true); if (rc) return rc;
  ARG(delta, "null delta");
  if (!h->linearized) do_linearize(h);
  rc = build_reduced(h, lambda); if (rc) return rc;
  rc = solve_step(h, lambda); if (rc) return rc;
  double s[4]; rc = read_scalars(h, s, true); if (rc) return rc;
  CK(cudaGetLastError());
  if (s[3] != 0.0) { h->err = "reduced system not positive definite"; return DYNOBA_ERR_INDETERMINATE; }
  return download_delta(h, delta);
}

int dynoba_retract(dynoba_handle h, const double* delta) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(delta, "null delta");
  const DevBand& B = h->band; const int64_t np = (int64_t)h->pose.size()/12, npt = h->cur.nl, nfl = h->cur.nf;
  std::vector<double> hr(B.n_pad, 0.0), hp((size_t)3*h->cur.nl_stride, 0.0), hf((size_t)2*h->cur.nf_stride, 0.0);
  for (int64_t i = 0; i < np; i++) for (int c = 0; c < 6; c++) hr[6*(size_t)h->pos[i] + c] = delta[6*i + c];
  const double* dp = delta + 6*np;
  for (int64_t i = 0; i < npt; i++) for (int c = 0; c < 3; c++) hp[(size_t)c*h->cur.nl_stride + h->pt_new[i]] = dp[3*i + c];
  const double* df = dp + 3*npt;
  for (int64_t i = 0; i < nfl; i++) for (int c = 0; c < 2; c++) hf[(size_t)c*h->cur.nf_stride + h->fl_new[i]] = df[2*i + c];
  const double* dn = df + 2*nfl;    // velocities (3), then biases (6)
  for (int64_t i = np; i < (int64_t)h->pos.size(); i++) {
    const int d = i < np + (int64_t)h->vel.size()/3 ? 3 : 6;
    for (int c = 0; c < d; c++) hr[6*(size_t)h->pos[i] + c] = *dn++;
  }
  CK(cudaMemcpyAsync(B.dp, hr.data(), hr.size()*8, cudaMemcpyHostToDevice, h->stream));
  if (npt) CK(cudaMemcpyAsync(h->dl_point, hp.data(), hp.size()*8, cudaMemcpyHostToDevice, h->stream));
  if (nfl) CK(cudaMemcpyAsync(h->dl_flow, hf.data(), hf.size()*8, cudaMemcpyHostToDevice, h->stream));
  h->launches += launch_retract(h->cur, h->cand, h->band, h->dl_point, h->dl_flow, h->stream);
  h->launches += launch_nav_retract(h->cur, h->cand, h->band, h->d_nav, h->n_nav, h->stream);
  CK(cudaStreamSynchronize(h->stream));
  std::swap(h->cur, h->cand);
  h->linearized = false;
  return DYNOBA_OK;
}

// Marginal information of the LAST n_keep pose-like variables (solver order) at the current values: every landmark and
// every other pose-like variable eliminated.  The band Cholesky already leaves a Schur complement in the columns it does
// not factor, so this is one plain band factorisation that stops at the tile holding the first kept variable; the few
// scalars of that tile that precede the kept block are eliminated on the host.
int dynoba_marginal(dynoba_handle h, int32_t n_keep, const int32_t* keep_pose_idx, double* G, double* g) {
  int rc = check_ready(h, true); if (rc) return rc;
  ARG(n_keep > 0 && keep_pose_idx && G && g, "bad arguments");
  if (has_nav(h)) { h->err = "dynoba_marginal is not available with velocity / bias variables"; return DYNOBA_ERR_UNSUPPORTED; }
  const int64_t np = h->cur.np;
  ARG(n_keep <= np, "more variables than there are");
  if (h->world > 1) { h->err = "dynoba_marginal is a single-GPU entry point"; return DYNOBA_ERR_UNSUPPORTED; }
  std::vector<int> slot(n_keep, -1);                    // kept variable k sits at solver position np - n_keep + slot
  for (int k = 0; k < n_keep; k++) {
    ARG(keep_pose_idx[k] >= 0 && keep_pose_idx[k] < np, "variable out of range");
    const int p = h->pos[keep_pose_idx[k]] - (int)(np - n_keep);
    if (p < 0) { h->err = "the kept variables must be the last ones of the elimination order (most recent frames)"; return DYNOBA_ERR_UNSUPPORTED; }
    slot[k] = p;
  }
  { std::vector<int> srt = slot; std::sort(srt.begin(), srt.end()); ARG(std::adjacent_find(srt.begin(), srt.end()) == srt.end(), "a variable is listed twice"); }
  if (!h->linearized) do_linearize(h);
  // a second, plain layout whose factorisation stops before the kept block
  BandPlan mp{}; mp.outer_weight = 0;
  if (band_plan_layout(mp, h->band.n, h->band.bw, -1, 0, 1)) { h->err = "band layout failed"; return DYNOBA_ERR_BAD_ARG; }
  const int p0 = 6*(int)(np - n_keep), K0 = p0/TILE, NT = mp.band.NT, WBm = mp.band.WB;
  if (NT - K0 > WBm + 1) { h->err = "the kept block is wider than the band of the reduced system"; return DYNOBA_ERR_UNSUPPORTED; }
  mp.chains[0].Kend = K0;
  double* dbuf; int* ibuf; char* desc;
  if ((rc = dalloc(h, &dbuf, mp.n_doubles, false))) return rc;
  if ((rc = dalloc(h, &ibuf, mp.n_ints, false))) return rc;
  if ((rc = dalloc(h, &desc, mp.n_desc_bytes))) return rc;
  band_plan_bind(mp, dbuf, ibuf, desc, nullptr);
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
  for (void* q : { (void*)dbuf, (void*)ibuf, (void*)desc }) {
    auto it = std::find_if(h->allocs.begin(), h->allocs.end(), [&](const std::pair<void*, size_t>& a) { return a.first == q; });
    if (it != h->allocs.end()) { g_devcache.give(h->device, it->first, it->second); h->allocs.erase(it); }
  }
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
  const int dim = 6*n_keep;
  for (int a = 0; a < n_keep; a++) for (int r = 0; r < 6; r++) {
    const int qi = e + 6*slot[a] + r;
    g[6*a + r] = rhs[qi];
    for (int b = 0; b < n_keep; b++) for (int c = 0; c < 6; c++) G[(size_t)(6*a + r)*dim + 6*b + c] = M[(size_t)qi*m + e + 6*slot[b] + c];
  }
  return DYNOBA_OK;
}

int dynoba_get_variables(dynoba_handle h, int kind, int64_t n, double* out) {
  int rc = check_ready(h, false); if (rc) return rc;
  ARG(out, "null out");
  const DevVars& V = h->cur;
  if (kind == DYNOBA_POSE6 || kind == DYNOBA_VEL3 || kind == DYNOBA_BIAS6) {
    const int64_t np = (int64_t)h->pose.size()/12, nv = (int64_t)h->vel.size()/3, w = kind_width(kind);
    ARG(n == (int64_t)var_store(h, kind)->size()/w, "size mismatch");
    const int64_t base = kind == DYNOBA_POSE6 ? 0 : (kind == DYNOBA_VEL3 ? np : np + nv);
    std::vector<double> soa((size_t)12*V.np_stride);
    CK(cudaMemcpy(soa.data(), V.pose, soa.size()*8, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; i++) for (int k = 0; k < w; k++) out[i*w + k] = soa[(size_t)k*V.np_stride + h->pos[base + i]];
  } else if (kind == DYNOBA_POINT3) {
    ARG(n == V.nl, "size mismatch");
    std::vector<double> soa((size_t)3*V.nl_stride);
    CK(cudaMemcpy(soa.data(), V.point, soa.size()*8, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; i++) for (int k = 0; k < 3; k++) out[i*3 + k] = soa[(size_t)k*V.nl_stride + h->pt_new[i]];
  } else if (kind == DYNOBA_FLOW2) {
    ARG(n == V.nf, "size mismatch");
    std::vector<double> soa((size_t)2*V.nf_stride);
    CK(cudaMemcpy(soa.data(), V.flow, soa.size()*8, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; i++) for (int k = 0; k < 2; k++) out[i*2 + k] = soa[(size_t)k*V.nf_stride + h->fl_new[i]];
  } else ARG(false, "bad kind");
  return DYNOBA_OK;
}

// LevenbergMarquardtOptimizer::optimize()  [GTSAM-ext nonlinear/{NonlinearOptimizer,LevenbergMarquardtOptimizer}.cpp]
int dynoba_optimize(dynoba_handle h, const dynoba_lm_params* prm, dynoba_lm_stats* st) {
  int rc = check_ready(h, true); if (rc) return rc;
  dynoba_lm_params P; if (prm) P = *prm; else dynoba_lm_default_params(&P);
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
  if (!(err <= P.error_tol) && P.max_iterations > 0) {
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
        const bool solved = sc[3] == 0.0 && std::isfinite(sc[1]);
        bool success = false, stop = false; double nerr = INFINITY;
        if (solved) {
          const double oldLin = sc[0], lin = sc[1];
          if (lin >= 0) {
            nerr = sc[2];
            const double cost = err - nerr;
            if (lin > DBL_EPSILON*oldLin) { const double fid = cost/lin; success = fid > P.min_model_fidelity; }
            if (std::fabs(cost) < P.relative_error_tol*err) stop = true;
          }
          if (P.verbosity > 0) std::fprintf(stderr, "[dynoba-lm] it %d inner %d lambda %.3e err %.12e -> %.12e lin %.6e %s\n", iterations, inner, lambda, err, nerr, lin, success ? "ok" : "rej");
        } else if (P.verbosity > 0) std::fprintf(stderr, "[dynoba-lm] it %d inner %d lambda %.3e solve failed (flag %.0f)\n", iterations, inner, lambda, sc[3]);
        if (success) { std::swap(h->cur, h->cand); h->linearized = false; lambda = std::max(P.lambda_lower_bound, lambda/P.lambda_factor); err = nerr; iterations++; inner++; break; }
        else if (!stop) { lambda *= P.lambda_factor; inner++; if (lambda >= P.lambda_upper_bound) break; }
        else break;
      }
      { float m2; cudaEventElapsedTime(&m2, ev[0], ev[1]); S.ms_linearize += m2; }
      newError = err;
    } while (iterations < P.max_iterations &&
             !((newError <= P.error_tol) ||
               ((P.relative_error_tol != 0.0) && ((currentError - newError)/currentError <= P.relative_error_tol)) ||
               ((currentError - newError) <= P.absolute_error_tol)) &&
             std::isfinite(currentError));
  }
  tick(7); cudaEventSynchronize(ev[7]); cudaEventElapsedTime(&ms, ev[6], ev[7]); S.ms_total = ms;
  S.iterations = iterations; S.inner_iterations = inner; S.error_final = err; S.lambda_final = lambda;
  S.kernel_launches = h->launches - launches0;
  if (st) *st = S;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return DYNOBA_ERR_CUDA; }
  return DYNOBA_OK;
}

}  // extern "C"
