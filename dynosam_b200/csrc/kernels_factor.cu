// kernels_factor.cu -- K1 materialising linearize (the roofline kernel) and K2 chi^2 sweep.
//
// K1 restates gtsam::NonlinearFactorGraph::linearize -> NoiseModelFactor::linearize ->
// noiseModel::Robust::WhitenSystem [GTSAM-ext], i.e. SURVEY.md 8a rows a2-a10, as ONE data-parallel pass
// per factor type: one thread per factor, coalesced SoA reads of the factor stream, L2-resident gathers of
// the pose/point variables (read-only path), SoA stores of the whitened Jacobian tiles and rhs.
// Algorithmic bytes per factor (DESIGN.md): POSE2POINT3/STEREO3 280 B, TERNARY3 332 B, HYBRID3 432 B.
#include "internal.cuh"

namespace dynoba {

constexpr int LIN_THREADS = 128;

__device__ __forceinline__ void load_pose(const double* __restrict__ base, int stride, int i, Pose& P) {
#pragma unroll
  for (int k = 0; k < 9; k++) P.R[k] = __ldg(base + (size_t)k*stride + i);
#pragma unroll
  for (int k = 0; k < 3; k++) P.t[k] = __ldg(base + (size_t)(9 + k)*stride + i);
}

template <int T>
__device__ __forceinline__ void gather_vars(const DevBlock& blk, const DevVars& v, int f, FVars& fv, Pose& aux) {
  constexpr TypeInfo ti = type_info(T);
  int pi = 0, li = 0;
#pragma unroll
  for (int k = 0; k < ti.arity; k++) {
    const int ix = __ldg(blk.idx + (size_t)k*blk.stride + f);
    if (ti.cls[k] == VC_POSE) { load_pose(v.pose, v.np_stride, ix, fv.pose[pi]); pi++; }
    else if (ti.cls[k] == VC_POINT) {
#pragma unroll
      for (int c = 0; c < 3; c++) fv.pt[li][c] = __ldg(v.point + (size_t)c*v.nl_stride + ix);
      li++;
    } else {
      fv.pt[li][0] = __ldg(v.flow + ix); fv.pt[li][1] = __ldg(v.flow + v.nf_stride + ix); fv.pt[li][2] = 0.0;
      li++;
    }
  }
  if (ti.needs_aux) load_pose(v.aux, v.naux_stride, __ldg(blk.aux + f), aux);
}

__device__ __forceinline__ double block_sum(double x, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sh[w] = x;
  __syncthreads();
  double t = 0;
  if (threadIdx.x == 0) for (int i = 0; i < (int)(blockDim.x >> 5); i++) t += sh[i];   // fixed order
  return t;
}

// K1.  partials[blockIdx.x] = sum over the block's factors of 0.5*|b|^2 (the linearised error at delta = 0).
// hybrid types: cap at 80 registers (6 CTAs/SM instead of 5) -- more bytes in flight for the HBM-bound store stream
template <int T>
__global__ void __launch_bounds__(LIN_THREADS, (T == F_HYBRID3 || T == F_HYBRID_STEREO3) ? 6 : 1) linearize_kernel(DevBlock blk, DevVars v, double* __restrict__ partials) {
  constexpr TypeInfo ti = type_info(T);
  constexpr int D = ti.dim, JC = ti.jcols, M = ti.meas;
  __shared__ double sh[LIN_THREADS/32];
  const int f = blockIdx.x*LIN_THREADS + threadIdx.x;
  double hb2 = 0.0;
  if (f < blk.n) {
    FVars fv; Pose aux;
    gather_vars<T>(blk, v, f, fv, aux);
    double z[M > 0 ? M : 1];
#pragma unroll
    for (int k = 0; k < M; k++) z[k] = __ldg(blk.meas + (size_t)k*blk.stride + f);
    double isig[D];
    if (blk.sigma_dim == 1) { isig[0] = __ldg(blk.isig + f); }
    else {
#pragma unroll
      for (int k = 0; k < D; k++) isig[k] = __ldg(blk.isig + (size_t)k*blk.stride + f);
    }
    double r[D], J[D*JC];
    factor_eval<T, true>(fv, z, aux, v.K, r, J);
    double err;
    const double sw = whiten_weight<D>(r, isig, blk.sigma_dim, blk.robust_k, &err);
#pragma unroll
    for (int k = 0; k < D; k++) {
      const double fk = (blk.sigma_dim == 1 ? isig[0] : isig[k])*sw;
#pragma unroll
      for (int c = 0; c < JC; c++) blk.J[(size_t)(k*JC + c)*blk.stride + f] = J[k*JC + c]*fk;
      const double bk = -r[k]*sw;
      blk.b[(size_t)k*blk.stride + f] = bk;
      hb2 += 0.5*bk*bk;
    }
  }
  const double tot = block_sum(hb2, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = tot;
}


// K1 for the numerically differentiated factor types (LandmarkMotionPoseFactor, HybridSmoothingFactor,
// LandmarkPoseSmoothingFactor): one thread per (factor, Jacobian column) instead of one thread per factor, so the
// 2 x 18 perturbed residual evaluations of gtsam::numericalDerivative run in parallel (18x more threads, 3 instead
// of 37 residual evaluations per thread).  Column arithmetic is identical to numeric_jacobian() in factors.cuh.
template <int T>
__global__ void __launch_bounds__(LIN_THREADS) linearize_numeric_kernel(DevBlock blk, DevVars v, double* __restrict__ partials) {
  constexpr TypeInfo ti = type_info(T);
  constexpr int D = ti.dim, JC = ti.jcols;
  __shared__ double sh[LIN_THREADS/32];
  // column-major thread map: a CTA (and every warp) works on ONE Jacobian column of 128 consecutive factors, so the
  // perturbed slot / direction is warp-uniform and the factor-stream loads stay coalesced
  const int cta_per_col = (blk.n + LIN_THREADS - 1)/LIN_THREADS;
  const int col = blockIdx.x/cta_per_col;
  const int f = (blockIdx.x - col*cta_per_col)*LIN_THREADS + threadIdx.x;
  double hb2 = 0.0;
  if (f < blk.n) {
    FVars fv; Pose aux;
    gather_vars<T>(blk, v, f, fv, aux);
    double isig[D];
    if (blk.sigma_dim == 1) { isig[0] = __ldg(blk.isig + f); }
    else {
#pragma unroll
      for (int k = 0; k < D; k++) isig[k] = __ldg(blk.isig + (size_t)k*blk.stride + f);
    }
    double hx[D], h1[D], h2[D];
    numeric_residual<T>(fv, aux, hx);
    // which key slot / tangent direction does this column perturb?
    int slot = 0, j = col;
#pragma unroll
    for (int k = 0; k < ti.arity; k++) if (col >= ti.coloff[k]) { slot = k; j = col - ti.coloff[k]; }
    int pi = 0, li = 0;
#pragma unroll
    for (int k = 0; k < ti.arity; k++) if (k < slot) { if (ti.cls[k] == VC_POSE) pi++; else li++; }
    constexpr double delta = 1e-5, factor = 1.0/(2.0*delta);
#pragma unroll
    for (int sgn = 0; sgn < 2; sgn++) {
      FVars w = fv;
      const double d = sgn == 0 ? delta : -delta;
      bool is_pose = false;
#pragma unroll
      for (int k = 0; k < ti.arity; k++) if (k == slot) is_pose = ti.cls[k] == VC_POSE;
      if (is_pose) {
        double xi[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int q = 0; q < 6; q++) if (q == j) xi[q] = d;
#pragma unroll
        for (int p = 0; p < 3; p++) if (p == pi) se3_retract(fv.pose[p], xi, w.pose[p]);
      } else {
#pragma unroll
        for (int p = 0; p < 2; p++)
#pragma unroll
          for (int q = 0; q < 3; q++) if (p == li && q == j) w.pt[p][q] += d;
      }
      numeric_residual<T>(w, aux, sgn == 0 ? h1 : h2);
    }
    double r[D];
#pragma unroll
    for (int k = 0; k < D; k++) r[k] = hx[k];
    double err;
    const double sw = whiten_weight<D>(r, isig, blk.sigma_dim, blk.robust_k, &err);
#pragma unroll
    for (int k = 0; k < D; k++) {
      const double fk = (blk.sigma_dim == 1 ? isig[0] : isig[k])*sw;
      blk.J[(size_t)(k*JC + col)*blk.stride + f] = ((h1[k] - hx[k]) - (h2[k] - hx[k]))*factor*fk;
      if (col == 0) { const double bk = -r[k]*sw; blk.b[(size_t)k*blk.stride + f] = bk; hb2 += 0.5*bk*bk; }
    }
  }
  const double tot = block_sum(hb2, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = tot;
}

// K2.  chi^2 sweep: nonlinear factor errors (Gaussian 0.5|r_w|^2 or Huber rho), no Jacobians.
template <int T>
__global__ void __launch_bounds__(LIN_THREADS) error_kernel(DevBlock blk, DevVars v, double* __restrict__ partials,
                                                            double* __restrict__ per_factor) {
  constexpr TypeInfo ti = type_info(T);
  constexpr int D = ti.dim, M = ti.meas;
  __shared__ double sh[LIN_THREADS/32];
  const int f = blockIdx.x*LIN_THREADS + threadIdx.x;
  double e = 0.0;
  if (f < blk.n) {
    FVars fv; Pose aux;
    gather_vars<T>(blk, v, f, fv, aux);
    double z[M > 0 ? M : 1];
#pragma unroll
    for (int k = 0; k < M; k++) z[k] = __ldg(blk.meas + (size_t)k*blk.stride + f);
    double isig[D];
    if (blk.sigma_dim == 1) { isig[0] = __ldg(blk.isig + f); }
    else {
#pragma unroll
      for (int k = 0; k < D; k++) isig[k] = __ldg(blk.isig + (size_t)k*blk.stride + f);
    }
    double r[D];
    factor_eval<T, false>(fv, z, aux, v.K, r, nullptr);
    whiten_weight<D>(r, isig, blk.sigma_dim, blk.robust_k, &e);
    if (per_factor) per_factor[f] = e;
  }
  const double tot = block_sum(e, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = tot;
}

// deterministic final reduction: fixed strided order per thread, fixed tree
__global__ void __launch_bounds__(1024) sum_kernel(const double* __restrict__ p, int n, double* __restrict__ out) {
  __shared__ double sh[1024];
  double s = 0;
  for (int i = threadIdx.x; i < n; i += 1024) s += p[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) *out = sh[0];
}

int linearize_grid(int n) { return (n + LIN_THREADS - 1)/LIN_THREADS; }
int numeric_grid(int type, int n) {
  if (!(type == F_MOTIONPOSE3 || type == F_SMOOTH_HYBRID6 || type == F_SMOOTH_POSE6)) return 0;
  return ((n + LIN_THREADS - 1)/LIN_THREADS)*type_info(type).jcols;
}


#define DISPATCH_TYPE(T, CALL)                       \
  switch (T) {                                       \
    case F_PRIOR6: { CALL(F_PRIOR6); } break;        \
    case F_BETWEEN6: { CALL(F_BETWEEN6); } break;    \
    case F_POSE2POINT3: { CALL(F_POSE2POINT3); } break; \
    case F_STEREO3: { CALL(F_STEREO3); } break;      \
    case F_TERNARY3: { CALL(F_TERNARY3); } break;    \
    case F_HYBRID3: { CALL(F_HYBRID3); } break;      \
    case F_HYBRID_STEREO3: { CALL(F_HYBRID_STEREO3); } break; \
    case F_MOTIONPOSE3: { CALL(F_MOTIONPOSE3); } break; \
    case F_SMOOTH_HYBRID6: { CALL(F_SMOOTH_HYBRID6); } break; \
    case F_SMOOTH_POSE6: { CALL(F_SMOOTH_POSE6); } break; \
    case F_FLOWPROJ2: { CALL(F_FLOWPROJ2); } break;  \
    default: break;                                  \
  }

__global__ void fold_partials_kernel(const double* __restrict__ in, int nin, double* __restrict__ out, int nout) {
  // deterministic fold of nin per-block sums into nout slots (slot k sums in[k], in[k+nout], ...)
  const int k = blockIdx.x*blockDim.x + threadIdx.x;
  if (k >= nout) return;
  double s = 0; for (int i = k; i < nin; i += nout) s += in[i];
  out[k] = s;
}

int launch_linearize(const DevBlock& blk, const DevVars& v, double* partials, cudaStream_t s) {
  if (blk.n == 0) return 0;
  if (is_nav_type(blk.type)) return launch_nav_linearize(blk, v, partials, s);
  if (is_linear_type(blk.type)) return launch_linear_factors(blk, v, true, partials, nullptr, s);
  const int grid = linearize_grid(blk.n);
  if (blk.type == F_MOTIONPOSE3 || blk.type == F_SMOOTH_HYBRID6 || blk.type == F_SMOOTH_POSE6) {
    const int g2 = numeric_grid(blk.type, blk.n);
    double* scratch = blk.num_scratch;
    if (blk.type == F_MOTIONPOSE3) linearize_numeric_kernel<F_MOTIONPOSE3><<<g2, LIN_THREADS, 0, s>>>(blk, v, scratch);
    else if (blk.type == F_SMOOTH_HYBRID6) linearize_numeric_kernel<F_SMOOTH_HYBRID6><<<g2, LIN_THREADS, 0, s>>>(blk, v, scratch);
    else linearize_numeric_kernel<F_SMOOTH_POSE6><<<g2, LIN_THREADS, 0, s>>>(blk, v, scratch);
    fold_partials_kernel<<<(grid + 127)/128, 128, 0, s>>>(scratch, g2, partials, grid);
    return 2;
  }
#define CALL_LIN(TT) linearize_kernel<TT><<<grid, LIN_THREADS, 0, s>>>(blk, v, partials)
  DISPATCH_TYPE(blk.type, CALL_LIN)
#undef CALL_LIN
  return 1;
}

int launch_error(const DevBlock& blk, const DevVars& v, double* partials, double* per_factor, cudaStream_t s) {
  if (blk.n == 0) return 0;
  if (is_nav_type(blk.type)) return launch_nav_error(blk, v, partials, per_factor, s);
  if (is_linear_type(blk.type)) return launch_linear_factors(blk, v, false, partials, per_factor, s);
  const int grid = linearize_grid(blk.n);
#define CALL_ERR(TT) error_kernel<TT><<<grid, LIN_THREADS, 0, s>>>(blk, v, partials, per_factor)
  DISPATCH_TYPE(blk.type, CALL_ERR)
#undef CALL_ERR
  return 1;
}

int launch_sum(const double* partials, int n, double* out, cudaStream_t s) {
  sum_kernel<<<1, 1024, 0, s>>>(partials, n, out);
  return 1;
}

}  // namespace dynoba
