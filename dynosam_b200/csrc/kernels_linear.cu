// kernels_linear.cu -- linearised landmark factors: gtsam::LinearContainerFactor holding a 3-row JacobianFactor over
// (camera pose, point) or (camera pose, object motion, point), the form in which the reference's sliding window hands the
// factors of its retained landmarks to the next window (dynosam_opt/src/SlidingWindowOptimization.cc:157-188:
// eliminatePartialMultifrontal leaves them untouched, ConvertLinearGraph wraps them).  [GTSAM-ext LinearContainerFactor]
//
//   d            = lin.localCoordinates(x):  Logmap(lin^-1 x) per Pose3 slot, x - lin for the Point3 slot
//   error(x)     = 1/2 |A d - b|^2
//   linearize(x) = JacobianFactor(A, b - A d)      (A is not corrected by the chart's derivative; GTSAM does not either)
//
// The factor's A and b are already whitened (NoiseModelFactor::linearize), so the types take no noise model: J = A is
// copied bit for bit and the device rhs is b - A d, in the layout of linearize_kernel (kernels_factor.cu).  One thread
// per factor, SoA.  Algorithmic bytes per factor: LINEAR_PP3 idx 8 + record 360 + J 216 + b 24 = 608 B, LINEAR_PPP3
// 12 + 600 + 360 + 24 = 996 B.  A window holds a few thousand such factors, so a launch is bound by its latency, not by HBM.
//
// The sliding window's marginal (api.cu: dynoba_marginal_keep_points) exports the factors of its kept points with
// linear_gather_kernel and takes them out of the Schur marginal with linear_mask_kernel.
#include "internal.cuh"

namespace dynoba {

constexpr int LINF_THREADS = 128;     // as LIN_THREADS: the launch writes linearize_grid(n) partial sums

template <int T, bool WJ>
__global__ void __launch_bounds__(LINF_THREADS) linear_factor_kernel(DevBlock blk, DevVars v, double* __restrict__ partials,
                                                                     double* __restrict__ per_factor) {
  constexpr TypeInfo ti = type_info(T);
  constexpr int NP = ti.npose, JC = ti.jcols, NA = 3*JC;     // record: A [3][JC] | b [3] | lin poses [NP][12] | lin point [3]
  __shared__ double sh[LINF_THREADS/32];
  const int f = blockIdx.x*LINF_THREADS + threadIdx.x;
  double e = 0.0;
  if (f < blk.n) {
    auto rec = [&](int k) { return __ldg(blk.meas + (size_t)k*blk.stride + f); };
    double d[JC];
#pragma unroll
    for (int s = 0; s < NP; s++) {
      const int pos = __ldg(blk.idx + (size_t)s*blk.stride + f);
      Pose L, X;
#pragma unroll
      for (int k = 0; k < 9; k++) { L.R[k] = rec(NA + 3 + 12*s + k); X.R[k] = __ldg(v.pose + (size_t)k*v.np_stride + pos); }
#pragma unroll
      for (int k = 0; k < 3; k++) { L.t[k] = rec(NA + 3 + 12*s + 9 + k); X.t[k] = __ldg(v.pose + (size_t)(9 + k)*v.np_stride + pos); }
      se3_local(L, X, d + 6*s);
    }
    const int l = __ldg(blk.idx + (size_t)NP*blk.stride + f);
#pragma unroll
    for (int c = 0; c < 3; c++) d[6*NP + c] = __ldg(v.point + (size_t)c*v.nl_stride + l) - rec(NA + 3 + 12*NP + c);
#pragma unroll
    for (int r = 0; r < 3; r++) {
      double q = rec(NA + r);
#pragma unroll
      for (int c = 0; c < JC; c++) {
        const double a = rec(r*JC + c);
        q -= a*d[c];
        if (WJ) blk.J[(size_t)(r*JC + c)*blk.stride + f] = a;
      }
      if (WJ) blk.b[(size_t)r*blk.stride + f] = q;
      e += 0.5*q*q;
    }
    if (per_factor) per_factor[f] = e;
  }
  // deterministic CTA sum (fixed shuffle tree, warps in order), as the other factor kernels
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = e;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < LINF_THREADS/32; w++) t += sh[w]; partials[blockIdx.x] = t; }
}

int launch_linear_factors(const DevBlock& blk, const DevVars& v, bool with_jacobian, double* partials, double* per_factor,
                          cudaStream_t s) {
  if (blk.n == 0) return 0;
  const int grid = (blk.n + LINF_THREADS - 1)/LINF_THREADS;
  if (blk.type == F_LINEAR_PP3) {
    if (with_jacobian) linear_factor_kernel<F_LINEAR_PP3, true><<<grid, LINF_THREADS, 0, s>>>(blk, v, partials, per_factor);
    else linear_factor_kernel<F_LINEAR_PP3, false><<<grid, LINF_THREADS, 0, s>>>(blk, v, partials, per_factor);
  } else {
    if (with_jacobian) linear_factor_kernel<F_LINEAR_PPP3, true><<<grid, LINF_THREADS, 0, s>>>(blk, v, partials, per_factor);
    else linear_factor_kernel<F_LINEAR_PPP3, false><<<grid, LINF_THREADS, 0, s>>>(blk, v, partials, per_factor);
  }
  return 1;
}

// out[row0 + i] = [A | 0 | b] of the factor at sorted position pos[i]: 3 rows of LINEAR_EXPORT_COLS doubles, A in columns
// [0, jcols), b in the last column
__global__ void linear_gather_kernel(DevBlock blk, int jcols, const int* __restrict__ pos, int n, double* __restrict__ out) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = pos[i];
  double* o = out + (size_t)i*3*LINEAR_EXPORT_COLS;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < LINEAR_EXPORT_COLS - 1; c++) o[r*LINEAR_EXPORT_COLS + c] = c < jcols ? blk.J[(size_t)(r*jcols + c)*blk.stride + f] : 0.0;
    o[r*LINEAR_EXPORT_COLS + LINEAR_EXPORT_COLS - 1] = blk.b[(size_t)r*blk.stride + f];
  }
}
// zero the pose columns [0, pcols) and the rhs of the factors at sorted positions pos[]: they then add exactly 0 to S, to
// g_S and to the landmark's g_l, whatever their point columns hold
__global__ void linear_mask_kernel(DevBlock blk, int jcols, int pcols, const int* __restrict__ pos, int n) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = pos[i];
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < pcols; c++) blk.J[(size_t)(r*jcols + c)*blk.stride + f] = 0.0;
    blk.b[(size_t)r*blk.stride + f] = 0.0;
  }
}

int launch_linear_export(const DevBlock& blk, const int* pos, int n, double* out, cudaStream_t s) {
  if (n == 0) return 0;
  const TypeInfo ti = type_info(blk.type);
  linear_gather_kernel<<<(n + 127)/128, 128, 0, s>>>(blk, ti.jcols, pos, n, out);
  linear_mask_kernel<<<(n + 127)/128, 128, 0, s>>>(blk, ti.jcols, 6*ti.npose, pos, n);
  return 2;
}

}  // namespace dynoba
