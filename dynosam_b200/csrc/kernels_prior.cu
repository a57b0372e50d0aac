// kernels_prior.cu -- dense quadratic prior over pose-like variables: the device side of gtsam::LinearContainerFactor
// holding a HessianFactor, which is how the reference's sliding-window optimiser carries the information of the
// marginalised variables into the next window (dynosam_opt/src/SlidingWindowOptimization.cc:67-121,165-190:
// CalculateMarginalFactors -> LinearContainerFactor::ConvertLinearGraph).
//
//   error(x)     = 1/2 d^T G d - g^T d + 1/2 f,   d_i = localCoordinates(lin_i, x_i)
//   linearize(x) = HessianFactor(G, g - G d, f + d^T G d - 2 d^T g)              [GTSAM-ext LinearContainerFactor::linearize]
// with d_i = Logmap(lin_i^-1 x_i) for a Pose3 slot and x_i - lin_i for a velocity (Vector3) or a bias (ConstantBias,
// [acc; gyro]) slot, as Values::localCoordinates takes them.  The factor adds G to the reduced system and (g - G d) to its
// right-hand side; G never changes.  Tangent scalar r of the prior sits at solver scalar P.sidx[r] (a velocity slot uses
// the first three scalars of its 6-wide block: the inert three are never touched).  A prior couples a few dozen
// variables: one CTA per prior.
#include "internal.cuh"
#include "se3.cuh"

namespace dynoba {

// d, gcur = g - G d, error -> partial[0]  (store: keep d and gcur for the solve of this linearisation)
__global__ void __launch_bounds__(256) prior_eval_kernel(DevPrior P, DevVars v, double* __restrict__ partial, int store) {
  extern __shared__ double sm[];                  // [dim] d | [256] reduction
  const int dim = P.dim;
  double* d = sm; double* red = sm + dim;
  for (int i = threadIdx.x; i < P.n; i += blockDim.x) {
    const int4 s = P.slot[i];                     // kind, solver position, first lin element, first tangent scalar
    if (s.x == DYNOBA_POSE6) {
      Pose L, X; double xi[6];
      for (int k = 0; k < 9; k++) { L.R[k] = P.lin[s.z + k]; X.R[k] = v.pose[(size_t)k*v.np_stride + s.y]; }
      for (int k = 0; k < 3; k++) { L.t[k] = P.lin[s.z + 9 + k]; X.t[k] = v.pose[(size_t)(9 + k)*v.np_stride + s.y]; }
      se3_local(L, X, xi);
      for (int k = 0; k < 6; k++) d[s.w + k] = xi[k];
    } else {                                      // vector spaces: rows 0..w-1 of the pose SoA
      const int w = s.x == DYNOBA_VEL3 ? 3 : 6;
      for (int k = 0; k < w; k++) d[s.w + k] = v.pose[(size_t)k*v.np_stride + s.y] - P.lin[s.z + k];
    }
  }
  __syncthreads();
  double e = 0.0;
  for (int r = threadIdx.x; r < dim; r += blockDim.x) {
    double gd = 0.0;
    for (int c = 0; c < dim; c++) gd += P.G[(size_t)r*dim + c]*d[c];
    e += d[r]*(0.5*gd - P.g[r]);
    if (store) { P.gcur[r] = P.g[r] - gd; P.delta[r] = d[r]; }
  }
  red[threadIdx.x] = e;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) partial[0] = red[0] + 0.5*P.f;
}
// S += G, g_S += gcur  (lower triangle of S in solver positions)
__global__ void prior_accum_kernel(DevPrior P, DevBand B) {
  const int dim = P.dim;
  for (int e = blockIdx.x*blockDim.x + threadIdx.x; e < dim*dim; e += gridDim.x*blockDim.x) {
    const int r = e/dim, c = e - r*dim;
    const int i = P.sidx[r], j = P.sidx[c];
    if (i > j || (i == j && r == c)) red_add(band_at(B, i, j), P.G[(size_t)r*dim + c]);
    // (two different prior slots on one variable would need G + G^T here; the entry points reject repeated variables)
  }
  for (int r = blockIdx.x*blockDim.x + threadIdx.x; r < dim; r += gridDim.x*blockDim.x) red_add(rhs_at(B, P.sidx[r]), P.gcur[r]);
}
// the prior's share of the linearised cost decrease: 1/2 gcur^T dp
__global__ void __launch_bounds__(256) prior_model_kernel(DevPrior P, DevBand B, double* __restrict__ partial) {
  __shared__ double red[256];
  double q = 0.0;
  for (int r = threadIdx.x; r < P.dim; r += blockDim.x) q += 0.5*P.gcur[r]*B.dp[P.sidx[r]];
  red[threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) partial[0] = red[0];
}

int launch_prior_eval(const DevPrior& P, const DevVars& v, double* partial, int store, cudaStream_t s) {
  prior_eval_kernel<<<1, 256, (size_t)(P.dim + 256)*sizeof(double), s>>>(P, v, partial, store);
  return 1;
}
int launch_prior_accum(const DevPrior& P, const DevBand& B, cudaStream_t s) {
  prior_accum_kernel<<<std::min(device_sm_count(), (P.dim*P.dim + 255)/256), 256, 0, s>>>(P, B);
  return 1;
}
int launch_prior_model(const DevPrior& P, const DevBand& B, double* partial, cudaStream_t s) {
  prior_model_kernel<<<1, 256, 0, s>>>(P, B, partial);
  return 1;
}

}  // namespace dynoba
