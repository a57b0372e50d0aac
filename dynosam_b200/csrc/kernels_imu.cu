// kernels_imu.cu -- the visual-inertial factors (PRIOR_VEL3, PRIOR_BIAS6, COMBINED_IMU15) and the navigation variables
// (velocity, IMU bias) of the reduced system.
//
// Velocities and biases are pose-like: they chain from frame to frame, so they are not eliminated per landmark but join
// the banded reduced system, each in a 6-wide block at its own position.  A velocity uses the first three scalars of its
// block; the other three are inert (unit diagonal, zero right-hand side, never damped, never retracted), so every band
// / cell / spike path addresses 6-wide blocks exactly as for poses.  Their values live in the pose SoA at their
// position (rows 0-2 velocity, rows 0-5 bias [accelerometer | gyroscope], the other rows zero).
//
// CombinedImuFactor (GTSAM 4.2.0, ManifoldPreintegration, no Coriolis) [GTSAM-ext navigation/CombinedImuFactor.cpp,
// PreintegrationBase.cpp, ManifoldPreintegration.cpp, NavState.cpp]:
//   dba = b_i.acc - biasHat.acc,  dbw = b_i.gyro - biasHat.gyro,  th = delRdelBiasOmega dbw
//   phi = Log(dR Exp(th)),  dPc = dp + delPdelBiasAcc dba + delPdelBiasOmega dbw,  dVc = dv + delVdelBiasAcc dba + delVdelBiasOmega dbw
//   correctPIM:  xP = dPc + dt R_i^T v_i + dt^2/2 R_i^T g,  xV = dVc + dt R_i^T g
//   predict = NavState(R_i, p_i, v_i).retract([phi, xP, xV]):  R_p = R_i Exp(phi), p_p = p_i + R_i xP, v_p = v_i + R_i xV
//   r = [Log(R_p^T R_j), R_p^T (p_j - p_p), R_p^T (v_j - v_p), b_i - b_j]   (traits<ConstantBias>::Between(b_j, b_i))
// The Jacobians below are the closed-form derivatives of r w.r.t. Pose3 retract (T Exp(xi)), the nav-frame velocities
// and the bias vectors -- what GTSAM's chain of H1..H6 evaluates.  Whitening is by the full square-root information R
// of noiseModel::Gaussian: r_w = R r, J_w = R J.
#include "internal.cuh"
#include "imu.cuh"

namespace dynoba {

constexpr int NAV_THREADS = 128;
constexpr int IMU_WARPS = 4;                    // factors per CTA of the IMU kernels (one warp each)

__device__ __forceinline__ double warp_sum_d(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// One warp per COMBINED_IMU15 factor: the record and R are staged in shared memory, lane 0 evaluates r and J (the 3x3
// algebra is serial), the warp whitens (R J: 450 dot products of length 15) and stores the SoA J / b tiles.  Lane 0
// doing the chain alone (240 registers) and the per-factor SoA stores (one row per lane, uncoalesced) are deliberate:
// a graph has one IMU factor per frame pair, so the kernel is a few microseconds per thousand factors (DESIGN.md §1)
// and spreading the 3x3 chain over lanes would buy nothing measurable.
// partials[blockIdx.x] = sum of the CTA's 0.5 |r_w|^2;  per_factor (error sweep) gets each factor's error.
struct ImuStage { double z[IMU_MEAS]; double R[IMU_SQRT_INFO]; double r[IMU_D]; double J[IMU_D*IMU_JC]; };
template <bool WJ>
__global__ void __launch_bounds__(IMU_WARPS*32) imu_kernel(DevBlock blk, DevVars v, double* __restrict__ partials,
                                                          double* __restrict__ per_factor) {
  __shared__ ImuStage st[IMU_WARPS];
  __shared__ double sh[IMU_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x*IMU_WARPS + warp;
  double e = 0.0;
  if (f < blk.n) {
    ImuStage& S = st[warp];
    for (int k = lane; k < IMU_MEAS; k += 32) S.z[k] = blk.meas[(size_t)k*blk.stride + f];
    for (int k = lane; k < IMU_SQRT_INFO; k += 32) S.R[k] = blk.isig[(size_t)k*blk.stride + f];
    __syncwarp();
    if (lane == 0) {
      int p[6];
      for (int k = 0; k < 6; k++) p[k] = blk.idx[(size_t)k*blk.stride + f];
      Pose Xi, Xj; double vi[3], vj[3], bi[6], bj[6];
      for (int k = 0; k < 9; k++) { Xi.R[k] = v.pose[(size_t)k*v.np_stride + p[0]]; Xj.R[k] = v.pose[(size_t)k*v.np_stride + p[2]]; }
      for (int k = 0; k < 3; k++) {
        Xi.t[k] = v.pose[(size_t)(9 + k)*v.np_stride + p[0]]; Xj.t[k] = v.pose[(size_t)(9 + k)*v.np_stride + p[2]];
        vi[k] = v.pose[(size_t)k*v.np_stride + p[1]]; vj[k] = v.pose[(size_t)k*v.np_stride + p[3]];
      }
      for (int k = 0; k < 6; k++) { bi[k] = v.pose[(size_t)k*v.np_stride + p[4]]; bj[k] = v.pose[(size_t)k*v.np_stride + p[5]]; }
      imu_eval(Xi, vi, Xj, vj, bi, bj, S.z, S.r, WJ ? S.J : nullptr);
    }
    __syncwarp();
    double rw = 0.0;
    if (lane < IMU_D) for (int k = 0; k < IMU_D; k++) rw += S.R[lane*IMU_D + k]*S.r[k];
    if (WJ) {
      for (int q = lane; q < IMU_D*IMU_JC; q += 32) {
        const int row = q/IMU_JC, col = q - row*IMU_JC;
        double s = 0.0;
        for (int k = 0; k < IMU_D; k++) s += S.R[row*IMU_D + k]*S.J[k*IMU_JC + col];
        blk.J[(size_t)q*blk.stride + f] = s;
      }
      if (lane < IMU_D) blk.b[(size_t)lane*blk.stride + f] = -rw;
    }
    e = warp_sum_d(0.5*rw*rw);
    if (per_factor && lane == 0) per_factor[f] = e;
  }
  if (lane == 0) sh[warp] = e;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < IMU_WARPS; w++) t += sh[w]; partials[blockIdx.x] = t; }
}

// PriorFactor<Vector3> / PriorFactor<ConstantBias>: e = x - prior, H = I, Isotropic or Diagonal noise.  One thread per factor.
template <int D, bool WJ>
__global__ void __launch_bounds__(NAV_THREADS) vec_prior_kernel(DevBlock blk, DevVars v, double* __restrict__ partials,
                                                               double* __restrict__ per_factor) {
  __shared__ double sh[NAV_THREADS];
  const int f = blockIdx.x*NAV_THREADS + threadIdx.x;
  double e = 0.0;
  if (f < blk.n) {
    const int p = blk.idx[f];
    for (int k = 0; k < D; k++) {
      const double is = blk.isig[(size_t)(blk.sigma_dim == 1 ? 0 : k)*blk.stride + f];
      const double rk = (v.pose[(size_t)k*v.np_stride + p] - blk.meas[(size_t)k*blk.stride + f])*is;
      if (WJ) {
        for (int c = 0; c < D; c++) blk.J[(size_t)(k*D + c)*blk.stride + f] = c == k ? is : 0.0;
        blk.b[(size_t)k*blk.stride + f] = -rk;
      }
      e += 0.5*rk*rk;
    }
    if (per_factor) per_factor[f] = e;
  }
  sh[threadIdx.x] = e;
  __syncthreads();
  for (int o = NAV_THREADS/2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) partials[blockIdx.x] = sh[0];
}

int nav_grid(int type, int n) {
  return type == F_COMBINED_IMU15 ? (n + IMU_WARPS - 1)/IMU_WARPS : (n + NAV_THREADS - 1)/NAV_THREADS;
}

static int launch_nav(const DevBlock& blk, const DevVars& v, double* partials, double* per_factor, bool wj, cudaStream_t s) {
  if (blk.n == 0) return 0;
  const int grid = nav_grid(blk.type, blk.n);
  if (blk.type == F_COMBINED_IMU15) {
    if (wj) imu_kernel<true><<<grid, IMU_WARPS*32, 0, s>>>(blk, v, partials, nullptr);
    else imu_kernel<false><<<grid, IMU_WARPS*32, 0, s>>>(blk, v, partials, per_factor);
  } else if (blk.type == F_PRIOR_VEL3) {
    if (wj) vec_prior_kernel<3, true><<<grid, NAV_THREADS, 0, s>>>(blk, v, partials, nullptr);
    else vec_prior_kernel<3, false><<<grid, NAV_THREADS, 0, s>>>(blk, v, partials, per_factor);
  } else {
    if (wj) vec_prior_kernel<6, true><<<grid, NAV_THREADS, 0, s>>>(blk, v, partials, nullptr);
    else vec_prior_kernel<6, false><<<grid, NAV_THREADS, 0, s>>>(blk, v, partials, per_factor);
  }
  return 1;
}
int launch_nav_linearize(const DevBlock& blk, const DevVars& v, double* partials, cudaStream_t s) {
  return launch_nav(blk, v, partials, nullptr, true, s);
}
int launch_nav_error(const DevBlock& blk, const DevVars& v, double* partials, double* per_factor, cudaStream_t s) {
  return launch_nav(blk, v, partials, per_factor, false, s);
}

// J^T J and J^T b of the navigation factor types into S / g_S.  One warp per factor, J and b staged in shared memory;
// lanes over the columns (rhs) and the column pairs of the lower block triangle (21 variable pairs of the IMU factor).
__device__ __forceinline__ int nav_slot(const TypeInfo& ti, int q) {
  int k = 0;
  for (int s = 1; s < ti.arity; s++) if (q >= ti.coloff[s]) k = s;
  return k;
}
__global__ void __launch_bounds__(IMU_WARPS*32) nav_factors_kernel(DevBlock blk, DevBand B) {
  __shared__ double sJ[IMU_WARPS][IMU_D*IMU_JC + IMU_D];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x*IMU_WARPS + warp;
  if (f >= blk.n) return;
  const TypeInfo ti = type_info(blk.type);
  const int D = ti.dim, JC = ti.jcols, ne = D*JC;
  double* J = sJ[warp]; double* bb = J + ne;
  for (int q = lane; q < ne; q += 32) J[q] = blk.J[(size_t)q*blk.stride + f];
  for (int q = lane; q < D; q += 32) bb[q] = blk.b[(size_t)q*blk.stride + f];
  __syncwarp();
  for (int q = lane; q < JC; q += 32) {
    const int k = nav_slot(ti, q), a = blk.idx[(size_t)k*blk.stride + f];
    double g = 0.0;
    for (int r = 0; r < D; r++) g += J[r*JC + q]*bb[r];
    red_add(rhs_at(B, a*6 + q - ti.coloff[k]), g);
  }
  for (int e = lane; e < JC*JC; e += 32) {
    const int q1 = e/JC, q2 = e - q1*JC;
    const int k1 = nav_slot(ti, q1), k2 = nav_slot(ti, q2);
    if (k2 > k1 || (k1 == k2 && q2 > q1)) continue;
    const int a = blk.idx[(size_t)k1*blk.stride + f], b = blk.idx[(size_t)k2*blk.stride + f];
    const int c = q1 - ti.coloff[k1], c2 = q2 - ti.coloff[k2];
    double m = 0.0;
    for (int r = 0; r < D; r++) m += J[r*JC + q1]*J[r*JC + q2];
    const BandBlockRef cref = band_block_ref(B, (a > b ? a : b)*6, (a < b ? a : b)*6);
    const int row = a*6 + c, col = b*6 + c2;
    if (a > b || k1 == k2) red_add(band_block_at(B, cref, row, col), m);
    else if (a < b) red_add(band_block_at(B, cref, col, row), m);
    else { const int hi = row > col ? row : col, lo = row > col ? col : row;
           red_add(band_block_at(B, cref, hi, lo), c == c2 ? 2.0*m : m); }
  }
}
int launch_nav_factors(const DevBlock& blk, const DevBand& B, cudaStream_t s) {
  if (blk.n == 0) return 0;
  nav_factors_kernel<<<(blk.n + IMU_WARPS - 1)/IMU_WARPS, IMU_WARPS*32, 0, s>>>(blk, B);
  return 1;
}

// the navigation factors' share of g^T delta:  0.5 * b^T (A delta_p).  One thread per factor, grid (n + 127)/128.
__global__ void __launch_bounds__(NAV_THREADS) nav_model_kernel(DevBlock blk, DevBand B, double* __restrict__ partials) {
  __shared__ double sh[NAV_THREADS];
  const int f = blockIdx.x*blockDim.x + threadIdx.x;
  double q = 0;
  if (f < blk.n) {
    const TypeInfo ti = type_info(blk.type);
    for (int r = 0; r < ti.dim; r++) {
      double u = 0;
      for (int k = 0; k < ti.arity; k++) {
        const int a = blk.idx[(size_t)k*blk.stride + f], n = class_dim(ti.cls[k]);
        for (int c = 0; c < n; c++) u += blk.J[(size_t)(r*ti.jcols + ti.coloff[k] + c)*blk.stride + f]*B.dp[a*6 + c];
      }
      q += blk.b[(size_t)r*blk.stride + f]*u;
    }
    q *= 0.5;
  }
  sh[threadIdx.x] = q;
  __syncthreads();
  for (int o = NAV_THREADS/2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) partials[blockIdx.x] = sh[0];
}
int launch_nav_model(const DevBlock& blk, const DevBand& B, double* partials, cudaStream_t s) {
  if (blk.n == 0) return 0;
  nav_model_kernel<<<(blk.n + NAV_THREADS - 1)/NAV_THREADS, NAV_THREADS, 0, s>>>(blk, B, partials);
  return 1;
}

// values.retract(delta) of the navigation variables: vector addition.  Runs after the pose retract, which has written
// an (unused) SE(3) retraction at these positions: every row is rewritten.
__global__ void nav_retract_kernel(DevVars cur, DevVars cand, const double* __restrict__ dp, const int2* __restrict__ nav, int n) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = nav[i].x, d = nav[i].y;
  for (int k = 0; k < 12; k++) {
    const size_t o = (size_t)k*cur.np_stride + p;
    cand.pose[o] = k < d ? cur.pose[o] + dp[p*6 + k] : cur.pose[o];
  }
}
int launch_nav_retract(const DevVars& cur, const DevVars& cand, const DevBand& B, const int2* nav, int n, cudaStream_t s) {
  if (n == 0) return 0;
  nav_retract_kernel<<<(n + 127)/128, 128, 0, s>>>(cur, cand, B.dp, nav, n);
  return 1;
}

// unit diagonal on the three inert scalars of every velocity block (after band_clear, which wrote lambda there)
__global__ void nav_inert_kernel(DevBand B, const int2* __restrict__ nav, int n) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= 3*n) return;
  const int2 e = nav[i/3];
  if (e.y != 3) return;
  const int s = e.x*6 + 3 + i%3;
  *band_at(B, s, s) = 1.0;
}
int launch_nav_inert(const DevBand& B, const int2* nav, int n, cudaStream_t s) {
  if (n == 0) return 0;
  nav_inert_kernel<<<(3*n + 127)/128, 128, 0, s>>>(B, nav, n);
  return 1;
}

}  // namespace dynoba
