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

namespace dynoba {

constexpr int NAV_THREADS = 128;
constexpr int IMU_WARPS = 4;                    // factors per CTA of the IMU kernels (one warp each)
constexpr int IMU_D = 15, IMU_JC = 30;

// SO(3) right Jacobian Jr(x) and its inverse [GTSAM-ext geometry/SO3.cpp ExpmapDerivative, LogmapDerivative]
__device__ void so3_jr(const double* x, double* J) {
  const double th2 = x[0]*x[0] + x[1]*x[1] + x[2]*x[2];
  double W[9], WW[9]; skew3(x, W); m3mul(W, W, WW);
  double a, b;
  if (th2 < 1e-10) { a = 0.5 - th2/24.0; b = 1.0/6.0 - th2/120.0; }
  else { const double th = sqrt(th2); a = (1.0 - cos(th))/th2; b = (th - sin(th))/(th2*th); }
  for (int i = 0; i < 9; i++) J[i] = -a*W[i] + b*WW[i];
  J[0] += 1; J[4] += 1; J[8] += 1;
}
__device__ void so3_jr_inv(const double* x, double* J) {
  const double th2 = x[0]*x[0] + x[1]*x[1] + x[2]*x[2];
  double W[9], WW[9]; skew3(x, W); m3mul(W, W, WW);
  double c;
  if (th2 < 1e-10) c = 1.0/12.0 + th2/720.0;
  else { const double th = sqrt(th2); c = 1.0/th2 - (1.0 + cos(th))/(2.0*th*sin(th)); }
  for (int i = 0; i < 9; i++) J[i] = 0.5*W[i] + c*WW[i];
  J[0] += 1; J[4] += 1; J[8] += 1;
}

// 3x3 block B (row-major) into J (IMU_JC columns) at (r0, c0), scaled by s
__device__ __forceinline__ void put3(double* J, int r0, int c0, const double* B, double s = 1.0) {
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) J[(r0 + i)*IMU_JC + c0 + j] = s*B[3*i + j];
}
__device__ __forceinline__ void m3t(const double* A, double* T) { for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) T[3*i + j] = A[3*j + i]; }

// unwhitened residual r[15] and, if J != nullptr, Jacobian J[15][30] (columns: pose_i | vel_i | pose_j | vel_j | bias_i | bias_j)
__device__ void imu_eval(const Pose& Xi, const double* vi, const Pose& Xj, const double* vj, const double* bi, const double* bj,
                         const double* z, double* r, double* J) {
  const double *dR = z, *dp = z + 9, *dv = z + 12, dt = z[15], *bh = z + 16;
  const double *JRw = z + 22, *JPa = z + 31, *JPw = z + 40, *JVa = z + 49, *JVw = z + 58, *g = z + 67;
  double dba[3], dbw[3], th[3];
  for (int k = 0; k < 3; k++) { dba[k] = bi[k] - bh[k]; dbw[k] = bi[3 + k] - bh[3 + k]; }
  m3vec(JRw, dbw, th);
  double Eth[9], Rc[9], phi[3], Ephi[9], Rp[9];
  so3_expmap(th, Eth); m3mul(dR, Eth, Rc); so3_logmap(Rc, phi);
  so3_expmap(phi, Ephi); m3mul(Xi.R, Ephi, Rp);
  double dPc[3], dVc[3], t1[3], t2[3], t3[3], t4[3];
  m3vec(JPa, dba, t1); m3vec(JPw, dbw, t2); m3vec(JVa, dba, t3); m3vec(JVw, dbw, t4);
  for (int k = 0; k < 3; k++) { dPc[k] = dp[k] + t1[k] + t2[k]; dVc[k] = dv[k] + t3[k] + t4[k]; }
  double Rtv[3], Rtg[3], xP[3], xV[3];
  m3tvec(Xi.R, vi, Rtv); m3tvec(Xi.R, g, Rtg);
  const double dt22 = 0.5*dt*dt;
  for (int k = 0; k < 3; k++) { xP[k] = dPc[k] + dt*Rtv[k] + dt22*Rtg[k]; xV[k] = dVc[k] + dt*Rtg[k]; }
  double RxP[3], RxV[3], pp[3], vp[3];
  m3vec(Xi.R, xP, RxP); m3vec(Xi.R, xV, RxV);
  for (int k = 0; k < 3; k++) { pp[k] = Xi.t[k] + RxP[k]; vp[k] = vi[k] + RxV[k]; }
  double E[9]; m3tmul(Rp, Xj.R, E);
  so3_logmap(E, r);
  double d[3];
  for (int k = 0; k < 3; k++) d[k] = Xj.t[k] - pp[k];
  m3tvec(Rp, d, r + 3);
  for (int k = 0; k < 3; k++) d[k] = vj[k] - vp[k];
  m3tvec(Rp, d, r + 6);
  for (int k = 0; k < 6; k++) r[9 + k] = bi[k] - bj[k];
  if (!J) return;
  for (int i = 0; i < IMU_D*IMU_JC; i++) J[i] = 0.0;
  double Jri[9], Jrt[9], EphiT[9], RpT[9], ET[9], A[9], Bm[9], C[9], S[9], JJ[9];
  so3_jr_inv(r, Jri); so3_jr(th, Jrt); m3t(Ephi, EphiT); m3t(Rp, RpT); m3t(E, ET);
  m3mul(Jrt, JRw, JJ);                                 // d(right tangent of R_p) / d(gyro bias)
  // rotation rows
  m3mul(Jri, ET, A); m3mul(A, EphiT, Bm); put3(J, 0, 0, Bm, -1.0);
  put3(J, 0, 9, Jri);
  m3mul(A, JJ, Bm); put3(J, 0, 21, Bm, -1.0);
  // position rows, velocity rows
  for (int q = 0; q < 2; q++) {
    const double* e = r + 3 + 3*q; const double* dc = q == 0 ? dPc : dVc;
    const double* Ja = q == 0 ? JPa : JVa; const double* Jw = q == 0 ? JPw : JVw;
    const int r0 = 3 + 3*q;
    skew3(e, S); m3mul(S, EphiT, A); skew3(dc, C); m3mul(EphiT, C, Bm);
    for (int i = 0; i < 9; i++) A[i] += Bm[i];
    put3(J, r0, 0, A);
    m3mul(EphiT, Ja, A); put3(J, r0, 18, A, -1.0);
    m3mul(S, JJ, A); m3mul(EphiT, Jw, Bm);
    for (int i = 0; i < 9; i++) A[i] -= Bm[i];
    put3(J, r0, 21, A);
  }
  put3(J, 3, 3, EphiT, -1.0);
  put3(J, 3, 6, RpT, -dt);
  put3(J, 3, 12, E);
  put3(J, 6, 6, RpT, -1.0);
  put3(J, 6, 15, RpT);
  for (int k = 0; k < 6; k++) { J[(9 + k)*IMU_JC + 18 + k] = 1.0; J[(9 + k)*IMU_JC + 24 + k] = -1.0; }
}

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
