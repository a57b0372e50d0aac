// imu.cuh -- the CombinedImuFactor residual and Jacobian (kernels_imu.cu's header comment states the mathematics) and the
// SO(3) right Jacobian it uses, as __host__ __device__ code so that tests/capi/imu_host.cu can build them for the host.
// The three functions are deliberately not forceinline: the compiler decides their inlining into imu_kernel as it did
// when they lived in kernels_imu.cu.  Each binary includes this header from one translation unit.
#pragma once
#include "se3.cuh"

namespace dynoba {

constexpr int IMU_D = 15, IMU_JC = 30;

// SO(3) right Jacobian Jr(x) and its inverse [GTSAM-ext geometry/SO3.cpp ExpmapDerivative, LogmapDerivative].
// 1 - cos(th) is formed as 2 sin^2(th/2), as so3_expmap does: the direct difference cancels to a relative error of
// eps/th^2 (1e-7 at th = 1e-5, where the series hands over).
__host__ __device__ void so3_jr(const double* x, double* J) {
  const double th2 = x[0]*x[0] + x[1]*x[1] + x[2]*x[2];
  double W[9], WW[9]; skew3(x, W); m3mul(W, W, WW);
  double a, b;
  if (th2 < 1e-10) { a = 0.5 - th2/24.0; b = 1.0/6.0 - th2/120.0; }
  else { const double th = sqrt(th2), s2 = sin(0.5*th); a = 2.0*s2*s2/th2; b = (th - sin(th))/(th2*th); }
  for (int i = 0; i < 9; i++) J[i] = -a*W[i] + b*WW[i];
  J[0] += 1; J[4] += 1; J[8] += 1;
}
__host__ __device__ void so3_jr_inv(const double* x, double* J) {
  const double th2 = x[0]*x[0] + x[1]*x[1] + x[2]*x[2];
  double W[9], WW[9]; skew3(x, W); m3mul(W, W, WW);
  double c;
  if (th2 < 1e-10) c = 1.0/12.0 + th2/720.0;
  else { const double th = sqrt(th2); c = 1.0/th2 - (1.0 + cos(th))/(2.0*th*sin(th)); }
  for (int i = 0; i < 9; i++) J[i] = 0.5*W[i] + c*WW[i];
  J[0] += 1; J[4] += 1; J[8] += 1;
}

// 3x3 block B (row-major) into J (IMU_JC columns) at (r0, c0), scaled by s
DYN_HD void put3(double* J, int r0, int c0, const double* B, double s = 1.0) {
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) J[(r0 + i)*IMU_JC + c0 + j] = s*B[3*i + j];
}
DYN_HD void m3t(const double* A, double* T) { for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) T[3*i + j] = A[3*j + i]; }

// unwhitened residual r[15] and, if J != nullptr, Jacobian J[15][30] (columns: pose_i | vel_i | pose_j | vel_j | bias_i | bias_j)
__host__ __device__ void imu_eval(const Pose& Xi, const double* vi, const Pose& Xj, const double* vj, const double* bi,
                                  const double* bj, const double* z, double* r, double* J) {
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

}  // namespace dynoba
