// preint.cuh -- combined IMU preintegration (GTSAM 4.2.0 PreintegratedCombinedMeasurements with ManifoldPreintegration,
// GTSAM_TANGENT_PREINTEGRATION=OFF, no Coriolis) as __host__ __device__ code, so that tests/capi/preint_host.cu can build
// it for the host and kernels_preint.cu runs it one warp per frame interval.
//
// One sample (acc, omega, dt) [GTSAM-ext navigation/ManifoldPreintegration.cpp update, NavState.cpp update / retract,
// PreintegrationBase.cpp correctMeasurementsBySensorPose]:
//   a = acc - biasHat.acc,  w = omega - biasHat.gyro;  with body_P_sensor = (bRs, arm):
//     w <- bRs w,  a <- bRs a - [w]x [w]x arm   (the centrifugal term only when arm != 0)
//   NavState (R, p, v) of the interval so far:  incR = Exp(w dt),  b_v = R^T v
//     R' = R incR,  p' = p + R (dt b_v + dt^2/2 a),  v' = v + R (dt a)
//   A (9x9), B, C (9x3): derivatives of (R', p', v') in NavState's chart (R Exp(dR), p + R dp, v + R dv) w.r.t. the old
//   state, a and w:
//     A = [[incR^T, 0, 0], [-dt^2/2 incR^T [a]x, incR^T, dt incR^T], [-dt incR^T [a]x, 0, incR^T]]
//     B = [0; dt^2/2 incR^T; dt incR^T],  C = [Jr(w dt) dt; 0; 0]
//   with body_P_sensor:  C <- C bRs,  C += B D_a_w (arm != 0),  B <- B bRs
//   bias Jacobians, with the rotation R BEFORE the step and the corrected a, w:
//     D = -R [a]x delRdelBiasOmega
//     delRdelBiasOmega <- incR^T delRdelBiasOmega - Jr(w dt) dt
//     delPdelBiasAcc += dt delVdelBiasAcc - dt^2/2 R,   delPdelBiasOmega += dt delVdelBiasOmega + dt^2/2 D
//     delVdelBiasAcc -= dt R,                          delVdelBiasOmega += dt D
// The covariance step (preint_F, preint_noise) and the square-root information (preint_sqrt_info) are stated at their
// functions; preint_predict is PreintegrationBase::predict.
#pragma once
#include "se3.cuh"
#include "../../include/dynoba.h"

namespace dynoba {

constexpr int PI_REC = 70, PI_D = 15, PI_COV = 225, PI_FR = 9;   // record, Sigma side, Sigma, rows of F that are not I

// ManifoldPreintegration's state: deltaXij (R, p, v), deltaTij and the five bias Jacobians
struct PreintState {
  double R[9], p[3], v[3], T;
  double JRw[9], JPa[9], JPw[9], JVa[9], JVw[9];
};

DYN_HD void preint_reset(PreintState& s) {
  for (int i = 0; i < 9; i++) { s.R[i] = (i % 4 == 0); s.JRw[i] = s.JPa[i] = s.JPw[i] = s.JVa[i] = s.JVw[i] = 0.0; }
  for (int i = 0; i < 3; i++) s.p[i] = s.v[i] = 0.0;
  s.T = 0.0;
}

// SO(3) right Jacobian Jr(x): imu.cuh's so3_jr (series below theta^2 = 1e-10, 1 - cos as 2 sin^2(theta/2)).  Restated
// here because imu.cuh's functions have external linkage and may be included from one translation unit per binary.
DYN_HD void preint_jr(const double* x, double* J) {
  const double th2 = x[0]*x[0] + x[1]*x[1] + x[2]*x[2];
  double W[9], WW[9]; skew3(x, W); m3mul(W, W, WW);
  double a, b;
  if (th2 < 1e-10) { a = 0.5 - th2/24.0; b = 1.0/6.0 - th2/120.0; }
  else { const double th = sqrt(th2), s2 = sin(0.5*th); a = 2.0*s2*s2/th2; b = (th - sin(th))/(th2*th); }
  for (int i = 0; i < 9; i++) J[i] = -a*W[i] + b*WW[i];
  J[0] += 1; J[4] += 1; J[8] += 1;
}

// correctMeasurementsBySensorPose [GTSAM-ext PreintegrationBase.cpp]: a, w in place (sensor -> body frame) and the
// Jacobians of the corrected values w.r.t. the unbiased ones: Daa = bRs, Dww = bRs, Daw = 0 or, with a lever arm,
// -((w . arm) I + w arm^T) bRs + 2 arm u^T (u = the unbiased omega)
DYN_HD void preint_sensor_pose(const dynoba_imu_params& P, double* a, double* w, double* Daa, double* Daw, double* Dww) {
  const double* bRs = P.body_P_sensor; const double* arm = P.body_P_sensor + 9;
  double u[3] = { w[0], w[1], w[2] }, ua[3] = { a[0], a[1], a[2] };
  m3vec(bRs, u, w); m3vec(bRs, ua, a);
  for (int i = 0; i < 9; i++) { Daa[i] = bRs[i]; Dww[i] = bRs[i]; Daw[i] = 0.0; }
  if (arm[0] != 0.0 || arm[1] != 0.0 || arm[2] != 0.0) {
    double W[9], Wa[3], WWa[3]; skew3(w, W); m3vec(W, arm, Wa); m3vec(W, Wa, WWa);
    for (int k = 0; k < 3; k++) a[k] -= WWa[k];
    const double wdp = w[0]*arm[0] + w[1]*arm[1] + w[2]*arm[2];
    double M[9], MR[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) M[3*i + j] = (i == j ? wdp : 0.0) + w[i]*arm[j];
    m3mul(M, bRs, MR);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Daw[3*i + j] = -MR[3*i + j] + 2.0*arm[i]*u[j];
  }
}

// one integrateMeasurement step of the state; A[81], B[27], C[27] row-major
DYN_HD void preint_step(const dynoba_imu_params& P, const double* bh, const double* acc, const double* omega, double dt,
                        PreintState& s, double* A, double* B, double* C) {
  double a[3], w[3];
  for (int k = 0; k < 3; k++) { a[k] = acc[k] - bh[k]; w[k] = omega[k] - bh[3 + k]; }
  double Daa[9], Daw[9], Dww[9];
  if (P.has_body_P_sensor) preint_sensor_pose(P, a, w, Daa, Daw, Dww);
  const double dt22 = 0.5*dt*dt;
  double th[3] = { w[0]*dt, w[1]*dt, w[2]*dt }, incR[9], incRt[9], Jr[9];
  so3_expmap(th, incR); preint_jr(th, Jr);
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) incRt[3*i + j] = incR[3*j + i];
  // bias Jacobians first: they use the rotation before this step
  double Sa[9], D[9], T9[9];
  skew3(a, Sa); m3mul(s.R, Sa, T9); m3mul(T9, s.JRw, D);
  for (int i = 0; i < 9; i++) D[i] = -D[i];
  m3mul(incRt, s.JRw, T9);
  for (int i = 0; i < 9; i++) {
    s.JRw[i] = T9[i] - Jr[i]*dt;
    s.JPa[i] += s.JVa[i]*dt - dt22*s.R[i];
    s.JPw[i] += dt*s.JVw[i] + dt22*D[i];
    s.JVa[i] += -s.R[i]*dt;
    s.JVw[i] += D[i]*dt;
  }
  // NavState::update
  double bv[3], dP[3], dV[3], RdP[3], RdV[3], Rn[9];
  m3tvec(s.R, s.v, bv);
  for (int k = 0; k < 3; k++) { dP[k] = dt*bv[k] + dt22*a[k]; dV[k] = dt*a[k]; }
  m3vec(s.R, dP, RdP); m3vec(s.R, dV, RdV); m3mul(s.R, incR, Rn);
  for (int k = 0; k < 3; k++) { s.p[k] += RdP[k]; s.v[k] += RdV[k]; }
  for (int i = 0; i < 9; i++) s.R[i] = Rn[i];
  s.T += dt;
  // A, B, C
  double M[9]; m3mul(incRt, Sa, M);
  for (int i = 0; i < 81; i++) A[i] = 0.0;
  for (int i = 0; i < 27; i++) B[i] = C[i] = 0.0;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    const double r = incRt[3*i + j];
    A[9*i + j] = r; A[9*(3 + i) + 3 + j] = r; A[9*(6 + i) + 6 + j] = r;
    A[9*(3 + i) + 6 + j] = dt*r;
    A[9*(3 + i) + j] = -dt22*M[3*i + j]; A[9*(6 + i) + j] = -dt*M[3*i + j];
    B[3*(3 + i) + j] = dt22*r; B[3*(6 + i) + j] = dt*r;
    C[3*i + j] = Jr[3*i + j]*dt;
  }
  if (P.has_body_P_sensor) {
    double t[9];
    m3mul(C, Dww, t); for (int i = 0; i < 9; i++) C[i] = t[i];
    if (P.body_P_sensor[9] != 0.0 || P.body_P_sensor[10] != 0.0 || P.body_P_sensor[11] != 0.0)
      for (int r = 0; r < 3; r++) { m3mul(B + 9*r, Daw, t); for (int i = 0; i < 9; i++) C[9*r + i] += t[i]; }
    for (int r = 0; r < 3; r++) { m3mul(B + 9*r, Daa, t); for (int i = 0; i < 9; i++) B[9*r + i] = t[i]; }
  }
}

// The first nine rows of F [GTSAM-ext navigation/CombinedImuFactor.cpp integrateMeasurement], F9[9][15]:
//   F = [[A, F_nb], [0, I_6]],  F_nb[0:3, 3:6] = -C[0:3] (theta by gyro bias),  F_nb[3:6, 0:3] = -B[3:6],
//   F_nb[6:9, 0:3] = -B[6:9] (position and velocity by accelerometer bias), every other entry of F_nb 0.
DYN_HD void preint_F(const double* A, const double* B, const double* C, double* F9) {
  for (int i = 0; i < 9; i++) {
    for (int j = 0; j < 9; j++) F9[15*i + j] = A[9*i + j];
    for (int j = 0; j < 6; j++) F9[15*i + 9 + j] = 0.0;
  }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    F9[15*i + 12 + j] = -C[3*i + j];
    F9[15*(3 + i) + 9 + j] = -B[3*(3 + i) + j];
    F9[15*(6 + i) + 9 + j] = -B[3*(6 + i) + j];
  }
}

// X Y Z^T of 3x3 blocks, scaled by s
DYN_HD void m3_xyzt(const double* X, const double* Y, const double* Z, double s, double* O) {
  double t[9]; m3mul(X, Y, t);
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) O[3*i + j] = s*(t[3*i]*Z[3*j] + t[3*i + 1]*Z[3*j + 1] + t[3*i + 2]*Z[3*j + 2]);
}

// The injected noise Q[15][15] of one step [GTSAM-ext navigation/CombinedImuFactor.cpp integrateMeasurement, G_measCov_Gt],
// rows / columns (theta, p, v, bias_acc, bias_gyro), with thH = -C[0:3], pH = -B[3:6], vH = -B[6:9] and the "Init"
// Jacobians their negatives (the sign cancels in every product below), bI = biasAccOmegaInt / dt in 3x3 blocks:
//   Q_pp = pH (aCov/dt) pH^T + pH bI11 pH^T + dt iCov      Q_vv = vH (aCov/dt) vH^T + vH bI11 vH^T
//   Q_RR = thH (wCov/dt) thH^T + thH bI22 thH^T            Q_aa = dt biasAccCov,  Q_gg = dt biasOmegaCov
//   Q_vp = vH (aCov/dt) pH^T + vH bI11 pH^T = Q_pv^T       Q_vR = vH bI12 thH^T = Q_Rv^T,  Q_pR = pH bI12 thH^T = Q_Rp^T
DYN_HD void preint_noise(const dynoba_imu_params& P, const double* B, const double* C, double dt, double* Q) {
  const double* thH = C; const double* pH = B + 9; const double* vH = B + 18;
  double bI11[9], bI12[9], bI22[9], aC[9], wC[9], t[9], u[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    bI11[3*i + j] = P.bias_acc_omega_int[6*i + j]/dt; bI12[3*i + j] = P.bias_acc_omega_int[6*i + 3 + j]/dt;
    bI22[3*i + j] = P.bias_acc_omega_int[6*(3 + i) + 3 + j]/dt;
    aC[3*i + j] = P.accelerometer_cov[3*i + j]/dt; wC[3*i + j] = P.gyroscope_cov[3*i + j]/dt;
  }
  for (int i = 0; i < PI_COV; i++) Q[i] = 0.0;
  auto put = [&](int r0, int c0, const double* M, bool mirror) {
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
      Q[15*(r0 + i) + c0 + j] = M[3*i + j];
      if (mirror) Q[15*(c0 + j) + r0 + i] = M[3*i + j];
    }
  };
  m3_xyzt(pH, aC, pH, 1.0, t); m3_xyzt(pH, bI11, pH, 1.0, u);
  for (int i = 0; i < 9; i++) t[i] += u[i] + dt*P.integration_cov[i];
  put(3, 3, t, false);
  m3_xyzt(vH, aC, vH, 1.0, t); m3_xyzt(vH, bI11, vH, 1.0, u);
  for (int i = 0; i < 9; i++) t[i] += u[i];
  put(6, 6, t, false);
  m3_xyzt(thH, wC, thH, 1.0, t); m3_xyzt(thH, bI22, thH, 1.0, u);
  for (int i = 0; i < 9; i++) t[i] += u[i];
  put(0, 0, t, false);
  for (int i = 0; i < 9; i++) { t[i] = dt*P.bias_acc_cov[i]; u[i] = dt*P.bias_omega_cov[i]; }
  put(9, 9, t, false); put(12, 12, u, false);
  m3_xyzt(vH, aC, pH, 1.0, t); m3_xyzt(vH, bI11, pH, 1.0, u);
  for (int i = 0; i < 9; i++) t[i] += u[i];
  put(6, 3, t, true);
  m3_xyzt(vH, bI12, thH, 1.0, t); put(6, 0, t, true);
  m3_xyzt(pH, bI12, thH, 1.0, t); put(3, 0, t, true);
}

// Sigma <- F Sigma F^T + Q, lanes l = 0..nl-1 over the entries (the host passes 0, 1; the warp its lanes and __syncwarp()
// between the two phases).  F's last six rows are the identity, so only T = F9 Sigma (9 x 15) is formed:
//   phase 1:  T = F9 Sigma
//   phase 2:  Sigma[i][j] = T[i] . F9[j] + Q (i <= j < 9),  Sigma[i][j] = T[i][j] + Q (i < 9 <= j),  Sigma[i][j] += Q (9 <= i <= j),
//             and the lower triangle mirrored
DYN_HD void preint_cov_phase1(const double* F9, const double* S, double* T, int l, int nl) {
  for (int e = l; e < PI_FR*PI_D; e += nl) {
    const int i = e/PI_D, j = e - i*PI_D;
    double t = 0.0;
    for (int k = 0; k < PI_D; k++) t += F9[PI_D*i + k]*S[PI_D*k + j];
    T[e] = t;
  }
}
DYN_HD void preint_cov_phase2(const double* F9, const double* T, const double* Q, double* S, int l, int nl) {
  for (int e = l; e < PI_COV; e += nl) {
    const int i = e/PI_D, j = e - i*PI_D;
    if (j < i) continue;
    double x;
    if (j < PI_FR) { x = 0.0; for (int k = 0; k < PI_D; k++) x += T[PI_D*i + k]*F9[PI_D*j + k]; x += Q[e]; }
    else if (i < PI_FR) x = T[PI_D*i + j] + Q[e];
    else x = S[e] + Q[e];
    S[e] = x; S[PI_D*j + i] = x;
  }
}

// noiseModel::Gaussian::Covariance(Sigma) [GTSAM-ext linear/NoiseModel.cpp]: R upper triangular with a positive diagonal
// and R^T R = Sigma^-1 (GTSAM: LLT of Sigma.inverse(), U factor).  That R is unique; it is formed here as the inverse of
// the upper factor U of Sigma = U U^T (the Cholesky factorisation taken from the last row up): Sigma^-1 = U^-T U^-1 and
// U^-1 is upper triangular.  Returns DYNOBA_PREINT_NOT_PD, with R zeroed, when a pivot of U is not > 0 or not finite.
DYN_HD int preint_sqrt_info(const double* S, double* U, double* R) {
  const int n = PI_D;
  for (int i = 0; i < n*n; i++) { U[i] = 0.0; R[i] = 0.0; }
  for (int j = n - 1; j >= 0; j--) {
    double d = S[n*j + j];
    for (int k = j + 1; k < n; k++) d -= U[n*j + k]*U[n*j + k];
    if (!(d > 0.0) || !(d < INFINITY)) { for (int i = 0; i < n*n; i++) U[i] = 0.0; return DYNOBA_PREINT_NOT_PD; }
    const double u = sqrt(d);
    U[n*j + j] = u;
    for (int i = 0; i < j; i++) {
      double x = S[n*i + j];
      for (int k = j + 1; k < n; k++) x -= U[n*i + k]*U[n*j + k];
      U[n*i + j] = x/u;
    }
  }
  for (int j = 0; j < n; j++) {
    R[n*j + j] = 1.0/U[n*j + j];
    for (int i = j - 1; i >= 0; i--) {
      double x = 0.0;
      for (int k = i + 1; k <= j; k++) x += U[n*i + k]*R[n*k + j];
      R[n*i + j] = -x/U[n*i + i];
    }
  }
  for (int i = 0; i < n*n; i++) if (!(fabs(R[i]) < INFINITY)) { for (int k = 0; k < n*n; k++) R[k] = 0.0; return DYNOBA_PREINT_NOT_PD; }
  return DYNOBA_PREINT_OK;
}

// the 70-double COMBINED_IMU15 record (include/dynoba.h) of the state
DYN_HD void preint_record(const PreintState& s, const double* bh, const double* g, double* z) {
  for (int i = 0; i < 9; i++) { z[i] = s.R[i]; z[22 + i] = s.JRw[i]; z[31 + i] = s.JPa[i]; z[40 + i] = s.JPw[i];
                                z[49 + i] = s.JVa[i]; z[58 + i] = s.JVw[i]; }
  for (int k = 0; k < 3; k++) { z[9 + k] = s.p[k]; z[12 + k] = s.v[k]; z[67 + k] = g[k]; }
  z[15] = s.T;
  for (int k = 0; k < 6; k++) z[16 + k] = bh[k];
}

// PreintegrationBase::predict(NavState(Xi, vi), bias_i) of a record [GTSAM-ext navigation/PreintegrationBase.cpp,
// ManifoldPreintegration.cpp biasCorrectedDelta, NavState.cpp correctPIM / retract], no Coriolis:
//   phi = Log(dR Exp(JRw dbw)),  dPc = dp + JPa dba + JPw dbw,  dVc = dv + JVa dba + JVw dbw
//   xP = dPc + dt R_i^T v_i + dt^2/2 R_i^T g,  xV = dVc + dt R_i^T g
//   R_j = R_i Exp(phi),  p_j = p_i + R_i xP,  v_j = v_i + R_i xV
DYN_HD void preint_predict(const double* z, const Pose& Xi, const double* vi, const double* bi, Pose& Xj, double* vj) {
  const double *dR = z, *dp = z + 9, *dv = z + 12, dt = z[15], *bh = z + 16;
  const double *JRw = z + 22, *JPa = z + 31, *JPw = z + 40, *JVa = z + 49, *JVw = z + 58, *g = z + 67;
  double dba[3], dbw[3], th[3], Eth[9], Rc[9], phi[3], Ephi[9];
  for (int k = 0; k < 3; k++) { dba[k] = bi[k] - bh[k]; dbw[k] = bi[3 + k] - bh[3 + k]; }
  m3vec(JRw, dbw, th); so3_expmap(th, Eth); m3mul(dR, Eth, Rc); so3_logmap(Rc, phi);
  so3_expmap(phi, Ephi); m3mul(Xi.R, Ephi, Xj.R);
  double t1[3], t2[3], t3[3], t4[3], Rtv[3], Rtg[3], xP[3], xV[3], RxP[3], RxV[3];
  m3vec(JPa, dba, t1); m3vec(JPw, dbw, t2); m3vec(JVa, dba, t3); m3vec(JVw, dbw, t4);
  m3tvec(Xi.R, vi, Rtv); m3tvec(Xi.R, g, Rtg);
  const double dt22 = 0.5*dt*dt;
  for (int k = 0; k < 3; k++) {
    xP[k] = dp[k] + t1[k] + t2[k] + dt*Rtv[k] + dt22*Rtg[k];
    xV[k] = dv[k] + t3[k] + t4[k] + dt*Rtg[k];
  }
  m3vec(Xi.R, xP, RxP); m3vec(Xi.R, xV, RxV);
  for (int k = 0; k < 3; k++) { Xj.t[k] = Xi.t[k] + RxP[k]; vj[k] = vi[k] + RxV[k]; }
}

}  // namespace dynoba
