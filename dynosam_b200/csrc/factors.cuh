// factors.cuh -- residual + Jacobian of every factor on the hot path (SURVEY.md 8a rows a3-a9, a15) as
// closed-form device functions.  Each function cites the reference code it must agree with; the reference's
// Adjoint chain rules (HybridFormulationFactors.cc:37-135) are replaced by their closed forms, which
// tests/test_oracle_kat.py::test_hybrid_closed_form_matches_chain pins against the literal chain.
#pragma once
#include "se3.cuh"

namespace dynoba {

enum : int {
  F_PRIOR6 = 0, F_BETWEEN6 = 1, F_POSE2POINT3 = 2, F_STEREO3 = 3, F_TERNARY3 = 4, F_HYBRID3 = 5,
  F_HYBRID_STEREO3 = 6, F_MOTIONPOSE3 = 7, F_SMOOTH_HYBRID6 = 8, F_SMOOTH_POSE6 = 9, F_FLOWPROJ2 = 10,
  F_PRIOR_VEL3 = 11, F_PRIOR_BIAS6 = 12, F_COMBINED_IMU15 = 13, F_LINEAR_PP3 = 14, F_LINEAR_PPP3 = 15,
  F_NUM_TYPES = 16
};
// VC_VEL / VC_BIAS: the navigation variables of the visual-inertial graphs.  Like poses they live in the reduced system,
// each in a 6-wide block (a velocity's last three scalars are inert), and are stored in the pose SoA at their position.
enum : int { VC_POSE = 0, VC_POINT = 1, VC_FLOW = 2, VC_VEL = 3, VC_BIAS = 4 };
__host__ __device__ constexpr bool is_poselike(int c) { return c == VC_POSE || c == VC_VEL || c == VC_BIAS; }
__host__ __device__ constexpr bool is_nav_type(int t) { return t == F_PRIOR_VEL3 || t == F_PRIOR_BIAS6 || t == F_COMBINED_IMU15; }
// linearised landmark factors (gtsam::LinearContainerFactor holding a 3-row JacobianFactor): kernels_linear.cu
__host__ __device__ constexpr bool is_linear_type(int t) { return t == F_LINEAR_PP3 || t == F_LINEAR_PPP3; }
constexpr int IMU_MEAS = 70;       // meas record of COMBINED_IMU15 (include/dynoba.h)
constexpr int IMU_SQRT_INFO = 225; // its 15 x 15 square-root information, row-major
constexpr int LINEAR_PP3_MEAS = 45;  // A (3 x 9) | b (3) | lin pose (12) | lin point (3)
constexpr int LINEAR_PPP3_MEAS = 75; // A (3 x 15) | b (3) | lin poses (2 x 12) | lin point (3)

// static type tables (host + device constexpr)
struct TypeInfo {
  int arity, dim, meas, jcols, npose, nlmk, ldim;
  int cls[6];      // variable class per key slot
  int coloff[6];   // first Jacobian column of the slot
  bool needs_aux;
};
__host__ __device__ constexpr TypeInfo type_info(int t) {
  switch (t) {
    case F_PRIOR6:         return { 1, 6, 12, 6, 1, 0, 0, { VC_POSE, -1, -1, -1 }, { 0, 0, 0, 0 }, false };
    case F_BETWEEN6:       return { 2, 6, 12, 12, 2, 0, 0, { VC_POSE, VC_POSE, -1, -1 }, { 0, 6, 0, 0 }, false };
    case F_POSE2POINT3:    return { 2, 3, 3, 9, 1, 1, 3, { VC_POSE, VC_POINT, -1, -1 }, { 0, 6, 0, 0 }, false };
    case F_STEREO3:        return { 2, 3, 3, 9, 1, 1, 3, { VC_POSE, VC_POINT, -1, -1 }, { 0, 6, 0, 0 }, false };
    case F_TERNARY3:       return { 3, 3, 0, 12, 1, 2, 3, { VC_POINT, VC_POINT, VC_POSE, -1 }, { 0, 3, 6, 0 }, false };
    case F_HYBRID3:        return { 3, 3, 3, 15, 2, 1, 3, { VC_POSE, VC_POSE, VC_POINT, -1 }, { 0, 6, 12, 0 }, true };
    case F_HYBRID_STEREO3: return { 3, 3, 3, 15, 2, 1, 3, { VC_POSE, VC_POSE, VC_POINT, -1 }, { 0, 6, 12, 0 }, true };
    case F_MOTIONPOSE3:    return { 4, 3, 0, 18, 2, 2, 3, { VC_POINT, VC_POINT, VC_POSE, VC_POSE }, { 0, 3, 6, 12 }, false };
    case F_SMOOTH_HYBRID6: return { 3, 6, 0, 18, 3, 0, 0, { VC_POSE, VC_POSE, VC_POSE, -1 }, { 0, 6, 12, 0 }, true };
    case F_SMOOTH_POSE6:   return { 3, 6, 0, 18, 3, 0, 0, { VC_POSE, VC_POSE, VC_POSE, -1 }, { 0, 6, 12, 0 }, false };
    case F_FLOWPROJ2:      return { 2, 2, 15, 8, 1, 1, 2, { VC_FLOW, VC_POSE, -1, -1 }, { 0, 2, 0, 0 }, false };
    case F_PRIOR_VEL3:     return { 1, 3, 3, 3, 0, 0, 0, { VC_VEL, -1, -1, -1, -1, -1 }, { 0, 0, 0, 0, 0, 0 }, false };
    case F_PRIOR_BIAS6:    return { 1, 6, 6, 6, 0, 0, 0, { VC_BIAS, -1, -1, -1, -1, -1 }, { 0, 0, 0, 0, 0, 0 }, false };
    case F_COMBINED_IMU15: return { 6, 15, IMU_MEAS, 30, 2, 0, 0, { VC_POSE, VC_VEL, VC_POSE, VC_VEL, VC_BIAS, VC_BIAS }, { 0, 6, 9, 15, 18, 24 }, false };
    case F_LINEAR_PP3:     return { 2, 3, LINEAR_PP3_MEAS, 9, 1, 1, 3, { VC_POSE, VC_POINT, -1, -1 }, { 0, 6, 0, 0 }, false };
    case F_LINEAR_PPP3:    return { 3, 3, LINEAR_PPP3_MEAS, 15, 2, 1, 3, { VC_POSE, VC_POSE, VC_POINT, -1 }, { 0, 6, 12, 0 }, false };
    default:               return { 0, 0, 0, 0, 0, 0, 0, { -1, -1, -1, -1 }, { 0, 0, 0, 0 }, false };
  }
}
__host__ __device__ constexpr int class_dim(int c) { return c == VC_POSE || c == VC_BIAS ? 6 : (c == VC_POINT || c == VC_VEL ? 3 : 2); }

// Variables of one factor, gathered into registers.  Pose slots fill pose[] in key order, point/flow
// slots fill pt[] in key order (a flow uses pt[.][0..1]).
struct FVars {
  Pose pose[3];
  double pt[2][3];
};

// gtsam StereoCamera::project2 at the camera-frame point q (4.2.0): returns false on cheirality (z <= 0)
DYN_HD bool stereo_project(const double* K, const double* q, double* z, double* Dq) {
  if (q[2] <= 0.0) return false;
  const double fx = K[0], fy = K[1], b = K[5], d = 1.0/q[2], x = q[0], y = q[1];
  z[0] = K[3] + d*fx*x; z[1] = K[3] + d*fx*(x - b); z[2] = K[4] + d*fy*y;
  Dq[0] = d*fx; Dq[1] = 0; Dq[2] = -d*d*fx*x;
  Dq[3] = d*fx; Dq[4] = 0; Dq[5] = -d*d*fx*(x - b);
  Dq[6] = 0; Dq[7] = d*fy; Dq[8] = -d*d*fy*y;
  return true;
}

// ---- residual-only forms of the numerically differentiated factors
// LandmarkMotionPoseFactor.cc:99-105: r = m_k - L_k L_{k-1}^-1 m_{k-1}
DYN_HD void motionpose_residual(const double* pprev, const double* pcur, const Pose& Lprev, const Pose& Lcur, double* r) {
  double a[3], q[3];
  se3_transform_to(Lprev, pprev, a); se3_transform_from(Lcur, a, q);
  r[0] = pcur[0] - q[0]; r[1] = pcur[1] - q[1]; r[2] = pcur[2] - q[2];
}
// HybridFormulationFactors.cc:306-322
DYN_HD void smooth_hybrid_residual(const Pose& E2, const Pose& E1, const Pose& E0, const Pose& Le, double* r) {
  Pose Lk2, Lk1, Lk, a, b, rel;
  se3_compose(E2, Le, Lk2); se3_compose(E1, Le, Lk1); se3_compose(E0, Le, Lk);
  se3_between(Lk2, Lk1, a); se3_between(Lk1, Lk, b); se3_between(a, b, rel);
  se3_logmap(rel, r);
}
// LandmarkPoseSmoothingFactor.cc:82-93
DYN_HD void smooth_pose_residual(const Pose& P2, const Pose& P1, const Pose& P0, double* r) {
  Pose i2, i1, a, b, hx;
  se3_inverse(P2, i2); se3_inverse(P1, i1);
  se3_compose(P1, i2, a); se3_compose(P0, i1, b);
  se3_between(a, b, hx); se3_logmap(hx, r);
}

template <int T>
DYN_HD void numeric_residual(const FVars& v, const Pose& aux, double* r) {
  if (T == F_MOTIONPOSE3) motionpose_residual(v.pt[0], v.pt[1], v.pose[0], v.pose[1], r);
  else if (T == F_SMOOTH_HYBRID6) smooth_hybrid_residual(v.pose[0], v.pose[1], v.pose[2], aux, r);
  else smooth_pose_residual(v.pose[0], v.pose[1], v.pose[2], r);
}

// gtsam::numericalDerivative (base/numericalDerivative.h, 4.2.0): central differences through retract,
// delta = 1e-5, column = ((h(x+d) - hx) - (h(x-d) - hx)) / (2 delta) -- the reference's own Jacobians for
// LandmarkMotionPoseFactor / HybridSmoothingFactor / LandmarkPoseSmoothingFactor.
template <int T>
__device__ void numeric_jacobian(const FVars& v, const Pose& aux, const double* hx, double* J) {
  constexpr TypeInfo ti = type_info(T);
  constexpr double delta = 1e-5, factor = 1.0/(2.0*delta);
  int pi = 0, li = 0;
  for (int k = 0; k < ti.arity; k++) {
    const int c = ti.cls[k], n = class_dim(c);
    for (int j = 0; j < n; j++) {
      double h1[6], h2[6];
      for (int s = 0; s < 2; s++) {
        FVars w = v;
        const double d = s == 0 ? delta : -delta;
        if (c == VC_POSE) { double xi[6] = {0, 0, 0, 0, 0, 0}; xi[j] = d; se3_retract(v.pose[pi], xi, w.pose[pi]); }
        else w.pt[li][j] += d;
        numeric_residual<T>(w, aux, s == 0 ? h1 : h2);
      }
      for (int i = 0; i < ti.dim; i++) J[i*ti.jcols + ti.coloff[k] + j] = ((h1[i] - hx[i]) - (h2[i] - hx[i]))*factor;
    }
    if (c == VC_POSE) pi++; else li++;
  }
}

// Unwhitened residual r[dim] and (if WJ) Jacobian J[dim][jcols] (row-major, key-order columns).
template <int T, bool WJ>
__device__ __forceinline__ void factor_eval(const FVars& v, const double* z, const Pose& aux, const double* K,
                                            double* r, double* J) {
  constexpr TypeInfo ti = type_info(T);
  if (WJ) {
#pragma unroll
    for (int i = 0; i < ti.dim*ti.jcols; i++) J[i] = 0.0;
  }
  if constexpr (T == F_PRIOR6) {
    // gtsam::PriorFactor<Pose3>::evaluateError: e = -Local(x, prior), H = I
    Pose prior;
#pragma unroll
    for (int i = 0; i < 9; i++) prior.R[i] = z[i];
#pragma unroll
    for (int i = 0; i < 3; i++) prior.t[i] = z[9+i];
    double e[6]; se3_local(v.pose[0], prior, e);
#pragma unroll
    for (int i = 0; i < 6; i++) { r[i] = -e[i]; if (WJ) J[i*6+i] = 1.0; }
  } else if constexpr (T == F_BETWEEN6) {
    // gtsam::BetweenFactor<Pose3>: hx = p1^-1 p2, H1 = -Ad(hx^-1), H2 = I, e = Local(measured, hx)
    Pose m, hx;
#pragma unroll
    for (int i = 0; i < 9; i++) m.R[i] = z[i];
#pragma unroll
    for (int i = 0; i < 3; i++) m.t[i] = z[9+i];
    se3_between(v.pose[0], v.pose[1], hx);
    se3_local(m, hx, r);
    if (WJ) {
      Pose hi; double Ad[36]; se3_inverse(hx, hi); se3_adjoint(hi, Ad);
#pragma unroll
      for (int a = 0; a < 6; a++) {
#pragma unroll
        for (int c = 0; c < 6; c++) J[a*12+c] = -Ad[a*6+c];
        J[a*12+6+a] = 1.0;
      }
    }
  } else if constexpr (T == F_POSE2POINT3) {
    // gtsam::PoseToPointFactor: e = X.transformTo(p) - z, dX = [[q]x -I], dp = R^T
    double q[3]; se3_transform_to(v.pose[0], v.pt[0], q);
#pragma unroll
    for (int i = 0; i < 3; i++) r[i] = q[i] - z[i];
    if (WJ) {
      J[0*9+1] = -q[2]; J[0*9+2] = q[1]; J[1*9+0] = q[2]; J[1*9+2] = -q[0]; J[2*9+0] = -q[1]; J[2*9+1] = q[0];
#pragma unroll
      for (int a = 0; a < 3; a++) {
        J[a*9+3+a] = -1.0;
#pragma unroll
        for (int c = 0; c < 3; c++) J[a*9+6+c] = v.pose[0].R[3*c+a];
      }
    }
  } else if constexpr (T == F_STEREO3) {
    // gtsam::GenericStereoFactor: e = StereoCamera(X,K).project(p) - z; cheirality -> zero J, e = 2 fx
    double q[3], zz[3], Dq[9]; se3_transform_to(v.pose[0], v.pt[0], q);
    if (!stereo_project(K, q, zz, Dq)) { r[0] = r[1] = r[2] = 2.0*K[0]; return; }
#pragma unroll
    for (int i = 0; i < 3; i++) r[i] = zz[i] - z[i];
    if (WJ) {
      double Dp[18] = { 0, -q[2], q[1], -1, 0, 0,  q[2], 0, -q[0], 0, -1, 0,  -q[1], q[0], 0, 0, 0, -1 };
#pragma unroll
      for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int c = 0; c < 6; c++) J[a*9+c] = Dq[3*a]*Dp[c] + Dq[3*a+1]*Dp[6+c] + Dq[3*a+2]*Dp[12+c];
#pragma unroll
        for (int c = 0; c < 3; c++)
          J[a*9+6+c] = Dq[3*a]*v.pose[0].R[3*c] + Dq[3*a+1]*v.pose[0].R[3*c+1] + Dq[3*a+2]*v.pose[0].R[3*c+2];
      }
    }
  } else if constexpr (T == F_TERNARY3) {
    // LandmarkMotionTernaryFactor.cc:41-72: e = m_{k-1} - H^-1 m_k, J1 = I, J2 = -R_H^T, J3 = [-[q]x I]
    double q[3]; se3_transform_to(v.pose[0], v.pt[1], q);
#pragma unroll
    for (int i = 0; i < 3; i++) r[i] = v.pt[0][i] - q[i];
    if (WJ) {
#pragma unroll
      for (int a = 0; a < 3; a++) {
        J[a*12+a] = 1.0;
#pragma unroll
        for (int c = 0; c < 3; c++) J[a*12+3+c] = -v.pose[0].R[3*c+a];
        J[a*12+9+a] = 1.0;
      }
      J[0*12+6+1] = q[2];  J[0*12+6+2] = -q[1];
      J[1*12+6+0] = -q[2]; J[1*12+6+2] = q[0];
      J[2*12+6+0] = q[1];  J[2*12+6+1] = -q[0];
    }
  } else if constexpr (T == F_HYBRID3 || T == F_HYBRID_STEREO3) {
    // HybridFormulationFactors.cc:96-187, 213-261: e = X^-1 * H * L_e * m_L - z  (closed form of the chain)
    const Pose& X = v.pose[0]; const Pose& H = v.pose[1];
    double qo[3], pw[3], q[3];
    se3_transform_from(aux, v.pt[0], qo);       // point in the key-frame world
    se3_transform_from(H, qo, pw);              // point in the world at k
    se3_transform_to(X, pw, q);                 // point in camera k
    double RXtRH[9]; m3tmul(X.R, H.R, RXtRH);
    double JX[18] = { 0, -q[2], q[1], -1, 0, 0,  q[2], 0, -q[0], 0, -1, 0,  -q[1], q[0], 0, 0, 0, -1 };
    double JH[18], Jm[9];
    if (WJ) {
      const double nqx[9] = { 0, qo[2], -qo[1], -qo[2], 0, qo[0], qo[1], -qo[0], 0 };  // -[qo]x
      double A[9]; m3mul(RXtRH, nqx, A);
#pragma unroll
      for (int a = 0; a < 3; a++)
#pragma unroll
        for (int c = 0; c < 3; c++) { JH[6*a+c] = A[3*a+c]; JH[6*a+3+c] = RXtRH[3*a+c]; }
      m3mul(RXtRH, aux.R, Jm);
    }
    if constexpr (T == F_HYBRID3) {
#pragma unroll
      for (int i = 0; i < 3; i++) r[i] = q[i] - z[i];
      if (WJ) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
#pragma unroll
          for (int c = 0; c < 6; c++) { J[a*15+c] = JX[6*a+c]; J[a*15+6+c] = JH[6*a+c]; }
#pragma unroll
          for (int c = 0; c < 3; c++) J[a*15+12+c] = Jm[3*a+c];
        }
      }
    } else {
      double zz[3], Dq[9];
      if (!stereo_project(K, q, zz, Dq)) { r[0] = r[1] = r[2] = 2.0*K[0]; return; }
#pragma unroll
      for (int i = 0; i < 3; i++) r[i] = zz[i] - z[i];
      if (WJ) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
#pragma unroll
          for (int c = 0; c < 6; c++) {
            J[a*15+c] = Dq[3*a]*JX[c] + Dq[3*a+1]*JX[6+c] + Dq[3*a+2]*JX[12+c];
            J[a*15+6+c] = Dq[3*a]*JH[c] + Dq[3*a+1]*JH[6+c] + Dq[3*a+2]*JH[12+c];
          }
#pragma unroll
          for (int c = 0; c < 3; c++) J[a*15+12+c] = Dq[3*a]*Jm[c] + Dq[3*a+1]*Jm[3+c] + Dq[3*a+2]*Jm[6+c];
        }
      }
    }
  } else if constexpr (T == F_MOTIONPOSE3 || T == F_SMOOTH_HYBRID6 || T == F_SMOOTH_POSE6) {
    numeric_residual<T>(v, aux, r);
    if (WJ) numeric_jacobian<T>(v, aux, r, J);
  } else if constexpr (T == F_FLOWPROJ2) {
    // Pose3FlowProjectionFactor.h:73-133; z = kp(2), depth, X_prev(12); K = Cal3_S2
    const double fx = K[0], fy = K[1], s = K[2], u0 = K[3], v0 = K[4];
    Pose Xp;
#pragma unroll
    for (int i = 0; i < 9; i++) Xp.R[i] = z[3+i];
#pragma unroll
    for (int i = 0; i < 3; i++) Xp.t[i] = z[12+i];
    const double depth = z[2];
    const double yn = (z[1] - v0)/fy, xn = (z[0] - u0 - s*yn)/fx;
    const double pc[3] = { xn*depth, yn*depth, depth };
    double Pw[3], Pc[3];
    se3_transform_from(Xp, pc, Pw); se3_transform_to(v.pose[0], Pw, Pc);
    if (Pc[2] <= 0.0) { r[0] = r[1] = 2.0*fx; return; }
    const double x = Pc[0], y = Pc[1], zc = Pc[2], z2 = zc*zc;
    const double un = x/zc, vn = y/zc;
    r[0] = z[0] + v.pt[0][0] - (fx*un + s*vn + u0);
    r[1] = z[1] + v.pt[0][1] - (fy*vn + v0);
    if (WJ) {
      J[0*8+0] = 1.0; J[1*8+1] = 1.0;
      J[0*8+2] = -(x*y/z2*fx); J[0*8+3] = (1 + (x*x/z2))*fx; J[0*8+4] = -(y/zc*fx);
      J[0*8+5] = 1.0/zc*fx;    J[0*8+6] = -0.0;              J[0*8+7] = -(x/z2*fx);
      J[1*8+2] = -((1 + y*y/z2)*fy); J[1*8+3] = x*y/z2*fy;   J[1*8+4] = x/zc*fy;
      J[1*8+5] = -0.0;         J[1*8+6] = 1.0/zc*fy;         J[1*8+7] = -(y/z2*fy);
    }
  }
}

// noiseModel::Diagonal/Isotropic whitening + noiseModel::Robust(Huber) weight.  r is whitened in place;
// returns sqrt(w) and the nonlinear factor error rho.  [GTSAM-ext linear/NoiseModel.cpp, LossFunctions.cpp]
template <int D>
DYN_HD double whiten_weight(double* r, const double* isig, int sigma_dim, double robust_k, double* err) {
  double n2 = 0;
#pragma unroll
  for (int k = 0; k < D; k++) { r[k] *= (sigma_dim == 1 ? isig[0] : isig[k]); n2 += r[k]*r[k]; }
  if (robust_k > 0) {
    const double n = sqrt(n2);
    if (n <= robust_k) { *err = 0.5*n2; return 1.0; }
    *err = robust_k*(n - 0.5*robust_k);
    return sqrt(robust_k/n);
  }
  *err = 0.5*n2;
  return 1.0;
}

}  // namespace dynoba
