/*
 * oracle/dynoba_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT).  See the header.
 *
 * Restates, in plain C / fp64:
 *   - GTSAM 4.2.0 Lie-group maps (Rot3/Pose3 Expmap, Logmap, AdjointMap; built with
 *     GTSAM_POSE3_EXPMAP=ON, GTSAM_ROT3_EXPMAP=ON, docker/Dockerfile.amd64:104-112)   [GTSAM-ext]
 *   - the reference's factors, each citing its source file:line below
 *   - noiseModel::{Isotropic,Diagonal,Robust(Huber)} whitening                         [GTSAM-ext]
 *   - LevenbergMarquardtOptimizer::{iterate,tryLambda} control flow                    [GTSAM-ext]
 *   - landmark Schur complement + banded Cholesky (the arithmetic GTSAM's multifrontal
 *     elimination performs, organised as in backend/rgbd/HybridEstimator.hpp:349-396,1007-1080)
 * Paths are relative to /root/reference/dynosam unless stated.
 */
#include "dynoba_oracle.h"
#include <float.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------ small linear algebra */
static void m3mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
    C[3*i+j] = A[3*i]*B[j] + A[3*i+1]*B[3+j] + A[3*i+2]*B[6+j];
}
static void m3tmul(const double* A, const double* B, double* C) { /* A^T B */
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
    C[3*i+j] = A[i]*B[j] + A[3+i]*B[3+j] + A[6+i]*B[6+j];
}
static void m3vec(const double* A, const double* v, double* o) {
  for (int i = 0; i < 3; i++) o[i] = A[3*i]*v[0] + A[3*i+1]*v[1] + A[3*i+2]*v[2];
}
static void m3tvec(const double* A, const double* v, double* o) {
  for (int i = 0; i < 3; i++) o[i] = A[i]*v[0] + A[3+i]*v[1] + A[6+i]*v[2];
}
static void skew3(const double* v, double* M) {
  M[0] = 0; M[1] = -v[2]; M[2] = v[1];
  M[3] = v[2]; M[4] = 0; M[5] = -v[0];
  M[6] = -v[1]; M[7] = v[0]; M[8] = 0;
}
static void matmul(const double* A, const double* B, double* C, int m, int k, int n) {
  for (int i = 0; i < m; i++) for (int j = 0; j < n; j++) {
    double s = 0; for (int l = 0; l < k; l++) s += A[i*k+l]*B[l*n+j];
    C[i*n+j] = s;
  }
}

/* ------------------------------------------------------------------ Lie groups [GTSAM-ext] */
/* gtsam/geometry/SO3.cpp ExpmapFunctor (4.2.0): nearZero iff theta^2 <= eps;
 * one_minus_cos = 2 sin^2(theta/2); R = I + sin(theta) K + (1-cos) K^2, K = [w]x/theta. */
static void so3_expmap(const double* w, double* R) {
  double th2 = w[0]*w[0] + w[1]*w[1] + w[2]*w[2];
  double W[9]; skew3(w, W);
  if (th2 <= DBL_EPSILON) {
    for (int i = 0; i < 9; i++) R[i] = W[i];
    R[0] += 1; R[4] += 1; R[8] += 1;
    return;
  }
  double th = sqrt(th2), s = sin(th), s2 = sin(0.5*th), omc = 2.0*s2*s2;
  double K[9], KK[9];
  for (int i = 0; i < 9; i++) K[i] = W[i]/th;
  m3mul(K, K, KK);
  for (int i = 0; i < 9; i++) R[i] = s*K[i] + omc*KK[i];
  R[0] += 1; R[4] += 1; R[8] += 1;
}
/* gtsam/geometry/SO3.cpp SO3::Logmap (4.2.0). */
static void so3_logmap(const double* R, double* w) {
  const double R11 = R[0], R12 = R[1], R13 = R[2], R21 = R[3], R22 = R[4], R23 = R[5],
               R31 = R[6], R32 = R[7], R33 = R[8];
  double tr = R11 + R22 + R33;
  if (tr + 1.0 < 1e-10) { /* theta = pi cases */
    if (fabs(R33 + 1.0) > 1e-5) {
      double f = M_PI / sqrt(2.0 + 2.0*R33);
      w[0] = f*R13; w[1] = f*R23; w[2] = f*(1.0 + R33);
    } else if (fabs(R22 + 1.0) > 1e-5) {
      double f = M_PI / sqrt(2.0 + 2.0*R22);
      w[0] = f*R12; w[1] = f*(1.0 + R22); w[2] = f*R32;
    } else {
      double f = M_PI / sqrt(2.0 + 2.0*R11);
      w[0] = f*(1.0 + R11); w[1] = f*R21; w[2] = f*R31;
    }
    return;
  }
  double mag, tr3 = tr - 3.0;
  if (tr3 < -1e-7) {
    double th = acos((tr - 1.0)/2.0);
    mag = th/(2.0*sin(th));
  } else {
    mag = 0.5 - tr3/12.0;
  }
  w[0] = mag*(R32 - R23); w[1] = mag*(R13 - R31); w[2] = mag*(R21 - R12);
}
/* gtsam/geometry/Pose3.cpp Pose3::Expmap (4.2.0), tangent order [omega; v]. */
void orc_se3_expmap(const double* xi, double* P) {
  const double* w = xi; const double* v = xi + 3;
  so3_expmap(w, P);
  double th2 = w[0]*w[0] + w[1]*w[1] + w[2]*w[2];
  if (th2 > DBL_EPSILON) {
    double wv = w[0]*v[0] + w[1]*v[1] + w[2]*v[2];
    double c[3] = { w[1]*v[2] - w[2]*v[1], w[2]*v[0] - w[0]*v[2], w[0]*v[1] - w[1]*v[0] };
    double Rc[3]; m3vec(P, c, Rc);
    for (int i = 0; i < 3; i++) P[9+i] = (c[i] - Rc[i] + w[i]*wv)/th2;
  } else {
    P[9] = v[0]; P[10] = v[1]; P[11] = v[2];
  }
}
/* gtsam/geometry/Pose3.cpp Pose3::Logmap (4.2.0). */
void orc_se3_logmap(const double* P, double* xi) {
  double w[3]; so3_logmap(P, w);
  const double* T = P + 9;
  double t = sqrt(w[0]*w[0] + w[1]*w[1] + w[2]*w[2]);
  xi[0] = w[0]; xi[1] = w[1]; xi[2] = w[2];
  if (t < 1e-10) { xi[3] = T[0]; xi[4] = T[1]; xi[5] = T[2]; return; }
  double wn[3] = { w[0]/t, w[1]/t, w[2]/t }, W[9];
  skew3(wn, W);
  double Tan = tan(0.5*t), WT[3], WWT[3];
  m3vec(W, T, WT); m3vec(W, WT, WWT);
  for (int i = 0; i < 3; i++) xi[3+i] = T[i] - (0.5*t)*WT[i] + (1.0 - t/(2.0*Tan))*WWT[i];
}
void orc_se3_compose(const double* a, const double* b, double* o) {
  double R[9], t[3]; m3mul(a, b, R); m3vec(a, b + 9, t);
  for (int i = 0; i < 9; i++) o[i] = R[i];
  for (int i = 0; i < 3; i++) o[9+i] = t[i] + a[9+i];
}
void orc_se3_inverse(const double* a, double* o) {
  double R[9], t[3];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[3*i+j] = a[3*j+i];
  m3vec(R, a + 9, t);
  for (int i = 0; i < 9; i++) o[i] = R[i];
  for (int i = 0; i < 3; i++) o[9+i] = -t[i];
}
static void se3_between(const double* a, const double* b, double* o) {
  double ai[12]; orc_se3_inverse(a, ai); orc_se3_compose(ai, b, o);
}
/* Pose3::retract with POSE3_EXPMAP: T * Expmap(xi). */
void orc_se3_retract(const double* P, const double* xi, double* o) {
  double E[12]; orc_se3_expmap(xi, E); orc_se3_compose(P, E, o);
}
static void se3_local(const double* a, const double* b, double* xi) { /* Logmap(a^-1 b) */
  double d[12]; se3_between(a, b, d); orc_se3_logmap(d, xi);
}
/* Pose3::AdjointMap: [[R,0],[[t]x R, R]] in [omega; v] order. */
static void se3_adjoint(const double* P, double* Ad) {
  double tx[9], txR[9]; skew3(P + 9, tx); m3mul(tx, P, txR);
  memset(Ad, 0, 36*sizeof(double));
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    Ad[6*i+j] = P[3*i+j];
    Ad[6*(i+3)+j] = txR[3*i+j];
    Ad[6*(i+3)+j+3] = P[3*i+j];
  }
}
static void se3_transform_from(const double* P, const double* p, double* o) {
  m3vec(P, p, o); o[0] += P[9]; o[1] += P[10]; o[2] += P[11];
}
static void se3_transform_to(const double* P, const double* p, double* o) {
  double d[3] = { p[0]-P[9], p[1]-P[10], p[2]-P[11] }; m3tvec(P, d, o);
}

/* ------------------------------------------------------------------ type tables */
enum { VC_POSE = 0, VC_POINT = 1, VC_FLOW = 2 };
static const int T_ARITY[ORC_NUM_TYPES] = { 1, 2, 2, 2, 3, 3, 3, 4, 3, 3, 2 };
static const int T_DIM[ORC_NUM_TYPES]   = { 6, 6, 3, 3, 3, 3, 3, 3, 6, 6, 2 };
static const int T_MEAS[ORC_NUM_TYPES]  = { 12, 12, 3, 3, 0, 3, 3, 0, 0, 0, 15 };
static const int T_CLS[ORC_NUM_TYPES][4] = {
  { VC_POSE, -1, -1, -1 },              /* PRIOR6 */
  { VC_POSE, VC_POSE, -1, -1 },         /* BETWEEN6 */
  { VC_POSE, VC_POINT, -1, -1 },        /* POSE2POINT3 (poseKey, pointKey) */
  { VC_POSE, VC_POINT, -1, -1 },        /* STEREO3 (poseKey, landmarkKey) */
  { VC_POINT, VC_POINT, VC_POSE, -1 },  /* TERNARY3 (prevPoint, curPoint, motion) */
  { VC_POSE, VC_POSE, VC_POINT, -1 },   /* HYBRID3 (X_k, e_H_k, m_L) */
  { VC_POSE, VC_POSE, VC_POINT, -1 },   /* HYBRID_STEREO3 */
  { VC_POINT, VC_POINT, VC_POSE, VC_POSE }, /* MOTIONPOSE3 (prevPt, curPt, prevPose, curPose) */
  { VC_POSE, VC_POSE, VC_POSE, -1 },    /* SMOOTH_HYBRID6 */
  { VC_POSE, VC_POSE, VC_POSE, -1 },    /* SMOOTH_POSE6 */
  { VC_FLOW, VC_POSE, -1, -1 },         /* FLOWPROJ2 (flow, pose) */
};
static int cls_dim(int c) { return c == VC_POSE ? 6 : (c == VC_POINT ? 3 : 2); }
int orc_type_arity(int t) { return T_ARITY[t]; }
int orc_type_dim(int t) { return T_DIM[t]; }
int orc_type_meas_dim(int t) { return T_MEAS[t]; }
int orc_type_jcols(int t) {
  int s = 0; for (int k = 0; k < T_ARITY[t]; k++) s += cls_dim(T_CLS[t][k]); return s;
}

void orc_lm_default_params(orc_lm_params* p) { /* LevenbergMarquardtParams defaults [GTSAM-ext] */
  p->lambda_initial = 1e-5; p->lambda_factor = 10.0; p->lambda_upper = 1e5; p->lambda_lower = 0.0;
  p->min_model_fidelity = 1e-3; p->rel_tol = 1e-5; p->abs_tol = 1e-5; p->err_tol = 0.0;
  p->max_iterations = 100; p->verbose = 0;
}

/* ------------------------------------------------------------------ factor residuals */
/* HybridFormulationFactors.cc:96-135  T = X^-1 * E * L with 6x6 Jacobians (literal chain). */
static void hybrid_camera_transform(const double* X, const double* E, const double* L, double* T,
                                    double* J1, double* J2) {
  double invX[12], comb1[12];
  orc_se3_inverse(X, invX);
  orc_se3_compose(E, L, comb1);
  orc_se3_compose(invX, comb1, T);
  if (J1 || J2) {
    double H_invX_X[36], AdX[36]; se3_adjoint(X, AdX);
    for (int i = 0; i < 36; i++) H_invX_X[i] = -AdX[i];           /* inverse: -Ad(X) */
    double Linv[12], H_comb1_E[36]; orc_se3_inverse(L, Linv); se3_adjoint(Linv, H_comb1_E); /* compose: Ad(L^-1) */
    double c1inv[12], H_res_invX[36]; orc_se3_inverse(comb1, c1inv); se3_adjoint(c1inv, H_res_invX);
    if (J1) matmul(H_res_invX, H_invX_X, J1, 6, 6, 6);            /* dRes/dX */
    if (J2) memcpy(J2, H_comb1_E, 36*sizeof(double));             /* dRes/dE = I * Ad(L^-1) */
  }
}
/* HybridFormulationFactors.cc:96-126 projectToCamera3: P = T * m_L; J = H_P_T * H_T_{X,E}, H_P_m = R_T. */
static void hybrid_project_to_camera3(const double* X, const double* E, const double* L, const double* m,
                                      double* p, double* JX, double* JE, double* Jm) {
  double T[12], H_T_X[36], H_T_E[36];
  hybrid_camera_transform(X, E, L, T, JX ? H_T_X : NULL, JE ? H_T_E : NULL);
  se3_transform_from(T, m, p);
  if (JX || JE) {
    double mx[9], Rmx[9], H_P_T[18]; skew3(m, mx); m3mul(T, mx, Rmx);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { H_P_T[6*i+j] = -Rmx[3*i+j]; H_P_T[6*i+3+j] = T[3*i+j]; }
    if (JX) matmul(H_P_T, H_T_X, JX, 3, 6, 6);
    if (JE) matmul(H_P_T, H_T_E, JE, 3, 6, 6);
  }
  if (Jm) memcpy(Jm, T, 9*sizeof(double));
}
/* HybridFormulationFactors.cc:37-94 projectToObject3: P = L^-1 * E^-1 * X * Z (literal chain). */
void orc_hybrid_project_to_object3(const double* X, const double* E, const double* L, const double* Z,
                                   double* out, double* JX, double* JE, double* JL) {
  double invL[12], invE[12], comb1[12], comb2[12];
  orc_se3_inverse(L, invL); orc_se3_inverse(E, invE);
  orc_se3_compose(invL, invE, comb1); orc_se3_compose(comb1, X, comb2);
  se3_transform_from(comb2, Z, out);
  if (!(JX || JE || JL)) return;
  double H_invL_L[36], H_invE_E[36], Ad[36];
  se3_adjoint(L, Ad); for (int i = 0; i < 36; i++) H_invL_L[i] = -Ad[i];
  se3_adjoint(E, Ad); for (int i = 0; i < 36; i++) H_invE_E[i] = -Ad[i];
  double H_comb1_invL[36]; /* compose(invL, invE): d/dinvL = Ad(invE^-1) = Ad(E); d/dinvE = I */
  se3_adjoint(E, H_comb1_invL);
  double Xinv[12], H_comb2_comb1[36]; orc_se3_inverse(X, Xinv); se3_adjoint(Xinv, H_comb2_comb1); /* d/dX = I */
  double zx[9], Rzx[9], H_res_comb2[18]; skew3(Z, zx); m3mul(comb2, zx, Rzx);
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { H_res_comb2[6*i+j] = -Rzx[3*i+j]; H_res_comb2[6*i+3+j] = comb2[3*i+j]; }
  if (JX) memcpy(JX, H_res_comb2, 18*sizeof(double));
  double t36[36], t18[18];
  if (JE) { matmul(H_res_comb2, H_comb2_comb1, t18, 3, 6, 6); matmul(t18, H_invE_E, JE, 3, 6, 6); }
  if (JL) { matmul(H_comb2_comb1, H_comb1_invL, t36, 6, 6, 6); matmul(H_res_comb2, t36, t18, 3, 6, 6);
            matmul(t18, H_invL_L, JL, 3, 6, 6); }
}

/* gtsam/geometry/StereoCamera.cpp project2 with an identity-or-given left pose (4.2.0):
 * d=1/z, uL=u0+fx x d, uR=u0+fx (x-b) d, v=v0+fy y d; z<=0 -> cheirality.  Returns 1 on cheirality.
 * Dq = d(uL,uR,v)/dq (3x3) for the point q in the camera frame. */
static int stereo_project_cam(const double* K, const double* q, double* z, double* Dq) {
  if (q[2] <= 0.0) return 1;
  double fx = K[0], fy = K[1], b = K[5], d = 1.0/q[2], x = q[0], y = q[1];
  z[0] = K[3] + d*fx*x; z[1] = K[3] + d*fx*(x - b); z[2] = K[4] + d*fy*y;
  if (Dq) {
    Dq[0] = d*fx; Dq[1] = 0; Dq[2] = -d*d*fx*x;
    Dq[3] = d*fx; Dq[4] = 0; Dq[5] = -d*d*fx*(x - b);
    Dq[6] = 0; Dq[7] = d*fy; Dq[8] = -d*d*fy*y;
  }
  return 0;
}

/* LandmarkMotionPoseFactor.cc:99-105 residual. */
static void motionpose_residual(const double* pprev, const double* pcur, const double* Lprev, const double* Lcur, double* r) {
  double Li[12], M[12], q[3];
  orc_se3_inverse(Lprev, Li); orc_se3_compose(Lcur, Li, M); se3_transform_from(M, pprev, q);
  for (int i = 0; i < 3; i++) r[i] = pcur[i] - q[i];
}
/* HybridFormulationFactors.cc:306-322 HybridSmoothingFactor::residual. */
static void smooth_hybrid_residual(const double* E2, const double* E1, const double* E0, const double* Le, double* r) {
  double Lk2[12], Lk1[12], Lk[12], a[12], b[12], rel[12];
  orc_se3_compose(E2, Le, Lk2); orc_se3_compose(E1, Le, Lk1); orc_se3_compose(E0, Le, Lk);
  se3_between(Lk2, Lk1, a); se3_between(Lk1, Lk, b); se3_between(a, b, rel);
  orc_se3_logmap(rel, r); /* Local(Identity, rel) = Logmap(rel) */
}
/* LandmarkPoseSmoothingFactor.cc:82-93 residual. */
static void smooth_pose_residual(const double* P2, const double* P1, const double* P0, double* r) {
  double i2[12], i1[12], a[12], b[12], hx[12];
  orc_se3_inverse(P2, i2); orc_se3_inverse(P1, i1);
  orc_se3_compose(P1, i2, a); orc_se3_compose(P0, i1, b);
  se3_between(a, b, hx); orc_se3_logmap(hx, r);
}

/* gtsam::numericalDerivative (base/numericalDerivative.h, 4.2.0): central differences through
 * retract with delta = 1e-5; column j = ((h(x+d) - hx) - (h(x-d) - hx)) / (2 delta). */
typedef void (*resid_fn)(const double* const* vars, const double* extra, double* r);
static void numerical_jacobian(resid_fn fn, const double** vars, const int* cls, int nvars, const double* extra,
                               int which, int dim, double* J, int jcols, int coloff) {
  const double delta = 1e-5, factor = 1.0/(2.0*delta);
  double hx[6], h1[6], h2[6], dx[6], tmp[12];
  const double* v2[4];
  for (int k = 0; k < nvars; k++) v2[k] = vars[k];
  fn(vars, extra, hx);
  int n = cls_dim(cls[which]);
  for (int j = 0; j < n; j++) {
    for (int s = 0; s < 2; s++) {
      memset(dx, 0, sizeof(dx)); dx[j] = s == 0 ? delta : -delta;
      if (cls[which] == VC_POSE) orc_se3_retract(vars[which], dx, tmp);
      else for (int i = 0; i < n; i++) tmp[i] = vars[which][i] + dx[i];
      v2[which] = tmp;
      fn(v2, extra, s == 0 ? h1 : h2);
    }
    v2[which] = vars[which];
    for (int i = 0; i < dim; i++) J[i*jcols + coloff + j] = ((h1[i] - hx[i]) - (h2[i] - hx[i]))*factor;
  }
}
static void fn_motionpose(const double* const* v, const double* e, double* r) { (void)e; motionpose_residual(v[0], v[1], v[2], v[3], r); }
static void fn_smooth_hybrid(const double* const* v, const double* e, double* r) { smooth_hybrid_residual(v[0], v[1], v[2], e, r); }
static void fn_smooth_pose(const double* const* v, const double* e, double* r) { (void)e; smooth_pose_residual(v[0], v[1], v[2], r); }

static const double* var_ptr(const orc_problem* P, int cls, int i) {
  return cls == VC_POSE ? P->pose + 12*(size_t)i : (cls == VC_POINT ? P->point + 3*(size_t)i : P->flow + 2*(size_t)i);
}

void orc_factor_eval(const orc_problem* P, const orc_block* b, int i, double* r, double* J) {
  const int t = b->type, ar = T_ARITY[t], jc = orc_type_jcols(t), d = T_DIM[t];
  const int32_t* ix = b->idx + (size_t)i*ar;
  const double* z = b->meas ? b->meas + (size_t)i*T_MEAS[t] : NULL;
  const double* v[4];
  for (int k = 0; k < ar; k++) v[k] = var_ptr(P, T_CLS[t][k], ix[k]);
  if (J) memset(J, 0, sizeof(double)*d*jc);
  switch (t) {
  case ORC_PRIOR6: { /* PriorFactor<Pose3>: e = -Local(x, prior), H = I  [GTSAM-ext nonlinear/PriorFactor.h] */
    double e[6]; se3_local(v[0], z, e);
    for (int k = 0; k < 6; k++) r[k] = -e[k];
    if (J) for (int k = 0; k < 6; k++) J[k*6+k] = 1.0;
  } break;
  case ORC_BETWEEN6: { /* BetweenFactor<Pose3>: hx = p1^-1 p2 (H1 = -Ad(hx^-1), H2 = I); e = Local(measured, hx);
                          default build does NOT chain the Logmap derivative (no GTSAM_SLOW_BUT_CORRECT_BETWEENFACTOR) */
    double hx[12]; se3_between(v[0], v[1], hx);
    se3_local(z, hx, r);
    if (J) {
      double hi[12], Ad[36]; orc_se3_inverse(hx, hi); se3_adjoint(hi, Ad);
      for (int a = 0; a < 6; a++) { for (int c = 0; c < 6; c++) J[a*12+c] = -Ad[a*6+c]; J[a*12+6+a] = 1.0; }
    }
  } break;
  case ORC_POSE2POINT3: { /* gtsam_unstable/slam/PoseToPointFactor.h: e = X.transformTo(p) - z; Dpose=[[q]x -I], Dpoint=R^T */
    double q[3]; se3_transform_to(v[0], v[1], q);
    for (int k = 0; k < 3; k++) r[k] = q[k] - z[k];
    if (J) {
      double qx[9]; skew3(q, qx);
      for (int a = 0; a < 3; a++) { for (int c = 0; c < 3; c++) { J[a*9+c] = qx[3*a+c]; J[a*9+6+c] = v[0][3*c+a]; } J[a*9+3+a] = -1.0; }
    }
  } break;
  case ORC_STEREO3: { /* GenericStereoFactor: e = StereoCamera(X,K).project(p) - z; cheirality -> zero J, e = 2 fx 1 */
    double q[3], zz[3], Dq[9]; se3_transform_to(v[0], v[1], q);
    if (stereo_project_cam(P->calib, q, zz, Dq)) { for (int k = 0; k < 3; k++) r[k] = 2.0*P->calib[0]; break; }
    for (int k = 0; k < 3; k++) r[k] = zz[k] - z[k];
    if (J) {
      double qx[9], Dp[18], Jx[18], Rt[9], Jp[9]; skew3(q, qx);
      for (int a = 0; a < 3; a++) for (int c = 0; c < 3; c++) { Dp[6*a+c] = qx[3*a+c]; Dp[6*a+3+c] = (a == c) ? -1.0 : 0.0; Rt[3*a+c] = v[0][3*c+a]; }
      matmul(Dq, Dp, Jx, 3, 3, 6); matmul(Dq, Rt, Jp, 3, 3, 3);
      for (int a = 0; a < 3; a++) { for (int c = 0; c < 6; c++) J[a*9+c] = Jx[6*a+c]; for (int c = 0; c < 3; c++) J[a*9+6+c] = Jp[3*a+c]; }
    }
  } break;
  case ORC_TERNARY3: { /* src/factors/LandmarkMotionTernaryFactor.cc:41-72 */
    double Hi[12], q[3]; orc_se3_inverse(v[2], Hi); se3_transform_from(Hi, v[1], q);
    for (int k = 0; k < 3; k++) r[k] = v[0][k] - q[k];
    if (J) {
      for (int a = 0; a < 3; a++) {
        J[a*12+a] = 1.0;                                        /* J1 = I */
        for (int c = 0; c < 3; c++) J[a*12+3+c] = -Hi[3*a+c];   /* J2 = -R_H^T */
        J[a*12+9+a] = 1.0;                                      /* J3 = [-[q]x I] */
      }
      J[0*12+6+1] = q[2];  J[0*12+6+2] = -q[1];
      J[1*12+6+0] = -q[2]; J[1*12+6+2] = q[0];
      J[2*12+6+0] = q[1];  J[2*12+6+1] = -q[0];
    }
  } break;
  case ORC_HYBRID3: { /* src/factors/HybridFormulationFactors.cc:137-187 HybridMotionFactor::evaluateError */
    const double* Le = P->aux_pose + 12*(size_t)b->aux_idx[i];
    double p[3], JX[18], JE[18], Jm[9];
    hybrid_project_to_camera3(v[0], v[1], Le, v[2], p, J ? JX : NULL, J ? JE : NULL, J ? Jm : NULL);
    for (int k = 0; k < 3; k++) r[k] = p[k] - z[k];
    if (J) for (int a = 0; a < 3; a++) {
      for (int c = 0; c < 6; c++) { J[a*15+c] = JX[6*a+c]; J[a*15+6+c] = JE[6*a+c]; }
      for (int c = 0; c < 3; c++) J[a*15+12+c] = Jm[3*a+c];
    }
  } break;
  case ORC_HYBRID_STEREO3: { /* HybridFormulationFactors.cc:213-261 StereoHybridMotionFactor::evaluateError */
    const double* Le = P->aux_pose + 12*(size_t)b->aux_idx[i];
    double p[3], JX[18], JE[18], Jm[9], zz[3], Dq[9];
    hybrid_project_to_camera3(v[0], v[1], Le, v[2], p, JX, JE, Jm);
    if (stereo_project_cam(P->calib, p, zz, Dq)) { for (int k = 0; k < 3; k++) r[k] = 2.0*P->calib[0]; break; }
    for (int k = 0; k < 3; k++) r[k] = zz[k] - z[k];
    if (J) {
      double A[18], B[18], C[9];
      matmul(Dq, JX, A, 3, 3, 6); matmul(Dq, JE, B, 3, 3, 6); matmul(Dq, Jm, C, 3, 3, 3);
      for (int a = 0; a < 3; a++) {
        for (int c = 0; c < 6; c++) { J[a*15+c] = A[6*a+c]; J[a*15+6+c] = B[6*a+c]; }
        for (int c = 0; c < 3; c++) J[a*15+12+c] = C[3*a+c];
      }
    }
  } break;
  case ORC_MOTIONPOSE3: { /* src/factors/LandmarkMotionPoseFactor.cc:42-105 (numerical Jacobians) */
    motionpose_residual(v[0], v[1], v[2], v[3], r);
    if (J) { int off = 0; for (int k = 0; k < 4; k++) { numerical_jacobian(fn_motionpose, v, T_CLS[t], 4, NULL, k, 3, J, jc, off); off += cls_dim(T_CLS[t][k]); } }
  } break;
  case ORC_SMOOTH_HYBRID6: { /* HybridFormulationFactors.cc:274-322 (numerical Jacobians) */
    const double* Le = P->aux_pose + 12*(size_t)b->aux_idx[i];
    smooth_hybrid_residual(v[0], v[1], v[2], Le, r);
    if (J) for (int k = 0; k < 3; k++) numerical_jacobian(fn_smooth_hybrid, v, T_CLS[t], 3, Le, k, 6, J, jc, 6*k);
  } break;
  case ORC_SMOOTH_POSE6: { /* src/factors/LandmarkPoseSmoothingFactor.cc:37-95 (numerical Jacobians) */
    smooth_pose_residual(v[0], v[1], v[2], r);
    if (J) for (int k = 0; k < 3; k++) numerical_jacobian(fn_smooth_pose, v, T_CLS[t], 3, NULL, k, 6, J, jc, 6*k);
  } break;
  case ORC_FLOWPROJ2: { /* include/dynosam/factors/Pose3FlowProjectionFactor.h:73-133; meas = kp(2), depth, pose_prev(12) */
    const double* K = P->calib; const double fx = K[0], fy = K[1], s = K[2], u0 = K[3], v0 = K[4];
    const double* kp = z; double depth = z[2]; const double* Xprev = z + 3;
    /* PinholeCamera(I,K).backproject(kp, depth): Cal3_S2::calibrate then scale by depth */
    double yn = (kp[1] - v0)/fy, xn = (kp[0] - u0 - s*yn)/fx;
    double pc[3] = { xn*depth, yn*depth, depth }, Pw[3], Pc[3];
    se3_transform_from(Xprev, pc, Pw);
    se3_transform_to(v[1], Pw, Pc);
    if (Pc[2] <= 0.0) { r[0] = r[1] = 2.0*fx; break; }   /* CheiralityException branch */
    double x = Pc[0], y = Pc[1], zc = Pc[2], z2 = zc*zc;
    double un = x/zc, vn = y/zc;
    double pu = fx*un + s*vn + u0, pv = fy*vn + v0;
    r[0] = kp[0] + v[0][0] - pu; r[1] = kp[1] + v[0][1] - pv;
    if (J) {
      J[0*8+0] = 1.0; J[1*8+1] = 1.0;
      double H[12];
      H[0] = x*y/z2*fx; H[1] = -(1 + (x*x/z2))*fx; H[2] = y/zc*fx; H[3] = -1.0/zc*fx; H[4] = 0; H[5] = x/z2*fx;
      H[6] = (1 + y*y/z2)*fy; H[7] = -x*y/z2*fy; H[8] = -x/zc*fy; H[9] = 0; H[10] = -1.0/zc*fy; H[11] = y/z2*fy;
      for (int a = 0; a < 2; a++) for (int c = 0; c < 6; c++) J[a*8+2+c] = -1.0*H[6*a+c];
    }
  } break;
  default: break;
  }
}

/* ------------------------------------------------------------------ noise [GTSAM-ext linear/NoiseModel.cpp, LossFunctions.cpp] */
static inline const double* sigma_row(const orc_block* b, int i) {
  return b->sigma_bcast ? b->sigma : b->sigma + (size_t)i*b->sigma_dim;
}
static inline double inv_sigma(const orc_block* b, const double* sg, int row) {
  return 1.0/(b->sigma_dim == 1 ? sg[0] : sg[row]);
}
/* whiten r in place, returns Huber weight w (1 when not robust) and the factor error */
static double whiten_and_weight(const orc_block* b, int i, int d, double* r, double* err) {
  const double* sg = sigma_row(b, i);
  double n2 = 0;
  for (int k = 0; k < d; k++) { r[k] *= inv_sigma(b, sg, k); n2 += r[k]*r[k]; }
  if (b->robust_k > 0) {
    double n = sqrt(n2), k = b->robust_k;
    if (err) *err = n <= k ? 0.5*n2 : k*(n - 0.5*k);   /* mEstimator::Huber::loss */
    return n <= k ? 1.0 : k/n;                          /* mEstimator::Huber::weight */
  }
  if (err) *err = 0.5*n2;
  return 1.0;
}

void orc_linearize_block(const orc_problem* P, const orc_block* b, double* A, double* bv) {
  const int t = b->type, d = T_DIM[t], jc = orc_type_jcols(t);
#pragma omp parallel for schedule(static)
  for (int i = 0; i < b->n; i++) {
    double r[6]; double* J = A + (size_t)i*d*jc;
    orc_factor_eval(P, b, i, r, J);
    const double* sg = sigma_row(b, i);
    double w = whiten_and_weight(b, i, d, r, NULL), sw = sqrt(w);
    for (int k = 0; k < d; k++) {
      double f = inv_sigma(b, sg, k)*sw;
      for (int c = 0; c < jc; c++) J[k*jc+c] *= f;
      bv[(size_t)i*d+k] = -r[k]*sw;
    }
  }
}
void orc_error_block(const orc_problem* P, const orc_block* b, double* err) {
  const int d = T_DIM[b->type];
#pragma omp parallel for schedule(static)
  for (int i = 0; i < b->n; i++) {
    double r[6], e; orc_factor_eval(P, b, i, r, NULL);
    whiten_and_weight(b, i, d, r, &e); err[i] = e;
  }
}
double orc_error(const orc_problem* P) {
  double tot = 0;
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; const int d = T_DIM[b->type];
    double s = 0;
#pragma omp parallel for schedule(static) reduction(+:s)
    for (int i = 0; i < b->n; i++) {
      double r[6], e; orc_factor_eval(P, b, i, r, NULL);
      whiten_and_weight(b, i, d, r, &e); s += e;
    }
    tot += s;
  }
  return tot;
}

/* ------------------------------------------------------------------ dense normal equations (small problems) */
static int dense_off(const orc_problem* P, int cls, int i) {
  return cls == VC_POSE ? 6*i : (cls == VC_POINT ? 6*P->n_pose + 3*i : 6*P->n_pose + 3*P->n_point + 2*i);
}
int orc_dense_dim(const orc_problem* P) { return 6*P->n_pose + 3*P->n_point + 2*P->n_flow; }
void orc_dense_normal(const orc_problem* P, double* H, double* g) {
  int n = orc_dense_dim(P);
  memset(H, 0, sizeof(double)*(size_t)n*n); memset(g, 0, sizeof(double)*n);
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; const int t = b->type, d = T_DIM[t], jc = orc_type_jcols(t), ar = T_ARITY[t];
    double* A = malloc(sizeof(double)*(size_t)b->n*d*jc); double* bv = malloc(sizeof(double)*(size_t)b->n*d);
    orc_linearize_block(P, b, A, bv);
    for (int i = 0; i < b->n; i++) {
      int cols[18], c = 0;
      for (int k = 0; k < ar; k++) { int o = dense_off(P, T_CLS[t][k], b->idx[(size_t)i*ar+k]); for (int q = 0; q < cls_dim(T_CLS[t][k]); q++) cols[c++] = o + q; }
      const double* J = A + (size_t)i*d*jc;
      for (int a = 0; a < jc; a++) {
        double s = 0; for (int k = 0; k < d; k++) s += J[k*jc+a]*bv[(size_t)i*d+k];
        g[cols[a]] += s;
        for (int e = 0; e < jc; e++) { double h = 0; for (int k = 0; k < d; k++) h += J[k*jc+a]*J[k*jc+e]; H[(size_t)cols[a]*n + cols[e]] += h; }
      }
    }
    free(A); free(bv);
  }
}

/* ------------------------------------------------------------------ Schur / band solver */
typedef struct { int blk, i; } fref;
typedef struct {
  int n_lmk;            /* points + flows */
  int* ldim; int* lgrp; /* per landmark: dim, group id */
  int n_grp;
  int* g_lptr; int* g_lmk;   /* CSR group -> landmarks */
  int* g_fptr; fref* g_fac;  /* CSR group -> factors */
  int n_pf; fref* pf;        /* pose-only factors */
  int* pos;                  /* pose -> position in solver order */
  int n, bw, ld;             /* reduced dim, half bandwidth (scalar), ld = bw+1 */
  double** A; double** bv;   /* per block linearization */
} schur_ws;

static int uf_find(int* p, int x) { while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; } return x; }
static int cmp_pos(const void* a, const void* b) {
  const int64_t* x = a; const int64_t* y = b; return x[0] < y[0] ? -1 : (x[0] > y[0] ? 1 : (x[1] < y[1] ? -1 : (x[1] > y[1])));
}
static int lmk_id(const orc_problem* P, int cls, int i) { return cls == VC_POINT ? i : P->n_point + i; }

static schur_ws* schur_setup(const orc_problem* P) {
  schur_ws* W = calloc(1, sizeof(schur_ws));
  int nl = P->n_point + P->n_flow; W->n_lmk = nl;
  W->ldim = malloc(sizeof(int)*(nl+1)); W->lgrp = malloc(sizeof(int)*(nl+1));
  for (int i = 0; i < nl; i++) W->ldim[i] = i < P->n_point ? 3 : 2;
  /* pose ordering */
  W->pos = malloc(sizeof(int)*(P->n_pose+1));
  if (P->pose_order) {
    int64_t* key = malloc(sizeof(int64_t)*2*(size_t)P->n_pose);
    for (int i = 0; i < P->n_pose; i++) { key[2*i] = P->pose_order[i]; key[2*i+1] = i; }
    qsort(key, P->n_pose, 2*sizeof(int64_t), cmp_pos);
    for (int i = 0; i < P->n_pose; i++) W->pos[key[2*i+1]] = i;
    free(key);
  } else for (int i = 0; i < P->n_pose; i++) W->pos[i] = i;
  /* union-find over landmarks linked by multi-landmark factors */
  int* uf = malloc(sizeof(int)*(nl+1)); for (int i = 0; i < nl; i++) uf[i] = i;
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; int t = b->type, ar = T_ARITY[t];
    for (int i = 0; i < b->n; i++) {
      int first = -1;
      for (int k = 0; k < ar; k++) if (T_CLS[t][k] != VC_POSE) {
        int l = lmk_id(P, T_CLS[t][k], b->idx[(size_t)i*ar+k]);
        if (first < 0) first = l; else { int a = uf_find(uf, first), c = uf_find(uf, l); if (a != c) uf[c] = a; }
      }
    }
  }
  int* gid = malloc(sizeof(int)*(nl+1)); int ng = 0;
  for (int i = 0; i < nl; i++) gid[i] = -1;
  for (int i = 0; i < nl; i++) { int r = uf_find(uf, i); if (gid[r] < 0) gid[r] = ng++; W->lgrp[i] = gid[r]; }
  W->n_grp = ng;
  W->g_lptr = calloc(ng+2, sizeof(int)); W->g_lmk = malloc(sizeof(int)*(nl+1));
  for (int i = 0; i < nl; i++) W->g_lptr[W->lgrp[i]+1]++;
  for (int g = 0; g < ng; g++) W->g_lptr[g+1] += W->g_lptr[g];
  int* cur = malloc(sizeof(int)*(ng+1)); memcpy(cur, W->g_lptr, sizeof(int)*(ng+1));
  for (int i = 0; i < nl; i++) W->g_lmk[cur[W->lgrp[i]]++] = i;
  /* factor lists */
  W->g_fptr = calloc(ng+2, sizeof(int)); size_t nf_l = 0, nf_p = 0;
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; int t = b->type, ar = T_ARITY[t]; int lslot = -1;
    for (int k = 0; k < ar; k++) if (T_CLS[t][k] != VC_POSE) { lslot = k; break; }
    if (lslot < 0) { nf_p += b->n; continue; }
    for (int i = 0; i < b->n; i++) { int g = W->lgrp[lmk_id(P, T_CLS[t][lslot], b->idx[(size_t)i*ar+lslot])]; W->g_fptr[g+1]++; nf_l++; }
  }
  for (int g = 0; g < ng; g++) W->g_fptr[g+1] += W->g_fptr[g];
  W->g_fac = malloc(sizeof(fref)*(nf_l+1)); W->pf = malloc(sizeof(fref)*(nf_p+1)); W->n_pf = 0;
  memcpy(cur, W->g_fptr, sizeof(int)*(ng+1));
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; int t = b->type, ar = T_ARITY[t]; int lslot = -1;
    for (int k = 0; k < ar; k++) if (T_CLS[t][k] != VC_POSE) { lslot = k; break; }
    for (int i = 0; i < b->n; i++) {
      fref f = { bi, i };
      if (lslot < 0) W->pf[W->n_pf++] = f;
      else { int g = W->lgrp[lmk_id(P, T_CLS[t][lslot], b->idx[(size_t)i*ar+lslot])]; W->g_fac[cur[g]++] = f; }
    }
  }
  /* bandwidth: max position spread within any group / pose-only factor */
  int maxspread = 0;
  for (int g = 0; g < ng; g++) {
    int lo = 1 << 30, hi = -1;
    for (int q = W->g_fptr[g]; q < W->g_fptr[g+1]; q++) {
      const orc_block* b = &P->blocks[W->g_fac[q].blk]; int t = b->type, ar = T_ARITY[t];
      for (int k = 0; k < ar; k++) if (T_CLS[t][k] == VC_POSE) { int p = W->pos[b->idx[(size_t)W->g_fac[q].i*ar+k]]; if (p < lo) lo = p; if (p > hi) hi = p; }
    }
    if (hi >= 0 && hi - lo > maxspread) maxspread = hi - lo;
  }
  for (int q = 0; q < W->n_pf; q++) {
    const orc_block* b = &P->blocks[W->pf[q].blk]; int ar = T_ARITY[b->type]; int lo = 1 << 30, hi = -1;
    for (int k = 0; k < ar; k++) { int p = W->pos[b->idx[(size_t)W->pf[q].i*ar+k]]; if (p < lo) lo = p; if (p > hi) hi = p; }
    if (hi - lo > maxspread) maxspread = hi - lo;
  }
  W->n = 6*P->n_pose; W->bw = 6*maxspread + 5; if (W->bw > W->n - 1) W->bw = W->n - 1; if (W->bw < 0) W->bw = 0;
  W->ld = W->bw + 1;
  W->A = calloc(P->n_blocks, sizeof(double*)); W->bv = calloc(P->n_blocks, sizeof(double*));
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; int d = T_DIM[b->type], jc = orc_type_jcols(b->type);
    W->A[bi] = malloc(sizeof(double)*((size_t)b->n*d*jc + 1)); W->bv[bi] = malloc(sizeof(double)*((size_t)b->n*d + 1));
  }
  free(uf); free(gid); free(cur);
  return W;
}
static void schur_free(const orc_problem* P, schur_ws* W) {
  for (int bi = 0; bi < P->n_blocks; bi++) { free(W->A[bi]); free(W->bv[bi]); }
  free(W->A); free(W->bv); free(W->ldim); free(W->lgrp); free(W->g_lptr); free(W->g_lmk); free(W->g_fptr);
  free(W->g_fac); free(W->pf); free(W->pos); free(W);
}
static void schur_linearize(const orc_problem* P, schur_ws* W) {
  for (int bi = 0; bi < P->n_blocks; bi++) orc_linearize_block(P, &P->blocks[bi], W->A[bi], W->bv[bi]);
}

/* add a dense symmetric contribution: rows/cols given as scalar indices in solver order */
static inline void band_add(double* AB, int ld, int i, int j, double v) {
  if (i < j) { int t = i; i = j; j = t; }
  double* p = AB + (size_t)j*ld + (i - j);
#pragma omp atomic
  *p += v;
}

#define MAXGP 256  /* max distinct pose variables touching one landmark group (a 128-frame hybrid track) */
#define MAXGL 96   /* max scalar landmark dims of one group */

/* Per-group quantities.  mode 0: accumulate reduced system into AB/gS.
 * mode 1: back-substitute delta_l given delta_p (dp, solver order), write into dl (per landmark offset). */
static int group_process(const orc_problem* P, const schur_ws* W, int g, double lambda, int mode,
                         double* AB, double* gS, const double* dp, double* dl_point, double* dl_flow) {
  int nlm = W->g_lptr[g+1] - W->g_lptr[g];
  int loff[64]; int nvl = 0;
  if (nlm > 64) return 2;
  const int* lm = W->g_lmk + W->g_lptr[g];
  for (int a = 0; a < nlm; a++) { loff[a] = nvl; nvl += W->ldim[lm[a]]; }
  if (nvl > MAXGL) return 2;
  int gp[MAXGP], ngp = 0;
  double V[MAXGL*MAXGL], gl[MAXGL];
  memset(V, 0, sizeof(double)*nvl*nvl); memset(gl, 0, sizeof(double)*nvl);
  int nf = W->g_fptr[g+1] - W->g_fptr[g];
  /* first pass: V, g_l, pose list */
  for (int q = 0; q < nf; q++) {
    fref f = W->g_fac[W->g_fptr[g]+q]; const orc_block* b = &P->blocks[f.blk];
    int t = b->type, ar = T_ARITY[t], d = T_DIM[t], jc = orc_type_jcols(t);
    const double* J = W->A[f.blk] + (size_t)f.i*d*jc; const double* bb = W->bv[f.blk] + (size_t)f.i*d;
    int coff = 0, lc[4], lo[4], nls = 0;
    for (int k = 0; k < ar; k++) {
      int c = T_CLS[t][k], ix = b->idx[(size_t)f.i*ar+k];
      if (c == VC_POSE) { int found = 0; for (int a = 0; a < ngp; a++) if (gp[a] == ix) { found = 1; break; } if (!found) { if (ngp >= MAXGP) return 2; gp[ngp++] = ix; } }
      else { int L = lmk_id(P, c, ix), a = 0; while (lm[a] != L) a++; lc[nls] = coff; lo[nls] = loff[a]; nls++; }
      coff += cls_dim(c);
    }
    for (int s1 = 0; s1 < nls; s1++) {
      int d1 = (t == ORC_FLOWPROJ2) ? 2 : 3;
      for (int a = 0; a < d1; a++) {
        double s = 0; for (int k = 0; k < d; k++) s += J[k*jc+lc[s1]+a]*bb[k];
        gl[lo[s1]+a] += s;
        for (int s2 = 0; s2 < nls; s2++) for (int e = 0; e < d1; e++) {
          double h = 0; for (int k = 0; k < d; k++) h += J[k*jc+lc[s1]+a]*J[k*jc+lc[s2]+e];
          V[(lo[s1]+a)*nvl + lo[s2]+e] += h;
        }
      }
    }
  }
  for (int a = 0; a < nvl; a++) V[a*nvl+a] += lambda;
  /* Cholesky V = L L^T (lower, in place) */
  for (int j = 0; j < nvl; j++) {
    double s = V[j*nvl+j]; for (int k = 0; k < j; k++) s -= V[j*nvl+k]*V[j*nvl+k];
    if (!(s > 0)) return 1;
    double dj = sqrt(s); V[j*nvl+j] = dj;
    for (int i = j+1; i < nvl; i++) { double u = V[i*nvl+j]; for (int k = 0; k < j; k++) u -= V[i*nvl+k]*V[j*nvl+k]; V[i*nvl+j] = u/dj; }
  }
  if (mode == 1) {
    /* delta_l = V^-1 (g_l - W^T dp),  W^T dp = sum_f B_f^T (A_f dp) */
    for (int q = 0; q < nf; q++) {
      fref f = W->g_fac[W->g_fptr[g]+q]; const orc_block* b = &P->blocks[f.blk];
      int t = b->type, ar = T_ARITY[t], d = T_DIM[t], jc = orc_type_jcols(t);
      const double* J = W->A[f.blk] + (size_t)f.i*d*jc;
      double u[6] = {0,0,0,0,0,0}; int coff = 0;
      for (int k = 0; k < ar; k++) { int c = T_CLS[t][k], ix = b->idx[(size_t)f.i*ar+k];
        if (c == VC_POSE) for (int r = 0; r < d; r++) for (int a = 0; a < 6; a++) u[r] += J[r*jc+coff+a]*dp[6*W->pos[ix]+a];
        coff += cls_dim(c); }
      coff = 0;
      for (int k = 0; k < ar; k++) { int c = T_CLS[t][k], ix = b->idx[(size_t)f.i*ar+k];
        if (c != VC_POSE) { int L = lmk_id(P, c, ix), a = 0; while (lm[a] != L) a++;
          for (int e = 0; e < cls_dim(c); e++) { double s = 0; for (int r = 0; r < d; r++) s += J[r*jc+coff+e]*u[r]; gl[loff[a]+e] -= s; } }
        coff += cls_dim(c); }
    }
    for (int i = 0; i < nvl; i++) { double s = gl[i]; for (int k = 0; k < i; k++) s -= V[i*nvl+k]*gl[k]; gl[i] = s/V[i*nvl+i]; }
    for (int i = nvl-1; i >= 0; i--) { double s = gl[i]; for (int k = i+1; k < nvl; k++) s -= V[k*nvl+i]*gl[k]; gl[i] = s/V[i*nvl+i]; }
    for (int a = 0; a < nlm; a++) { int L = lm[a];
      if (L < P->n_point) for (int e = 0; e < 3; e++) dl_point[3*(size_t)L+e] = gl[loff[a]+e];
      else for (int e = 0; e < 2; e++) dl_flow[2*(size_t)(L-P->n_point)+e] = gl[loff[a]+e]; }
    return 0;
  }
  /* mode 0: Wh = W L^-T  (6*ngp x nvl), S_local = sum A^T A - Wh Wh^T, g_local = sum A^T b - Wh y */
  int np6 = 6*ngp;
  /* per-thread scratch, grown on demand and zeroed per group (a calloc/free pair of several hundred KB per landmark goes
   * through mmap/munmap and dominated the elimination) */
  static __thread double* tl_buf = NULL; static __thread size_t tl_cap = 0;
  const size_t need = (size_t)np6*nvl + (size_t)np6*np6 + np6 + 1;
  if (need > tl_cap) { free(tl_buf); tl_cap = need + need/2; tl_buf = (double*)malloc(tl_cap*sizeof(double)); if (!tl_buf) { tl_cap = 0; return 2; } }
  double* Wm = tl_buf; memset(Wm, 0, need*sizeof(double));
  double* Sl = Wm + (size_t)np6*nvl; double* gloc = Sl + (size_t)np6*np6;
  for (int q = 0; q < nf; q++) {
    fref f = W->g_fac[W->g_fptr[g]+q]; const orc_block* b = &P->blocks[f.blk];
    int t = b->type, ar = T_ARITY[t], d = T_DIM[t], jc = orc_type_jcols(t);
    const double* J = W->A[f.blk] + (size_t)f.i*d*jc; const double* bb = W->bv[f.blk] + (size_t)f.i*d;
    int coff = 0, pc[4], po[4], npz = 0, lc[4], lo[4], ld_[4], nls = 0;
    for (int k = 0; k < ar; k++) { int c = T_CLS[t][k], ix = b->idx[(size_t)f.i*ar+k];
      if (c == VC_POSE) { int a = 0; while (gp[a] != ix) a++; pc[npz] = coff; po[npz] = 6*a; npz++; }
      else { int L = lmk_id(P, c, ix), a = 0; while (lm[a] != L) a++; lc[nls] = coff; lo[nls] = loff[a]; ld_[nls] = cls_dim(c); nls++; }
      coff += cls_dim(c); }
    for (int s1 = 0; s1 < npz; s1++) for (int a = 0; a < 6; a++) {
      double s = 0; for (int k = 0; k < d; k++) s += J[k*jc+pc[s1]+a]*bb[k];
      gloc[po[s1]+a] += s;
      for (int s2 = 0; s2 < npz; s2++) for (int e = 0; e < 6; e++) { double h = 0; for (int k = 0; k < d; k++) h += J[k*jc+pc[s1]+a]*J[k*jc+pc[s2]+e]; Sl[(size_t)(po[s1]+a)*np6 + po[s2]+e] += h; }
      for (int s2 = 0; s2 < nls; s2++) for (int e = 0; e < ld_[s2]; e++) { double h = 0; for (int k = 0; k < d; k++) h += J[k*jc+pc[s1]+a]*J[k*jc+lc[s2]+e]; Wm[(size_t)(po[s1]+a)*nvl + lo[s2]+e] += h; }
    }
  }
  /* y = L^-1 g_l */
  for (int i = 0; i < nvl; i++) { double s = gl[i]; for (int k = 0; k < i; k++) s -= V[i*nvl+k]*gl[k]; gl[i] = s/V[i*nvl+i]; }
  /* rows of Wm: solve x L^T = w  -> forward substitution along columns */
  for (int r = 0; r < np6; r++) { double* w = Wm + (size_t)r*nvl;
    for (int i = 0; i < nvl; i++) { double s = w[i]; for (int k = 0; k < i; k++) s -= V[i*nvl+k]*w[k]; w[i] = s/V[i*nvl+i]; } }
  for (int r = 0; r < np6; r++) { const double* wr = Wm + (size_t)r*nvl;
    double s = 0; for (int k = 0; k < nvl; k++) s += wr[k]*gl[k]; gloc[r] -= s;
    for (int c = 0; c <= r; c++) { const double* wc = Wm + (size_t)c*nvl; double h = 0; for (int k = 0; k < nvl; k++) h += wr[k]*wc[k]; Sl[(size_t)r*np6+c] -= h; } }
  for (int a = 0; a < ngp; a++) { int oa = 6*W->pos[gp[a]];
    for (int r = 0; r < 6; r++) {
      double* gp_ = gS + oa + r;
#pragma omp atomic
      *gp_ += gloc[6*a+r];
    }
    for (int c = 0; c < ngp; c++) { int oc = 6*W->pos[gp[c]];
      for (int r = 0; r < 6; r++) for (int e = 0; e < 6; e++) {
        int gi = oa + r, gj = oc + e; if (gi < gj) continue;           /* lower triangle only */
        int li = 6*a + r, lj = 6*c + e; double v = li >= lj ? Sl[(size_t)li*np6+lj] : Sl[(size_t)lj*np6+li];
        band_add(AB, W->ld, gi, gj, v);
      } } }
  return 0;
}

static void pose_factors_accumulate(const orc_problem* P, const schur_ws* W, double* AB, double* gS) {
  for (int q = 0; q < W->n_pf; q++) {
    fref f = W->pf[q]; const orc_block* b = &P->blocks[f.blk]; int t = b->type, ar = T_ARITY[t], d = T_DIM[t], jc = orc_type_jcols(t);
    const double* J = W->A[f.blk] + (size_t)f.i*d*jc; const double* bb = W->bv[f.blk] + (size_t)f.i*d;
    for (int k1 = 0; k1 < ar; k1++) { int o1 = 6*W->pos[b->idx[(size_t)f.i*ar+k1]];
      for (int a = 0; a < 6; a++) { double s = 0; for (int k = 0; k < d; k++) s += J[k*jc+6*k1+a]*bb[k]; gS[o1+a] += s;
        for (int k2 = 0; k2 < ar; k2++) { int o2 = 6*W->pos[b->idx[(size_t)f.i*ar+k2]];
          for (int e = 0; e < 6; e++) { if (o1 + a < o2 + e) continue; double h = 0; for (int k = 0; k < d; k++) h += J[k*jc+6*k1+a]*J[k*jc+6*k2+e]; AB[(size_t)(o2+e)*W->ld + (o1+a-o2-e)] += h; } } } }
  }
}

static int build_reduced(const orc_problem* P, const schur_ws* W, double lambda, double* AB, double* gS) {
  memset(AB, 0, sizeof(double)*(size_t)W->n*W->ld); memset(gS, 0, sizeof(double)*W->n);
  for (int i = 0; i < W->n; i++) AB[(size_t)i*W->ld] = lambda;
  pose_factors_accumulate(P, W, AB, gS);
  int fail = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(|:fail)
  for (int g = 0; g < W->n_grp; g++) fail |= group_process(P, W, g, lambda, 0, AB, gS, NULL, NULL, NULL);
  return fail;
}

/* banded Cholesky, lower band storage AB[j*ld + (i-j)], blocked right-looking.  returns 1 if not SPD */
static int band_cholesky(double* AB, int n, int bw, int ld) {
  const int NB = 32;
  for (int j0 = 0; j0 < n; j0 += NB) {
    int jb = n - j0 < NB ? n - j0 : NB;
    /* factor the diagonal block + panel columns, unblocked within the panel */
    for (int j = j0; j < j0 + jb; j++) {
      double* cj = AB + (size_t)j*ld;
      if (!(cj[0] > 0)) return 1;
      double dj = sqrt(cj[0]); cj[0] = dj;
      int m = n - 1 - j < bw ? n - 1 - j : bw;
      for (int i = 1; i <= m; i++) cj[i] /= dj;
      /* update the remaining columns of the panel only */
      int kend = j0 + jb - 1 - j; if (kend > m) kend = m;
      for (int k = 1; k <= kend; k++) { double l = cj[k]; double* ck = AB + (size_t)(j+k)*ld; for (int i = k; i <= m; i++) ck[i-k] -= cj[i]*l; }
    }
    /* trailing update with the whole panel: columns c in (j0+jb .. j0+jb-1+bw] */
    int cend = j0 + jb - 1 + bw; if (cend > n - 1) cend = n - 1;
#pragma omp parallel for schedule(static)
    for (int c = j0 + jb; c <= cend; c++) {
      double* cc = AB + (size_t)c*ld;
      for (int j = j0; j < j0 + jb; j++) {
        int off = c - j; if (off > bw) continue;
        const double* cj = AB + (size_t)j*ld; double l = cj[off];
        int m = n - 1 - j < bw ? n - 1 - j : bw;
        for (int i = off; i <= m; i++) cc[i-off] -= cj[i]*l;
      }
    }
  }
  return 0;
}
static void band_solve(const double* AB, int n, int bw, int ld, double* x) {
  for (int j = 0; j < n; j++) { const double* cj = AB + (size_t)j*ld; x[j] /= cj[0]; double xj = x[j];
    int m = n - 1 - j < bw ? n - 1 - j : bw; for (int i = 1; i <= m; i++) x[j+i] -= cj[i]*xj; }
  for (int j = n-1; j >= 0; j--) { const double* cj = AB + (size_t)j*ld; double s = x[j];
    int m = n - 1 - j < bw ? n - 1 - j : bw; for (int i = 1; i <= m; i++) s -= cj[i]*x[j+i]; x[j] = s/cj[0]; }
}

int orc_reduced_dense(const orc_problem* P, double lambda, double* S, double* gS, int32_t* pose_pos) {
  schur_ws* W = schur_setup(P); schur_linearize(P, W);
  double* AB = malloc(sizeof(double)*(size_t)W->n*W->ld);
  build_reduced(P, W, lambda, AB, gS);
  int n = W->n;
  memset(S, 0, sizeof(double)*(size_t)n*n);
  for (int j = 0; j < n; j++) for (int k = 0; k <= W->bw && j + k < n; k++) { double v = AB[(size_t)j*W->ld+k]; S[(size_t)(j+k)*n+j] = v; S[(size_t)j*n+j+k] = v; }
  for (int i = 0; i < P->n_pose; i++) pose_pos[i] = W->pos[i];
  free(AB); schur_free(P, W);
  return n;
}

static int solve_damped(const orc_problem* P, schur_ws* W, double lambda, double* AB, double* dp, double* dl_point, double* dl_flow, double* tm) {
  double t0 = 0, t1 = 0, t2 = 0;
#ifdef _OPENMP
  t0 = omp_get_wtime();
#endif
  if (build_reduced(P, W, lambda, AB, dp)) return 1;
#ifdef _OPENMP
  t1 = omp_get_wtime();
#endif
  if (band_cholesky(AB, W->n, W->bw, W->ld)) return 1;
  band_solve(AB, W->n, W->bw, W->ld, dp);
#ifdef _OPENMP
  t2 = omp_get_wtime();
#endif
  int fail = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(|:fail)
  for (int g = 0; g < W->n_grp; g++) fail |= group_process(P, W, g, lambda, 1, NULL, NULL, dp, dl_point, dl_flow);
  if (tm) {
    tm[0] += t1 - t0; tm[1] += t2 - t1;
#ifdef _OPENMP
    tm[2] += omp_get_wtime() - t2;
#endif
  }
  return fail;
}

int orc_schur_solve(const orc_problem* P, double lambda, double* delta) {
  schur_ws* W = schur_setup(P); schur_linearize(P, W);
  double* AB = malloc(sizeof(double)*(size_t)W->n*W->ld); double* dp = malloc(sizeof(double)*(W->n+1));
  double* dlp = delta + 6*(size_t)P->n_pose; double* dlf = dlp + 3*(size_t)P->n_point;
  int rc = solve_damped(P, W, lambda, AB, dp, dlp, dlf, NULL);
  for (int i = 0; i < P->n_pose; i++) for (int a = 0; a < 6; a++) delta[6*(size_t)i+a] = dp[6*(size_t)W->pos[i]+a];
  free(AB); free(dp); schur_free(P, W);
  return rc;
}

void orc_retract(orc_problem* P, const double* delta) {
#pragma omp parallel for schedule(static)
  for (int i = 0; i < P->n_pose; i++) { double o[12]; orc_se3_retract(P->pose + 12*(size_t)i, delta + 6*(size_t)i, o); memcpy(P->pose + 12*(size_t)i, o, sizeof(o)); }
  const double* dl = delta + 6*(size_t)P->n_pose;
  for (size_t i = 0; i < 3*(size_t)P->n_point; i++) P->point[i] += dl[i];
  dl += 3*(size_t)P->n_point;
  for (size_t i = 0; i < 2*(size_t)P->n_flow; i++) P->flow[i] += dl[i];
}

/* GaussianFactorGraph::error(delta) = sum 0.5 |A delta - b|^2 over the stored linearization */
static double linear_error(const orc_problem* P, const schur_ws* W, const double* delta) {
  double tot = 0;
  for (int bi = 0; bi < P->n_blocks; bi++) {
    const orc_block* b = &P->blocks[bi]; int t = b->type, ar = T_ARITY[t], d = T_DIM[t], jc = orc_type_jcols(t);
    double s = 0;
#pragma omp parallel for schedule(static) reduction(+:s)
    for (int i = 0; i < b->n; i++) {
      const double* J = W->A[bi] + (size_t)i*d*jc; const double* bb = W->bv[bi] + (size_t)i*d;
      double e[6]; for (int k = 0; k < d; k++) e[k] = -bb[k];
      if (delta) { int coff = 0;
        for (int k = 0; k < ar; k++) { int c = T_CLS[t][k]; const double* dv = delta + dense_off(P, c, b->idx[(size_t)i*ar+k]);
          for (int r = 0; r < d; r++) for (int a = 0; a < cls_dim(c); a++) e[r] += J[r*jc+coff+a]*dv[a];
          coff += cls_dim(c); } }
      double q = 0; for (int k = 0; k < d; k++) q += e[k]*e[k];
      s += 0.5*q;
    }
    tot += s;
  }
  return tot;
}

static double now_s(void) {
#ifdef _OPENMP
  return omp_get_wtime();
#else
  return 0.0;
#endif
}

int orc_lm_optimize(orc_problem* P, const orc_lm_params* prm, orc_lm_stats* st) {
  double T0 = now_s();
  schur_ws* W = schur_setup(P);
  size_t nd = (size_t)orc_dense_dim(P);
  double* AB = malloc(sizeof(double)*(size_t)W->n*W->ld);
  double* dp = malloc(sizeof(double)*(W->n+1)); double* delta = calloc(nd+1, sizeof(double));
  double* pose0 = malloc(sizeof(double)*12*(size_t)(P->n_pose+1)); double* pt0 = malloc(sizeof(double)*3*(size_t)(P->n_point+1));
  double* fl0 = malloc(sizeof(double)*2*(size_t)(P->n_flow+1));
  memset(st, 0, sizeof(*st)); st->bandwidth = W->bw; st->reduced_dim = W->n;
  double tm[3] = {0,0,0};
  double lambda = prm->lambda_initial, t;
  t = now_s(); double err = orc_error(P); st->t_error += now_s() - t;
  st->error_initial = err;
  int iterations = 0, inner = 0;
  if (!(err <= prm->err_tol) && prm->max_iterations > 0) {
    double newError = err, currentError;
    do {
      currentError = newError;
      /* iterate(): linearize once, then tryLambda until it returns true */
      t = now_s(); schur_linearize(P, W); st->t_linearize += now_s() - t;
      for (;;) {
        int solved = !solve_damped(P, W, lambda, AB, dp, delta + 6*(size_t)P->n_pose, delta + 6*(size_t)P->n_pose + 3*(size_t)P->n_point, tm);
        int success = 0, stop = 0; double nerr = INFINITY;
        if (solved) {
          for (int i = 0; i < P->n_pose; i++) for (int a = 0; a < 6; a++) delta[6*(size_t)i+a] = dp[6*(size_t)W->pos[i]+a];
          double oldLin = linear_error(P, W, NULL), newLin = linear_error(P, W, delta), lin = oldLin - newLin;
          if (lin >= 0) {
            memcpy(pose0, P->pose, sizeof(double)*12*(size_t)P->n_pose); memcpy(pt0, P->point, sizeof(double)*3*(size_t)P->n_point);
            if (P->n_flow) memcpy(fl0, P->flow, sizeof(double)*2*(size_t)P->n_flow);
            orc_retract(P, delta);
            t = now_s(); nerr = orc_error(P); st->t_error += now_s() - t;
            double cost = err - nerr;
            if (lin > DBL_EPSILON*oldLin) { double fid = cost/lin; success = fid > prm->min_model_fidelity; }
            if (fabs(cost) < prm->rel_tol*err) stop = 1;
            if (prm->verbose) fprintf(stderr, "[orc-lm] it %d inner %d lambda %.3e err %.12e -> %.12e lin %.6e %s\n", iterations, inner, lambda, err, nerr, lin, success ? "ok" : "rej");
            if (!success) { memcpy(P->pose, pose0, sizeof(double)*12*(size_t)P->n_pose); memcpy(P->point, pt0, sizeof(double)*3*(size_t)P->n_point);
              if (P->n_flow) memcpy(P->flow, fl0, sizeof(double)*2*(size_t)P->n_flow); }
          }
        }
        /* LevenbergMarquardtState::{decrease,increase}Lambda each count one inner iteration */
        if (success) { lambda /= prm->lambda_factor; if (lambda < prm->lambda_lower) lambda = prm->lambda_lower; err = nerr; iterations++; inner++; break; }
        else if (!stop) { lambda *= prm->lambda_factor; inner++; if (lambda >= prm->lambda_upper) break; }
        else break;
      }
      newError = err;
    } while (iterations < prm->max_iterations &&
             !((newError <= prm->err_tol) ||
               ((prm->rel_tol != 0.0) && ((currentError - newError)/currentError <= prm->rel_tol)) ||
               ((currentError - newError) <= prm->abs_tol)) &&
             isfinite(currentError));
  }
  st->iterations = iterations; st->inner_iterations = inner; st->error_final = err; st->lambda_final = lambda;
  st->t_schur = tm[0]; st->t_solve = tm[1]; st->t_backsub = tm[2]; st->t_total = now_s() - T0;
  free(AB); free(dp); free(delta); free(pose0); free(pt0); free(fl0); schur_free(P, W);
  return 0;
}
