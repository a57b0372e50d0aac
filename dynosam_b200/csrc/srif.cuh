// srif.cuh -- one object's step of ObjectMotionSolverFilter (dynosam/src/frontend/vision/MotionSolver.cc:1734-2063): the
// square-root information filter HybridObjectMotionSRIF (:1395-1725) over the key-framed object motion H = H_W_e_k.
//
// State (DYNOBA_SRIF_STATE doubles, include/dynoba.h): R (6x6 upper, row-major) | d (6) | H_lin | L_e | prev_H | X_K (12 each,
// R row-major | t).  The tangent is GTSAM's [omega; v] and retract(T, x) = T Expmap(x) (se3.cuh).
//
//   mean            H_mean = retract(H_lin, R^-1 d)
//   reset(L_e)      R = chol_upper(P0^-1), d = 0, H_lin = prev_H = X_K = I                                 (:1689-1725)
//   predict         P = (R^T R)^-1;  F2F = H_mean prev_H^-1;  prev_H = H_mean;  H_lin = F2F H_mean;  d = 0;
//                   R = chol_upper((P + Q)^-1).  Its pose argument is never used by the reference.      (:1445-1482)
//   update(X, z)    X_K = X.  At the linearisation point, A = X^-1 H_lin, camera C = (A L_e)^-1:          (:1484-1687)
//                     a tracklet without a point gets m = L_e^-1 H_lin^-1 X p_cam (projectToObject3) BEFORE the stereo
//                     test; with valid stereo and q = C^-1 m in front of the camera (q_z > 0), its rows are
//                     J = J_pi (-Ad(A)), y = z - h (J_pi: StereoCamera::project2's pose derivative), error e0 = |y|_Rn;
//                     otherwise its rows stay zero.
//                   IRLS, irls_iterations times: project at retract(H_lin, R^-1 d); weight 1 if e <= k else k/e with
//                     e^2 = y^T Rn^-1 y (0 for invalid stereo or cheirality; the reweighted error of a point is written only
//                     when it projects and is never reset within the update); rows with w < 1e-6 are dropped, the others
//                     premultiplied by chol_lower(Rn / w)^-1; [R | d] = the triangle of the QR of the rows stacked over
//                     the update's ORIGINAL prior [R0 | d0].
//                   error = |e0|, reweighted_error = |reweighted errors|.
// A QR factor is unique up to the signs of its rows; R is returned with a non-negative diagonal (every observable --
// R^-1 d, R^T R, the poses -- is invariant to those signs).
//
// The functions below are the sequential statement; kernels_srif.cu runs the same per-correspondence functions one thread
// per correspondence and the QR as a warp-parallel TSQR.  tests/capi/srif_host.cu compiles this header for the host.
#pragma once
#include "factors.cuh"
#include "../../include/dynoba.h"

namespace dynoba {

constexpr int SRIF_R = 0, SRIF_D = 36, SRIF_H = 42, SRIF_LE = 54, SRIF_PREV = 66, SRIF_XK = 78;
constexpr int SRIF_LIN = 21;          // one correspondence at the linearisation point: 3 rows of [J (6) | y]
constexpr double SRIF_MIN_W = 1e-6;   // MotionSolver.cc:1643
static_assert(SRIF_XK + 12 == DYNOBA_SRIF_STATE, "state layout");

DYN_HD void srif_pose_ld(const double* p, Pose& P) {
  for (int i = 0; i < 9; i++) P.R[i] = p[i];
  for (int i = 0; i < 3; i++) P.t[i] = p[9 + i];
}
DYN_HD void srif_pose_st(const Pose& P, double* p) {
  for (int i = 0; i < 9; i++) p[i] = P.R[i];
  for (int i = 0; i < 3; i++) p[9 + i] = P.t[i];
}
DYN_HD void srif_eye(double* p) { for (int i = 0; i < 12; i++) p[i] = (i == 0 || i == 4 || i == 8) ? 1.0 : 0.0; }

// A = L L^T from A's lower triangle (N x N row-major); false unless every pivot is positive
template <int N>
DYN_HD bool srif_chol(const double* A, double* L) {
  for (int i = 0; i < N*N; i++) L[i] = 0.0;
  for (int j = 0; j < N; j++) {
    double s = A[j*N + j];
    for (int k = 0; k < j; k++) s -= L[j*N + k]*L[j*N + k];
    if (!(s > 0.0)) return false;
    const double l = sqrt(s);
    L[j*N + j] = l;
    for (int i = j + 1; i < N; i++) {
      double t = A[i*N + j];
      for (int k = 0; k < j; k++) t -= L[i*N + k]*L[j*N + k];
      L[i*N + j] = t/l;
    }
  }
  return true;
}
// inverse of a lower-triangular L
template <int N>
DYN_HD void srif_lower_inv(const double* L, double* Li) {
  for (int i = 0; i < N*N; i++) Li[i] = 0.0;
  for (int j = 0; j < N; j++) {
    Li[j*N + j] = 1.0/L[j*N + j];
    for (int i = j + 1; i < N; i++) {
      double s = 0.0;
      for (int k = j; k < i; k++) s -= L[i*N + k]*Li[k*N + j];
      Li[i*N + j] = s/L[i*N + i];
    }
  }
}
// W = Li^T Li for a lower-triangular Li
DYN_HD void srif_gram_t(const double* Li, double* W) {
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) {
      double s = 0.0;
      for (int k = (i > j ? i : j); k < 6; k++) s += Li[k*6 + i]*Li[k*6 + j];
      W[i*6 + j] = s;
    }
}
// R upper with R^T R = M^-1 for an SPD M (the reference's M.inverse().llt().matrixU())
DYN_HD bool srif_info_root(const double* M, double* R) {
  double L[36], Li[36], W[36];
  if (!srif_chol<6>(M, L)) return false;
  srif_lower_inv<6>(L, Li);
  srif_gram_t(Li, W);
  if (!srif_chol<6>(W, L)) return false;
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) R[i*6 + j] = L[j*6 + i];
  return true;
}
// (R^T R)^-1 = R^-1 R^-T
DYN_HD void srif_cov(const double* R, double* P) {
  double Lt[36], Li[36];
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) Lt[i*6 + j] = R[j*6 + i];
  srif_lower_inv<6>(Lt, Li);                  // Li = R^-T
  srif_gram_t(Li, P);
}
// R x = d by back-substitution
DYN_HD void srif_delta(const double* R, const double* d, double* x) {
  for (int i = 5; i >= 0; i--) {
    double s = d[i];
    for (int k = i + 1; k < 6; k++) s -= R[i*6 + k]*x[k];
    x[i] = s/R[i*6 + i];
  }
}
DYN_HD void srif_mean(const double* st, Pose& Hm) {
  Pose H; srif_pose_ld(st + SRIF_H, H);
  double x[6]; srif_delta(st + SRIF_R, st + SRIF_D, x);
  se3_retract(H, x, Hm);
}
// 3x3 inverse by cofactors (the reference's R.inverse() of the measurement covariance)
DYN_HD void srif_inv3(const double* A, double* B) {
  const double c0 = A[4]*A[8] - A[5]*A[7], c1 = A[5]*A[6] - A[3]*A[8], c2 = A[3]*A[7] - A[4]*A[6];
  const double det = A[0]*c0 + A[1]*c1 + A[2]*c2;
  B[0] = c0/det; B[1] = (A[2]*A[7] - A[1]*A[8])/det; B[2] = (A[1]*A[5] - A[2]*A[4])/det;
  B[3] = c1/det; B[4] = (A[0]*A[8] - A[2]*A[6])/det; B[5] = (A[2]*A[3] - A[0]*A[5])/det;
  B[6] = c2/det; B[7] = (A[1]*A[6] - A[0]*A[7])/det; B[8] = (A[0]*A[4] - A[1]*A[3])/det;
}

// construct_initial_frame (:1768-1787): L_e = (I, X_k-1 * sum / n)
DYN_HD void srif_keyframe(const Pose& Xp, const double* sum, int n, Pose& Le) {
  const double c[3] = { sum[0]/n, sum[1]/n, sum[2]/n };
  for (int i = 0; i < 9; i++) Le.R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  se3_transform_from(Xp, c, Le.t);
}
DYN_HD void srif_reset(double* st, const double* P0, const Pose& Le) {
  srif_info_root(P0, st + SRIF_R);
  for (int i = 0; i < 6; i++) st[SRIF_D + i] = 0.0;
  srif_eye(st + SRIF_H); srif_eye(st + SRIF_PREV); srif_eye(st + SRIF_XK);
  srif_pose_st(Le, st + SRIF_LE);
}
DYN_HD void srif_predict(double* st, const double* Q) {
  Pose Hm, prev, pinv, F, Hn;
  srif_mean(st, Hm);
  srif_pose_ld(st + SRIF_PREV, prev);
  double P[36]; srif_cov(st + SRIF_R, P);
  for (int i = 0; i < 36; i++) P[i] += Q[i];
  se3_inverse(prev, pinv); se3_compose(Hm, pinv, F);
  se3_compose(F, Hm, Hn);
  srif_pose_st(Hm, st + SRIF_PREV);
  srif_pose_st(Hn, st + SRIF_H);
  for (int i = 0; i < 6; i++) st[SRIF_D + i] = 0.0;
  srif_info_root(P, st + SRIF_R);
}

// the stereo camera of the update, C = (X^-1 H L_e)^-1, and (if nAd) -Ad(X^-1 H)
DYN_HD void srif_camera(const Pose& X, const Pose& H, const Pose& Le, Pose& C, double* nAd) {
  Pose Xi, A, G;
  se3_inverse(X, Xi); se3_compose(Xi, H, A); se3_compose(A, Le, G); se3_inverse(G, C);
  if (nAd) {
    se3_adjoint(A, nAd);
    for (int i = 0; i < 36; i++) nAd[i] = -nAd[i];
  }
}
// HybridObjectMotion::projectToObject3 (HybridFormulationFactors.cc:37-60): L_e^-1 H^-1 X p
DYN_HD void srif_init_point(const Pose& X, const Pose& H, const Pose& Le, const double* pc, double* m) {
  Pose Li, Hi, T1, T2;
  se3_inverse(Le, Li); se3_inverse(H, Hi); se3_compose(Li, Hi, T1); se3_compose(T1, X, T2);
  se3_transform_from(T2, pc, m);
}
// StereoCamera(C, K).project2(m): y = z - h and (if Jpi) the 3x6 derivative by the camera pose (as STEREO3); false on
// cheirality.  K = (fx, fy, skew, u0, v0, baseline); StereoCamera ignores the skew.
DYN_HD bool srif_project(const Pose& C, const double* K, const double* z, const double* m, double* y, double* Jpi) {
  double q[3], h[3], Dq[9];
  se3_transform_to(C, m, q);
  if (!stereo_project(K, q, h, Dq)) return false;
  for (int r = 0; r < 3; r++) y[r] = z[r] - h[r];
  if (Jpi) {
    const double Dp[18] = { 0, -q[2], q[1], -1, 0, 0,  q[2], 0, -q[0], 0, -1, 0,  -q[1], q[0], 0, 0, 0, -1 };
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 6; c++) Jpi[6*r + c] = Dq[3*r]*Dp[c] + Dq[3*r + 1]*Dp[6 + c] + Dq[3*r + 2]*Dp[12 + c];
  }
  return true;
}
// e = sqrt(y^T Rn^-1 y)
DYN_HD double srif_mahal(const double* y, const double* Rinv) {
  double s = 0.0;
  for (int c = 0; c < 3; c++) s += (y[0]*Rinv[c] + y[1]*Rinv[3 + c] + y[2]*Rinv[6 + c])*y[c];
  return sqrt(s);
}
// Huber weight (:1630); clipped = the measurement was scaled down
DYN_HD double srif_huber(double e, double k, bool* clipped) {
  const bool inside = e <= k;
  *clipped = !inside;
  return inside ? 1.0 : k/e;
}

// One correspondence at the linearisation point (:1512-1565).  Returns whether its point was initialised here.
DYN_HD bool srif_lin_one(const Pose& X, const Pose& H, const Pose& Le, const Pose& C, const double* nAd, const double* K,
                         const double* Rinv, const double* z, bool valid, const double* pc, double* m, uint8_t* has,
                         double* rows, double* e0) {
  bool fresh = false;
  if (!*has) { srif_init_point(X, H, Le, pc, m); *has = 1; fresh = true; }
  for (int e = 0; e < SRIF_LIN; e++) rows[e] = 0.0;
  *e0 = 0.0;
  if (!valid) return fresh;
  double y[3], Jpi[18];
  if (!srif_project(C, K, z, m, y, Jpi)) return fresh;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 6; c++) {
      double s = 0.0;
      for (int k = 0; k < 6; k++) s += Jpi[6*r + k]*nAd[6*k + c];
      rows[7*r + c] = s;
    }
    rows[7*r + 6] = y[r];
  }
  *e0 = srif_mahal(y, Rinv);
  return fresh;
}
// One correspondence's IRLS weight at the current mean (:1594-1635); writes its reweighted error when it projects.
DYN_HD double srif_weight_one(const Pose& C, const double* K, const double* Rinv, double huber_k, const double* z, bool valid,
                              const double* m, double* rwe, bool* clipped) {
  *clipped = false;
  if (!valid) return 0.0;
  double y[3];
  if (!srif_project(C, K, z, m, y, nullptr)) return 0.0;
  const double e = srif_mahal(y, Rinv);
  *rwe = e;
  return srif_huber(e, huber_k, clipped);
}
// row r of chol_lower(Rn / w)^-1 [J | y] (:1645-1659)
DYN_HD void srif_whiten_row(const double* Rn, double w, const double* rows, int r, double* out) {
  double A[9], L[9], Li[9];
  for (int i = 0; i < 9; i++) A[i] = Rn[i]/w;
  srif_chol<3>(A, L);
  srif_lower_inv<3>(L, Li);
  for (int c = 0; c < 7; c++) out[c] = Li[3*r]*rows[c] + Li[3*r + 1]*rows[7 + c] + Li[3*r + 2]*rows[14 + c];
}

// Householder QR of [T (7 x 7 upper) ; rows (nr x 7)] -> T (LAPACK dlarfg reflectors; a column with nothing below its
// diagonal is left alone)
DYN_HD void srif_fold(double* T, const double* rows, int nr) {
  double A[10*7];
  for (int i = 0; i < 49; i++) A[i] = T[i];
  for (int i = 0; i < 7*nr; i++) A[49 + i] = rows[i];
  const int M = 7 + nr;
  for (int j = 0; j < 7; j++) {
    double s = 0.0;
    for (int i = j + 1; i < M; i++) s += A[7*i + j]*A[7*i + j];
    if (s == 0.0) continue;
    const double alpha = A[7*j + j], nrm = sqrt(alpha*alpha + s), beta = alpha >= 0.0 ? -nrm : nrm;
    const double tau = (beta - alpha)/beta, sc = 1.0/(alpha - beta);
    double v[10];
    for (int i = j + 1; i < M; i++) v[i] = A[7*i + j]*sc;
    for (int c = j + 1; c < 7; c++) {
      double w = A[7*j + c];
      for (int i = j + 1; i < M; i++) w += v[i]*A[7*i + c];
      w *= tau;
      A[7*j + c] -= w;
      for (int i = j + 1; i < M; i++) A[7*i + c] -= v[i]*w;
    }
    A[7*j + j] = beta;
    for (int i = j + 1; i < M; i++) A[7*i + j] = 0.0;
  }
  for (int i = 0; i < 49; i++) T[i] = A[i];
}
// [R | d] of the triangle, rows signed to a non-negative diagonal
DYN_HD void srif_take_row(const double* Trow, int r, double* st) {
  const double sg = Trow[r] < 0.0 ? -1.0 : 1.0;
  for (int c = 0; c < 6; c++) st[SRIF_R + 6*r + c] = c < r ? 0.0 : sg*Trow[c];
  st[SRIF_D + r] = sg*Trow[6];
}

// outputs of a step: F2F motion, key-framed motion, object pose (updatePoses, :2065-2078), covariance
DYN_HD void srif_outputs(const double* st, double* motion, double* cov) {
  Pose Hm, prev, pinv, F, Le, L;
  srif_mean(st, Hm);
  srif_pose_ld(st + SRIF_PREV, prev); srif_pose_ld(st + SRIF_LE, Le);
  se3_inverse(prev, pinv); se3_compose(Hm, pinv, F); se3_compose(Hm, Le, L);
  srif_pose_st(F, motion); srif_pose_st(Hm, motion + 12); srif_pose_st(L, motion + 24);
  srif_cov(st + SRIF_R, cov);
}
// the admission of an object (solveImpl :1867-1891, and the zero-inlier key frame)
DYN_HD int srif_admit(int mode, int n, int min_new_inliers) {
  if (mode == DYNOBA_SRIF_NEW && n < min_new_inliers) return DYNOBA_SRIF_TOO_FEW;
  if (mode != DYNOBA_SRIF_CONTINUE && n == 0) return DYNOBA_SRIF_NO_INLIERS;
  return DYNOBA_SRIF_OK;
}

// ---- the sequential statement of one object's step (the host build runs it; kernels_srif.cu parallelises it)
struct SrifObject {                  // the object's slices of the batch arrays
  int mode, n, pnp_status;
  const double *Xp, *Xc, *K;         // [12], [12], [6]
  const double* z; const uint8_t* valid; const double* pc;    // [n][6], [n][2], [n][6]
  double* m; uint8_t* has;           // [n][3], [n]
};
struct SrifOut { int status, solved, n_new, n_clipped; double motion[36], cov[36], error, rerror, before[12]; };

// update(frame f) over the object (:1484-1687); lin [n][21], e0 / rwe [n] scratch
DYN_HD void srif_update_seq(double* st, const SrifObject& o, int f, const dynoba_object_srif_params& P, const double* Rinv,
                            double* lin, double* e0, double* rwe, SrifOut& out) {
  Pose X, H, Le, C; double nAd[36];
  srif_pose_ld(f == 0 ? o.Xp : o.Xc, X); srif_pose_ld(st + SRIF_H, H); srif_pose_ld(st + SRIF_LE, Le);
  srif_pose_st(X, st + SRIF_XK);
  srif_camera(X, H, Le, C, nAd);
  for (int i = 0; i < o.n; i++) {
    out.n_new += srif_lin_one(X, H, Le, C, nAd, o.K, Rinv, o.z + 6*i + 3*f, o.valid[2*i + f] != 0, o.pc + 6*i + 3*f,
                              o.m + 3*i, o.has + i, lin + SRIF_LIN*i, e0 + i);
    rwe[i] = 0.0;
  }
  double prior[42];
  for (int i = 0; i < 42; i++) prior[i] = st[i];
  for (int it = 0; it < P.irls_iterations; it++) {
    Pose Hc; srif_mean(st, Hc); srif_camera(X, Hc, Le, C, nullptr);
    double T[49];
    for (int r = 0; r < 7; r++)
      for (int c = 0; c < 7; c++) T[7*r + c] = r < 6 ? (c < 6 ? prior[SRIF_R + 6*r + c] : prior[SRIF_D + r]) : 0.0;
    out.n_clipped = 0;
    for (int i = 0; i < o.n; i++) {
      bool clipped;
      const double w = srif_weight_one(C, o.K, Rinv, P.huber_k, o.z + 6*i + 3*f, o.valid[2*i + f] != 0, o.m + 3*i, rwe + i, &clipped);
      out.n_clipped += clipped;
      if (w < SRIF_MIN_W) continue;
      double rows[21];
      for (int r = 0; r < 3; r++) srif_whiten_row(P.R_noise, w, lin + SRIF_LIN*i, r, rows + 7*r);
      srif_fold(T, rows, 3);
    }
    for (int r = 0; r < 6; r++) srif_take_row(T + 7*r, r, st);
  }
  double s0 = 0.0, s1 = 0.0;
  for (int i = 0; i < o.n; i++) { s0 += e0[i]*e0[i]; s1 += rwe[i]*rwe[i]; }
  out.error = sqrt(s0); out.rerror = sqrt(s1);
}

// one object's step for the frame: admission, key frame / reset, [predict, update(k-1)], predict, update(k), outputs
DYN_HD void srif_object_seq(const double* st_in, double* st, const SrifObject& o, const dynoba_object_srif_params& P,
                            const double* Rinv, double* lin, double* e0, double* rwe, SrifOut& out) {
  for (int i = 0; i < DYNOBA_SRIF_STATE; i++) st[i] = st_in[i];
  out.status = srif_admit(o.mode, o.n, P.min_new_inliers);
  out.solved = 0; out.n_new = 0; out.n_clipped = 0; out.error = out.rerror = 0.0;
  srif_eye(out.before);
  for (int i = 0; i < 36; i++) out.motion[i] = (i % 12 == 0 || i % 12 == 4 || i % 12 == 8) ? 1.0 : 0.0;
  for (int i = 0; i < 36; i++) out.cov[i] = 0.0;
  if (out.status != DYNOBA_SRIF_OK) return;
  if (o.mode != DYNOBA_SRIF_CONTINUE) {
    Pose Xp, Le; srif_pose_ld(o.Xp, Xp);
    double sum[3] = { 0.0, 0.0, 0.0 };
    for (int i = 0; i < o.n; i++) for (int c = 0; c < 3; c++) sum[c] += o.pc[6*i + c];
    srif_keyframe(Xp, sum, o.n, Le);
    if (o.mode == DYNOBA_SRIF_RESET) for (int i = 0; i < 12; i++) out.before[i] = st[SRIF_H + i];
    srif_reset(st, P.P0, Le);
    for (int i = 0; i < o.n; i++) o.has[i] = 0;
  }
  for (int f = o.mode == DYNOBA_SRIF_CONTINUE ? 1 : 0; f < 2; f++) {
    srif_predict(st, P.Q);
    srif_update_seq(st, o, f, P, Rinv, lin, e0, rwe, out);
  }
  srif_outputs(st, out.motion, out.cov);
  out.solved = o.pnp_status == DYNOBA_TRACK_VALID;
}

}  // namespace dynoba
