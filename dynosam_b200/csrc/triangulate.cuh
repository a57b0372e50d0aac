// triangulate.cuh -- one landmark's triangulation as the reference's stereo formulation runs it
// (StaticFormulationUpdater::StereoProjection::addLandmark, dynosam/include/dynosam/backend/Formulation-impl.hpp:258-411):
// gtsam::triangulateSafe over a set of pinhole cameras with default TriangulationParameters, then the 3 px test on the norm
// of the stacked reprojection errors.  The GTSAM 4.2.0 parts are restated from upstream [GTSAM-ext geometry/triangulation.h,
// triangulation.cpp, base/Matrix.cpp DLT]:
//
//   cameras        PinholeCamera<Cal3_S2>(X_c, K), K = [fx s u0; 0 fy v0; 0 0 1]; measurement (x_c, y_c).
//   degenerate     fewer than 2 cameras.
//   DLT            P_c = K [R_c^T | -R_c^T t_c];  A (2m x 4) has rows x_c P_c[2] - P_c[0] and y_c P_c[2] - P_c[1].
//                  SVD of A: rank = #{ sigma_j > rank_tol } (rankTolerance 1.0), rank < 3 is degenerate; v = the right singular
//                  vector of the smallest singular value, point = v[0:3] / v[3].  No nonlinear refinement (enableEPI false),
//                  no distance or outlier threshold inside triangulateSafe, no LOST.
//   cheirality     (GTSAM_THROW_CHEIRALITY_EXCEPTION) z of R_c^T (point - t_c) <= 0 in any camera: behind camera.
//   outlier        |stacked (project_c(point) - (x_c, y_c))|_2 > reproj_threshold (the reference's 3.0), project_c(p) =
//                  (fx x + s y + u0, fy y + v0) with (x, y, 1) ~ R_c^T (p - t_c).
// One divergence: where v[3] == 0 (or the quotient is not finite) the reference goes on with a point at infinity, whose
// depths and reprojection errors are NaN and so pass both tests; here the problem is DEGENERATE.
//
// The SVD is a one-sided (Hestenes) Jacobi SVD on A's four columns with A held implicitly: V (4x4) accumulates the
// rotations and column j of the rotated matrix is A V[:, j].  Pairs run in the fixed cyclic order (0,1) (0,2) (0,3) (1,2)
// (1,3) (2,3); pair (p, q) is rotated unless |a_p . a_q| <= TRI_TOL |a_p| |a_q|; the sweeps stop after the first sweep
// that rotates no pair, or after TRI_MAX_SWEEPS.  sigma_j = |A V[:, j]|.
//
// Every sum over A's rows is fixed-order: row r belongs to lane r mod 32, each lane sums its rows in row order, and the 32
// partial sums meet in the butterfly tree of __shfl_xor_sync (offsets 16, 8, 4, 2, 1).  kernels_triangulate.cu runs that tree
// on a warp; tri_solve below runs the same tree over 32 emulated lanes, so that the host build (the builder's CPU path,
// tests/capi/triangulate_host.cu) performs the same operations in the same order.  With multiply-add contraction off
// (kernels_triangulate.cu is compiled with -fmad=false; only the explicit operations below round) the two agree bit for bit.
#pragma once
#include <cmath>
#include "se3.cuh"
#include "../../include/dynoba.h"

namespace dynoba {

constexpr int TRI_LANES = 32;
constexpr int TRI_MAX_SWEEPS = 30;
constexpr double TRI_TOL = 8.0*2.220446049250313e-16;

// the two rows of A of one camera: X[12] (R row-major | t), K5 = fx fy s u0 v0, kp = (x, y)
DYN_HD void tri_rows(const double* X, const double* K5, const double* kp, double* r0, double* r1) {
  double M[12];                                                     // [R^T | -R^T t]
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) M[4*i + j] = X[3*j + i];
    M[4*i + 3] = -(X[i]*X[9] + X[3 + i]*X[10] + X[6 + i]*X[11]);
  }
  const double fx = K5[0], fy = K5[1], s = K5[2], u0 = K5[3], v0 = K5[4];
  for (int j = 0; j < 4; j++) {
    const double P0 = fx*M[j] + s*M[4 + j] + u0*M[8 + j], P1 = fy*M[4 + j] + v0*M[8 + j], P2 = M[8 + j];
    r0[j] = kp[0]*P2 - P0;
    r1[j] = kp[1]*P2 - P1;
  }
}

DYN_HD double tri_dot4(const double* a, const double* V, int j) {
  return a[0]*V[j] + a[1]*V[4 + j] + a[2]*V[8 + j] + a[3]*V[12 + j];
}

// one Jacobi rotation of columns p, q of V from alpha = |a_p|^2, beta = |a_q|^2, gamma = a_p . a_q; false if the pair is
// already orthogonal to TRI_TOL
DYN_HD bool tri_rotate(double alpha, double beta, double gamma, double* V, int p, int q) {
  if (!(std::fabs(gamma) > TRI_TOL*sqrt(alpha)*sqrt(beta))) return false;
  const double zeta = (beta - alpha)/(2.0*gamma);
  const double t = (zeta >= 0.0 ? 1.0 : -1.0)/(std::fabs(zeta) + sqrt(1.0 + zeta*zeta));
  const double c = 1.0/sqrt(1.0 + t*t), s = c*t;
  for (int i = 0; i < 4; i++) {
    const double vp = V[4*i + p], vq = V[4*i + q];
    V[4*i + p] = c*vp - s*vq;
    V[4*i + q] = s*vp + c*vq;
  }
  return true;
}

// depth of p in camera X (the z of R^T (p - t)) and, if it is positive, the squared reprojection error against kp
DYN_HD double tri_depth_err(const double* X, const double* K5, const double* kp, const double* p, double* e2) {
  const double d0 = p[0] - X[9], d1 = p[1] - X[10], d2 = p[2] - X[11];
  const double q0 = X[0]*d0 + X[3]*d1 + X[6]*d2, q1 = X[1]*d0 + X[4]*d1 + X[7]*d2, q2 = X[2]*d0 + X[5]*d1 + X[8]*d2;
  *e2 = 0.0;
  if (q2 > 0.0) {
    const double x = q0/q2, y = q1/q2;
    const double eu = (K5[0]*x + K5[2]*y + K5[3]) - kp[0], ev = (K5[1]*y + K5[4]) - kp[1];
    *e2 = eu*eu + ev*ev;
  }
  return q2;
}

struct TriOut { int status; double point[3]; double reproj; double sv[4]; };

// One problem: m cameras X[m][12], key-points kp[m][2]; A[2m][4] is scratch.  `lanes` runs per-lane work and reduces partial
// sums over the lanes: lanes.each(f) runs f(lane) for every lane; lanes.template sum<N>(f, out) has f(lane, part[N]) fill
// the lane's N partial sums and out[N] receive the N totals (kernels_triangulate.cu: the warp's shuffle tree; TriHostLanes:
// the same tree over emulated lanes).  Each lane writes and reads only its own rows of A.  The control flow depends only on
// reduced values, so it is uniform over a warp.
template <class Lanes>
DYN_HD void tri_solve(int m, const double* X, const double* kp, const double* K5, double rank_tol, double thr, double* A, Lanes& lanes,
                      TriOut& o) {
  const double nan = (double)NAN;
  o.reproj = nan;
  for (int k = 0; k < 3; k++) o.point[k] = nan;
  for (int k = 0; k < 4; k++) o.sv[k] = nan;
  if (m < 2) { o.status = DYNOBA_TRI_DEGENERATE; return; }
  const int rows = 2*m;
  lanes.each([&](int lane) {                                        // the lane's rows of A
    for (int r = lane; r < rows; r += TRI_LANES) {
      double r0[4], r1[4];
      tri_rows(X + 12*(r >> 1), K5, kp + 2*(r >> 1), r0, r1);
      for (int j = 0; j < 4; j++) A[4*r + j] = (r & 1) ? r1[j] : r0[j];
    }
  });
  double V[16];
  for (int i = 0; i < 16; i++) V[i] = (i % 5 == 0) ? 1.0 : 0.0;
  const int PP[6] = {0, 0, 0, 1, 1, 2}, QQ[6] = {1, 2, 3, 2, 3, 3};
  for (int sweep = 0; sweep < TRI_MAX_SWEEPS; sweep++) {
    bool rotated = false;
#pragma unroll
    for (int k = 0; k < 6; k++) {
      const int p = PP[k], q = QQ[k];
      double d[3];
      lanes.template sum<3>([&](int lane, double* part) {
        double a = 0.0, b = 0.0, c = 0.0;
        for (int r = lane; r < rows; r += TRI_LANES) {
          const double ap = tri_dot4(A + 4*r, V, p), aq = tri_dot4(A + 4*r, V, q);
          a += ap*ap; b += aq*aq; c += ap*aq;
        }
        part[0] = a; part[1] = b; part[2] = c;
      }, d);
      rotated = tri_rotate(d[0], d[1], d[2], V, p, q) || rotated;
    }
    if (!rotated) break;
  }
  double s2[4];
  lanes.template sum<4>([&](int lane, double* part) {
    for (int j = 0; j < 4; j++) part[j] = 0.0;
    for (int r = lane; r < rows; r += TRI_LANES)
      for (int j = 0; j < 4; j++) { const double a = tri_dot4(A + 4*r, V, j); part[j] += a*a; }
  }, s2);
  double sg[4]; int rank = 0, jmin = 0;
  for (int j = 0; j < 4; j++) { sg[j] = sqrt(s2[j]); if (sg[j] > rank_tol) rank++; if (sg[j] < sg[jmin]) jmin = j; }
  for (int k = 0; k < 4; k++) {                                     // descending, as JacobiSVD returns them
    int best = -1;
    for (int j = 0; j < 4; j++) {
      int before = 0;                                               // rank of sg[j] in descending order, ties by index
      for (int i = 0; i < 4; i++) before += (sg[i] > sg[j]) || (sg[i] == sg[j] && i < j);
      if (before == k) best = j;
    }
    o.sv[k] = sg[best];
  }
  if (rank < 3) { o.status = DYNOBA_TRI_DEGENERATE; return; }
  double v[4];                                                      // V[:, jmin], selected without indexing V at run time
  for (int k = 0; k < 4; k++) v[k] = jmin == 0 ? V[4*k] : jmin == 1 ? V[4*k + 1] : jmin == 2 ? V[4*k + 2] : V[4*k + 3];
  double p[3];
  for (int k = 0; k < 3; k++) p[k] = v[k]/v[3];
  for (int k = 0; k < 3; k++) o.point[k] = p[k];
  if (!(std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]))) { o.status = DYNOBA_TRI_DEGENERATE; return; }
  double ce[2];
  lanes.template sum<2>([&](int lane, double* part) {
    double behind = 0.0, e = 0.0;
    for (int c = lane; c < m; c += TRI_LANES) {
      double e2;
      if (tri_depth_err(X + 12*c, K5, kp + 2*c, p, &e2) <= 0.0) behind += 1.0;
      e += e2;
    }
    part[0] = behind; part[1] = e;
  }, ce);
  if (ce[0] > 0.0) { o.status = DYNOBA_TRI_BEHIND_CAMERA; return; }
  o.reproj = sqrt(ce[1]);
  o.status = (o.reproj > thr) ? DYNOBA_TRI_OUTLIER : DYNOBA_TRI_OK;
}

// the lanes of a warp, emulated in order: every lane's partial sums, then the butterfly tree (lane 0's value)
struct TriHostLanes {
  template <class F> __host__ __device__ void each(F f) { for (int l = 0; l < TRI_LANES; l++) f(l); }
  template <int N, class F> __host__ __device__ void sum(F f, double* out) {
    double part[TRI_LANES][N];
    for (int l = 0; l < TRI_LANES; l++) f(l, part[l]);
    for (int k = 0; k < N; k++) {
      double x[TRI_LANES], y[TRI_LANES];
      for (int l = 0; l < TRI_LANES; l++) x[l] = part[l][k];
      for (int off = TRI_LANES/2; off > 0; off >>= 1) {
        for (int l = 0; l < TRI_LANES; l++) y[l] = x[l] + x[l ^ off];
        for (int l = 0; l < TRI_LANES; l++) x[l] = y[l];
      }
      out[k] = x[0];
    }
  }
};

}  // namespace dynoba
