// kernels_star.cu -- SURVEY.md 8f-2: many small "star" Levenberg-Marquardt problems in ONE launch.
//
// The front end refines, per frame and per object,
//   (1) a camera pose (or object motion) jointly with the optical flow of its features: OpticalFlowAndPoseOptimizer::optimize
//       (dynosam/include/dynosam/frontend/vision/MotionSolver-inl.hpp:88-278) builds, for every tracked feature i, a
//       Pose3FlowProjectionFactor(flow_i, pose; kp_i, depth_i, X_prev, K) with Robust(Huber) noise and a
//       PriorFactor<Point2>(flow_i, measured flow), runs gtsam::LevenbergMarquardtOptimizer (maxIterations 10) and then up to four
//       outlier rounds (drop the flow factors whose Gaussian error exceeds the chi-square bound, reset the pose, optimise again);
//   (2) an object motion from 3D point pairs: MotionOnlyRefinementOptimizer::optimize (:291-470) -- per tracklet two
//       GenericProjectionFactors (X_k-1, m_k-1), (X_k, m_k) and a LandmarkMotionTernaryFactor(m_k-1, m_k, H), tight priors on the
//       two camera poses, LM with maxIterations 5.
// One tiny LM (6 + 2N or 18 + 6N unknowns, N <= a few hundred) per object per frame.  Here every problem gets one CTA that runs
// the WHOLE optimisation on the device (no host round trip per iteration or per outlier round): linearise, eliminate the
// per-feature unknowns in registers, reduce the small pose system in a fixed order (deterministic), factor it, back-substitute,
// retract, evaluate, and GTSAM's tryLambda control (LevenbergMarquardtOptimizer.cpp, SURVEY Appendix A.4) -- the decisions
// of lm_control.cuh, which api.cu::dynoba_optimize takes as well.
#include <cfloat>
#include <algorithm>
#include <mutex>
#include <vector>
#include "../../include/dynoba.h"
#include "internal.cuh"
#include "se3.cuh"

namespace dynoba {

constexpr int STAR_THREADS = 256;
constexpr int STAR_WARPS = STAR_THREADS/32;

// deterministic block sums of NV values per thread (fixed tree order); every thread may read the sums in out[] afterwards
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* red /* [NV][STAR_WARPS] */, double* out /* [NV] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; k++) {
    double x = v[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) red[k*STAR_WARPS + warp] = x;
  }
  __syncthreads();
  if (threadIdx.x < NV) { double s = 0; for (int w = 0; w < STAR_WARPS; w++) s += red[threadIdx.x*STAR_WARPS + w]; out[threadIdx.x] = s; }
  __syncthreads();
}

// LevenbergMarquardtOptimizer::optimize / iterate / tryLambda for a problem object PB whose methods are CTA-collective:
//   error_cur()                             total error at the current values
//   try_step(lambda, oldLin, newLin, nerr)  damped solve at the current values, candidate values, linear model error at the step,
//                                           nonlinear error at the candidate; false if the damped system is not positive definite
//   accept()                                candidate -> current
// Every thread takes the same decisions from the same block sums.
template <class PB>
__device__ void run_lm(PB& pb, const dynoba_lm_params& P, double& err, int& iterations, int& inner) {
  err = pb.error_cur();
  double lambda = P.lambda_initial;
  int its = 0;
  if (lm_starts(err, P)) {
    double newError = err, currentError;
    do {
      currentError = newError;
      for (;;) {      // tryLambda (lm_control.cuh)
        double oldLin = 0, newLin = 0, nerr = INFINITY;
        const bool solved = pb.try_step(lambda, oldLin, newLin, nerr);
        const LmDecision d = lm_decide(solved, oldLin, oldLin - newLin, err, nerr, P);
        if (d.success) pb.accept();
        if (lm_update(d, nerr, P, lambda, err, its, inner)) break;
      }
      newError = err;
    } while (lm_continues(its, currentError, newError, P));
  }
  iterations += its;
}

// in-place Cholesky of the lower triangle of an N x N row-major matrix (one thread); false if not positive definite
template <int N>
__device__ bool chol_lower(double* L) {
  for (int j = 0; j < N; j++) {
    double d = L[j*N + j]; for (int k = 0; k < j; k++) d -= L[j*N + k]*L[j*N + k];
    if (!(d > 0.0)) return false;
    d = sqrt(d); L[j*N + j] = d;
    for (int i = j + 1; i < N; i++) { double s = L[i*N + j]; for (int k = 0; k < j; k++) s -= L[i*N + k]*L[j*N + k]; L[i*N + j] = s/d; }
  }
  return true;
}
template <int N>
__device__ void chol_solve(const double* L, const double* g, double* x) {
  double y[N];
  for (int i = 0; i < N; i++) { double s = g[i]; for (int k = 0; k < i; k++) s -= L[i*N + k]*y[k]; y[i] = s/L[i*N + i]; }
  for (int i = N - 1; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < N; k++) s -= L[k*N + i]*x[k]; x[i] = s/L[i*N + i]; }
}

// =====================================================================================================================
// (1) joint optical flow + pose
// =====================================================================================================================
struct FlowPoseBatch {
  int nprob; const int* off;                    // [nprob + 1] feature ranges
  const double* pose0; const double* pose_prev; const double* calib;    // [nprob][12], [nprob][12], [nprob][5] (fx fy s u0 v0)
  const double* kp; const double* depth; const double* flow0;           // [total][2], [total], [total][2] (prior mean = initial value)
  double isig_flow, isig_prior, huber_k, outlier_thr;
  int outlier_rounds;
  dynoba_lm_params prm;
  double* flow_cur; double* flow_cand;          // [total][2] work
  unsigned char* active; unsigned char* outl;   // [total] flow factor still in the graph / marked by the last outlier test
  double* pose_out; double* err_before; double* err_after; int* iterations; int* inner; int* rounds;
};

// one feature: whitened, Huber-weighted flow-projection factor (if still in the graph) + Gaussian flow prior at (X, flow)
struct FlowFactor { double A[2][6]; double a[2]; double b[2]; double bp[2]; double err; double gauss; };
__device__ __forceinline__ void flow_factor(const FlowPoseBatch& S, int i, bool act, const Pose& X, const Pose& Xp, const double* K6, const double* flow,
                                            FlowFactor& F, bool want_j) {
  const double rp0 = (flow[0] - S.flow0[2*i])*S.isig_prior, rp1 = (flow[1] - S.flow0[2*i + 1])*S.isig_prior;
  F.err = 0.5*(rp0*rp0 + rp1*rp1); F.bp[0] = -rp0; F.bp[1] = -rp1; F.gauss = 0.0;
  F.b[0] = F.b[1] = 0.0; F.a[0] = F.a[1] = 0.0;
#pragma unroll
  for (int c = 0; c < 6; c++) F.A[0][c] = F.A[1][c] = 0.0;
  if (!act) return;
  FVars v; v.pose[0] = X; v.pt[0][0] = flow[0]; v.pt[0][1] = flow[1]; v.pt[0][2] = 0.0;
  double z[15] = { S.kp[2*i], S.kp[2*i + 1], S.depth[i] };
  for (int k = 0; k < 9; k++) z[3 + k] = Xp.R[k];
  for (int k = 0; k < 3; k++) z[12 + k] = Xp.t[k];
  double r[2], J[16]; Pose none{};
  if (want_j) factor_eval<F_FLOWPROJ2, true>(v, z, none, K6, r, J); else factor_eval<F_FLOWPROJ2, false>(v, z, none, K6, r, J);
  double e = 0.0;
  const double isig = S.isig_flow;
  const double sw = whiten_weight<2>(r, &isig, 1, S.huber_k, &e);       // r is whitened in place
  F.gauss = 0.5*(r[0]*r[0] + r[1]*r[1]);
  F.err += e;
  F.b[0] = -sw*r[0]; F.b[1] = -sw*r[1];
  if (want_j) {
    const double sc = sw*isig;
    F.a[0] = sc*J[0*8 + 0]; F.a[1] = sc*J[1*8 + 1];
#pragma unroll
    for (int c = 0; c < 6; c++) { F.A[0][c] = sc*J[0*8 + 2 + c]; F.A[1][c] = sc*J[1*8 + 2 + c]; }
  }
}

struct FlowPoseProblem {
  const FlowPoseBatch& S; int f0, f1; Pose Xp; double K6[6];
  double* red; double* sums; double* sh_dp; double* sh_L; Pose* sh_cur; Pose* sh_cand; int* sh_ok;

  __device__ double error_at(const Pose& X, const double* flows) {
    double e[1] = { 0.0 };
    for (int i = f0 + threadIdx.x; i < f1; i += STAR_THREADS) { FlowFactor F; flow_factor(S, i, S.active[i] != 0, X, Xp, K6, flows + 2*i, F, false); e[0] += F.err; }
    block_sum<1>(e, red, sums);
    const double r = sums[0];
    __syncthreads();
    return r;
  }
  __device__ double error_cur() { const Pose X = *sh_cur; return error_at(X, S.flow_cur); }

  __device__ bool try_step(double lambda, double& oldLin, double& newLin, double& nerr) {
    // reduced pose system at (cur, lambda): S6 = sum A^T A + lambda I - sum_k W_k W_k^T / v_k,  g6 likewise; 1/2 sum b^2.
    // The 2x2 block of a flow variable is diagonal (d r / d flow = I): v_k = a_k^2 + 1/sigma_p^2 + lambda.
    double acc[28];
#pragma unroll
    for (int k = 0; k < 28; k++) acc[k] = 0.0;
    const Pose X = *sh_cur;
    const double ip2 = S.isig_prior*S.isig_prior;
    for (int i = f0 + threadIdx.x; i < f1; i += STAR_THREADS) {
      FlowFactor F; flow_factor(S, i, S.active[i] != 0, X, Xp, K6, S.flow_cur + 2*i, F, true);
      int e = 0;
      for (int r = 0; r < 6; r++) for (int c = 0; c <= r; c++, e++) {
        double u = F.A[0][r]*F.A[0][c] + F.A[1][r]*F.A[1][c];
        for (int k = 0; k < 2; k++) { const double v = F.a[k]*F.a[k] + ip2 + lambda; u -= (F.A[k][r]*F.a[k])*(F.A[k][c]*F.a[k])/v; }
        acc[e] += u;
      }
      for (int r = 0; r < 6; r++) {
        double g = F.A[0][r]*F.b[0] + F.A[1][r]*F.b[1];
        for (int k = 0; k < 2; k++) { const double v = F.a[k]*F.a[k] + ip2 + lambda; const double gl = F.a[k]*F.b[k] + S.isig_prior*F.bp[k]; g -= (F.A[k][r]*F.a[k])*gl/v; }
        acc[21 + r] += g;
      }
      acc[27] += 0.5*(F.b[0]*F.b[0] + F.b[1]*F.b[1] + F.bp[0]*F.bp[0] + F.bp[1]*F.bp[1]);
    }
    block_sum<28>(acc, red, sums);
    if (threadIdx.x == 0) {
      double* L = sh_L; int e = 0;
      for (int r = 0; r < 6; r++) for (int c = 0; c <= r; c++, e++) L[r*6 + c] = sums[e] + (r == c ? lambda : 0.0);
      const bool ok = chol_lower<6>(L);
      if (ok) { chol_solve<6>(L, sums + 21, sh_dp); Pose cand; se3_retract(*sh_cur, sh_dp, cand); *sh_cand = cand; }
      *sh_ok = ok ? 1 : 0;
    }
    __syncthreads();
    const bool solved = *sh_ok != 0;
    oldLin = sums[27];
    __syncthreads();
    if (!solved) return false;
    // back-substitute the flows, linear model at the step, candidate values
    double m[1] = { 0.0 };
    for (int i = f0 + threadIdx.x; i < f1; i += STAR_THREADS) {
      FlowFactor F; flow_factor(S, i, S.active[i] != 0, X, Xp, K6, S.flow_cur + 2*i, F, true);
      for (int k = 0; k < 2; k++) {
        double Ad = 0.0; for (int c = 0; c < 6; c++) Ad += F.A[k][c]*sh_dp[c];
        const double v = F.a[k]*F.a[k] + ip2 + lambda, gl = F.a[k]*F.b[k] + S.isig_prior*F.bp[k];
        const double dl = (gl - F.a[k]*Ad)/v;                 // W_k^T dp = a_k (A_k . dp)
        const double rf = Ad + F.a[k]*dl - F.b[k], rpk = S.isig_prior*dl - F.bp[k];
        m[0] += 0.5*(rf*rf + rpk*rpk);
        S.flow_cand[2*i + k] = S.flow_cur[2*i + k] + dl;
      }
    }
    block_sum<1>(m, red, sums);
    newLin = sums[0];
    __syncthreads();
    const Pose Xc = *sh_cand;
    nerr = error_at(Xc, S.flow_cand);
    return true;
  }
  __device__ void accept() {
    __syncthreads();
    if (threadIdx.x == 0) *sh_cur = *sh_cand;
    for (int i = f0 + threadIdx.x; i < f1; i += STAR_THREADS) { S.flow_cur[2*i] = S.flow_cand[2*i]; S.flow_cur[2*i + 1] = S.flow_cand[2*i + 1]; }
    __syncthreads();
  }
  // factor_graph_tools::determineFactorOutliers<Pose3FlowProjectionFactor> (dynosam_opt/FactorGraphTools.hpp:74-111): the GAUSSIAN
  // error of every factor still in the graph against 0.5 chi2inv(0.99, dim)
  __device__ int mark_outliers() {
    double n[1] = { 0.0 };
    const Pose X = *sh_cur;
    for (int i = f0 + threadIdx.x; i < f1; i += STAR_THREADS) {
      unsigned char o = 0;
      if (S.active[i]) { FlowFactor F; flow_factor(S, i, true, X, Xp, K6, S.flow_cur + 2*i, F, false); o = F.gauss > S.outlier_thr ? 1 : 0; }
      S.outl[i] = o; n[0] += o;
    }
    block_sum<1>(n, red, sums);
    const int r = (int)sums[0];
    __syncthreads();
    return r;
  }
};

__global__ void __launch_bounds__(STAR_THREADS) flow_pose_kernel(FlowPoseBatch S) {
  __shared__ double red[28*STAR_WARPS];
  __shared__ double sums[28];
  __shared__ double sh_dp[6], sh_L[36];
  __shared__ Pose sh_cur, sh_cand;
  __shared__ int sh_ok;
  const int pb = blockIdx.x;
  FlowPoseProblem Q{ S, S.off[pb], S.off[pb + 1], Pose{}, {0, 0, 0, 0, 0, 0}, red, sums, sh_dp, sh_L, &sh_cur, &sh_cand, &sh_ok };
  Pose X0;
  for (int k = 0; k < 9; k++) { Q.Xp.R[k] = S.pose_prev[12*pb + k]; X0.R[k] = S.pose0[12*pb + k]; }
  for (int k = 0; k < 3; k++) { Q.Xp.t[k] = S.pose_prev[12*pb + 9 + k]; X0.t[k] = S.pose0[12*pb + 9 + k]; }
  for (int k = 0; k < 5; k++) Q.K6[k] = S.calib[5*pb + k];
  if (threadIdx.x == 0) sh_cur = X0;
  for (int i = Q.f0 + threadIdx.x; i < Q.f1; i += STAR_THREADS) { S.flow_cur[2*i] = S.flow0[2*i]; S.flow_cur[2*i + 1] = S.flow0[2*i + 1]; S.active[i] = 1; S.outl[i] = 0; }
  __syncthreads();
  const double err0 = Q.error_cur();                  // result.error_before = graph.error(values)
  double err = 0; int iterations = 0, inner = 0, rounds = 0;
  run_lm(Q, S.prm, err, iterations, inner);
  __syncthreads();
  if (S.outlier_rounds > 0) {                         // MotionSolver-inl.hpp:201-247
    int nout = Q.mark_outliers();
    if (nout > 0) for (int itr = 0; itr < S.outlier_rounds; itr++) {
      for (int i = Q.f0 + threadIdx.x; i < Q.f1; i += STAR_THREADS) if (S.outl[i]) S.active[i] = 0;
      if (threadIdx.x == 0) sh_cur = X0;              // optimised_values.update(pose_key, initial_pose); the flows keep their values
      __syncthreads();
      run_lm(Q, S.prm, err, iterations, inner);
      rounds++;
      nout = Q.mark_outliers();
      if (nout == 0) break;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < 9; k++) S.pose_out[12*pb + k] = sh_cur.R[k];
    for (int k = 0; k < 3; k++) S.pose_out[12*pb + 9 + k] = sh_cur.t[k];
    S.err_before[pb] = err0; S.err_after[pb] = err; S.iterations[pb] = iterations; S.inner[pb] = inner; S.rounds[pb] = rounds;
  }
}

// =====================================================================================================================
// (2) object motion from 3D point pairs
// =====================================================================================================================
struct MotionBatch {
  int nprob; const int* off;                    // [nprob + 1] tracklet ranges
  const double* pose_a; const double* pose_b; const double* motion0; const double* calib;   // [nprob][12] x3, [nprob][5]
  const double* kp_a; const double* kp_b; const double* pt0;            // [total][2], [total][2], [total][6] (m_k-1 | m_k, world)
  double isig_proj, isig_motion, isig_prior, huber_k;
  dynoba_lm_params prm;
  double* pt_cur; double* pt_cand;              // [total][6]
  double* scratch;                              // per problem: [MR_SCR][n] (entry-major)
  double* motion_out; double* poses_out; double* motion_err; double* err_before; double* err_after; int* iterations; int* inner;
};
// scratch entries per tracklet
constexpr int MR_Y = 0, MR_L = 108, MR_YL = 129, MR_DA = 135, MR_DB = 147, MR_TH = 159, MR_B = 177, MR_SCR = 184;

// gtsam::GenericProjectionFactor<Pose3, Point3, Cal3_S2>::evaluateError (throwCheirality = false): PinholeCamera::project
// (CalibratedCamera Dpose / Dpoint, Cal3_S2::uncalibrate) - measured; behind the camera: zero Jacobians, error = (2 fx, 2 fx)
__device__ __forceinline__ void projection_factor(const Pose& X, const double* p, const double* K5, const double* z, double* r, double* Jx /* [2][6] */, double* Jp /* [2][3] */) {
  double q[3]; se3_transform_to(X, p, q);
#pragma unroll
  for (int i = 0; i < 12; i++) Jx[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; i++) Jp[i] = 0.0;
  if (q[2] <= 0.0) { r[0] = r[1] = 2.0*K5[0]; return; }
  const double d = 1.0/q[2], u = q[0]*d, v = q[1]*d, fx = K5[0], fy = K5[1], s = K5[2];
  r[0] = fx*u + s*v + K5[3] - z[0]; r[1] = fy*v + K5[4] - z[1];
  const double Dx[12] = { u*v, -1.0 - u*u, v, -d, 0.0, d*u,   1.0 + v*v, -u*v, -u, 0.0, -d, d*v };
  double Dp[6];
#pragma unroll
  for (int c = 0; c < 3; c++) {     // Rt = R^T: Rt(a, c) = R[3*c + a]
    Dp[c] = d*(X.R[3*c + 0] - u*X.R[3*c + 2]); Dp[3 + c] = d*(X.R[3*c + 1] - v*X.R[3*c + 2]);
  }
#pragma unroll
  for (int c = 0; c < 6; c++) { Jx[c] = fx*Dx[c] + s*Dx[6 + c]; Jx[6 + c] = fy*Dx[6 + c]; }
#pragma unroll
  for (int c = 0; c < 3; c++) { Jp[c] = fx*Dp[c] + s*Dp[3 + c]; Jp[3 + c] = fy*Dp[3 + c]; }
}

// one tracklet, whitened and Huber-weighted: rows 0-1 projection at k-1 (X_a, m_a), rows 2-3 projection at k (X_b, m_b),
// rows 4-6 motion factor m_a - H^-1 m_b (H, m_a, m_b).  P = columns of the two points, Da / Db / Th = columns of X_a / X_b / H.
struct TrackLin { double Da[12], Db[12], Th[18]; double P[7][6]; double b[7]; double err; };
__device__ __forceinline__ void track_lin(const MotionBatch& S, int i, const Pose& Xa, const Pose& Xb, const Pose& H, const double* K5, const double* m, TrackLin& T) {
  T.err = 0.0;
#pragma unroll
  for (int r = 0; r < 7; r++)
#pragma unroll
    for (int c = 0; c < 6; c++) T.P[r][c] = 0.0;
  {
    double r[2], Jp[6]; projection_factor(Xa, m, K5, S.kp_a + 2*i, r, T.Da, Jp);
    double e; const double isig = S.isig_proj; const double sw = whiten_weight<2>(r, &isig, 1, S.huber_k, &e); const double sc = sw*isig;
    T.err += e; T.b[0] = -sw*r[0]; T.b[1] = -sw*r[1];
#pragma unroll
    for (int c = 0; c < 12; c++) T.Da[c] *= sc;
#pragma unroll
    for (int c = 0; c < 3; c++) { T.P[0][c] = sc*Jp[c]; T.P[1][c] = sc*Jp[3 + c]; }
  }
  {
    double r[2], Jp[6]; projection_factor(Xb, m + 3, K5, S.kp_b + 2*i, r, T.Db, Jp);
    double e; const double isig = S.isig_proj; const double sw = whiten_weight<2>(r, &isig, 1, S.huber_k, &e); const double sc = sw*isig;
    T.err += e; T.b[2] = -sw*r[0]; T.b[3] = -sw*r[1];
#pragma unroll
    for (int c = 0; c < 12; c++) T.Db[c] *= sc;
#pragma unroll
    for (int c = 0; c < 3; c++) { T.P[2][3 + c] = sc*Jp[c]; T.P[3][3 + c] = sc*Jp[3 + c]; }
  }
  {
    FVars v; v.pose[0] = H;
#pragma unroll
    for (int c = 0; c < 3; c++) { v.pt[0][c] = m[c]; v.pt[1][c] = m[3 + c]; }
    double r[3], J[36]; Pose none{};
    factor_eval<F_TERNARY3, true>(v, nullptr, none, K5, r, J);          // columns: m_a (3), m_b (3), H (6)
    double e; const double isig = S.isig_motion; const double sw = whiten_weight<3>(r, &isig, 1, S.huber_k, &e); const double sc = sw*isig;
    T.err += e;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      T.b[4 + a] = -sw*r[a];
#pragma unroll
      for (int c = 0; c < 6; c++) { T.P[4 + a][c] = sc*J[a*12 + c]; T.Th[a*6 + c] = sc*J[a*12 + 6 + c]; }
    }
  }
}
// nonlinear error only (+ the Gaussian error of the motion factor)
__device__ __forceinline__ double track_error(const MotionBatch& S, int i, const Pose& Xa, const Pose& Xb, const Pose& H, const double* K5, const double* m, double* gauss_motion) {
  double err = 0.0, e, Jx[12], Jp[6], r[3];
  const double ip = S.isig_proj, im = S.isig_motion;
  projection_factor(Xa, m, K5, S.kp_a + 2*i, r, Jx, Jp); whiten_weight<2>(r, &ip, 1, S.huber_k, &e); err += e;
  projection_factor(Xb, m + 3, K5, S.kp_b + 2*i, r, Jx, Jp); whiten_weight<2>(r, &ip, 1, S.huber_k, &e); err += e;
  FVars v; v.pose[0] = H;
#pragma unroll
  for (int c = 0; c < 3; c++) { v.pt[0][c] = m[c]; v.pt[1][c] = m[3 + c]; }
  Pose none{}; double J[1];
  factor_eval<F_TERNARY3, false>(v, nullptr, none, K5, r, J);
  whiten_weight<3>(r, &im, 1, S.huber_k, &e); err += e;
  if (gauss_motion) *gauss_motion = 0.5*(r[0]*r[0] + r[1]*r[1] + r[2]*r[2]);
  return err;
}

struct MotionProblem {
  const MotionBatch& S; int f0, n; double K5[5]; Pose prior_a, prior_b;
  double* scr; double* red; double* sums; double* sh_S; double* sh_g; double* sh_dp; double* sh_bpr; Pose* sh_cur; Pose* sh_cand; int* sh_ok;

  // PriorFactor<Pose3>(X, prior, Isotropic): e = -Local(x, prior), J = I
  __device__ double prior_error(const Pose* X) {
    double e = 0.0, r[6];
    se3_local(X[0], prior_a, r); for (int k = 0; k < 6; k++) e += 0.5*(r[k]*S.isig_prior)*(r[k]*S.isig_prior);
    se3_local(X[1], prior_b, r); for (int k = 0; k < 6; k++) e += 0.5*(r[k]*S.isig_prior)*(r[k]*S.isig_prior);
    return e;
  }
  __device__ double error_at(const Pose* Xs, const double* pts) {
    const Pose Xa = Xs[0], Xb = Xs[1], H = Xs[2];
    double e[1] = { 0.0 };
    for (int i = threadIdx.x; i < n; i += STAR_THREADS) e[0] += track_error(S, f0 + i, Xa, Xb, H, K5, pts + 6*(size_t)(f0 + i), nullptr);
    block_sum<1>(e, red, sums);
    const double r = sums[0] + prior_error(Xs);
    __syncthreads();
    return r;
  }
  __device__ double error_cur() { return error_at(sh_cur, S.pt_cur); }

  __device__ bool try_step(double lambda, double& oldLin, double& newLin, double& nerr) {
    const Pose Xa = sh_cur[0], Xb = sh_cur[1], H = sh_cur[2];
    if (threadIdx.x == 0) *sh_ok = 1;
    __syncthreads();
    // ---- phase 1, a thread per tracklet: eliminate (m_a, m_b): V = P^T P + lambda I = L L^T, Y = W L^-T, yl = L^-1 P^T b
    double ob[1] = { 0.0 };
    for (int i = threadIdx.x; i < n; i += STAR_THREADS) {
      TrackLin T; track_lin(S, f0 + i, Xa, Xb, H, K5, S.pt_cur + 6*(size_t)(f0 + i), T);
      double L[36];
      for (int r = 0; r < 6; r++) for (int c = 0; c <= r; c++) { double s = (r == c) ? lambda : 0.0; for (int k = 0; k < 7; k++) s += T.P[k][r]*T.P[k][c]; L[r*6 + c] = s; }
      if (!chol_lower<6>(L)) { *sh_ok = 0; continue; }
      double* out = scr + i;
      // W rows: X_a (6) = Da^T P[0:2], X_b (6) = Db^T P[2:4], H (6) = Th^T P[4:7]; a Y row = forward substitution with L
      for (int r = 0; r < 18; r++) {
        double w[6];
        for (int c = 0; c < 6; c++) {
          if (r < 6) w[c] = T.Da[r]*T.P[0][c] + T.Da[6 + r]*T.P[1][c];
          else if (r < 12) w[c] = T.Db[r - 6]*T.P[2][c] + T.Db[r]*T.P[3][c];
          else w[c] = T.Th[r - 12]*T.P[4][c] + T.Th[r - 6]*T.P[5][c] + T.Th[r]*T.P[6][c];
        }
        for (int c = 0; c < 6; c++) { double s = w[c]; for (int k = 0; k < c; k++) s -= L[c*6 + k]*w[k]; w[c] = s/L[c*6 + c]; out[(size_t)(MR_Y + r*6 + c)*n] = w[c]; }
      }
      { int e = 0; for (int r = 0; r < 6; r++) for (int c = 0; c <= r; c++, e++) out[(size_t)(MR_L + e)*n] = L[r*6 + c]; }
      double gl[6];
      for (int c = 0; c < 6; c++) { double s = 0.0; for (int k = 0; k < 7; k++) s += T.P[k][c]*T.b[k]; gl[c] = s; }
      for (int c = 0; c < 6; c++) { double s = gl[c]; for (int k = 0; k < c; k++) s -= L[c*6 + k]*gl[k]; gl[c] = s/L[c*6 + c]; out[(size_t)(MR_YL + c)*n] = gl[c]; }
      for (int c = 0; c < 12; c++) { out[(size_t)(MR_DA + c)*n] = T.Da[c]; out[(size_t)(MR_DB + c)*n] = T.Db[c]; }
      for (int c = 0; c < 18; c++) out[(size_t)(MR_TH + c)*n] = T.Th[c];
      for (int c = 0; c < 7; c++) { out[(size_t)(MR_B + c)*n] = T.b[c]; ob[0] += 0.5*T.b[c]*T.b[c]; }
    }
    block_sum<1>(ob, red, sums);
    double old_lin = sums[0];
    __syncthreads();                                  // scratch written (block_sum's barriers), sh_ok final
    if (*sh_ok == 0) { __syncthreads(); return false; }
    // ---- phase 2, a thread per entry of the 18x18 pose system (lower triangle) and of its right-hand side: fixed summation order
    for (int e = threadIdx.x; e < 171 + 18; e += STAR_THREADS) {
      double s = 0.0;
      if (e < 171) {
        int r = 0; while ((r + 1)*(r + 2)/2 <= e) r++;
        const int c = e - r*(r + 1)/2;
        const int br = r/6, bc = c/6, rr = r%6, cc = c%6;
        const double* yr = scr + (size_t)(MR_Y + r*6)*n; const double* yc = scr + (size_t)(MR_Y + c*6)*n;
        const int rows = br == 2 ? 3 : 2; const int ab = br == 0 ? MR_DA : (br == 1 ? MR_DB : MR_TH);
        for (int i = 0; i < n; i++) {
          double t = 0.0;
          if (br == bc) for (int k = 0; k < rows; k++) t += scr[(size_t)(ab + k*6 + rr)*n + i]*scr[(size_t)(ab + k*6 + cc)*n + i];
          for (int k = 0; k < 6; k++) t -= yr[(size_t)k*n + i]*yc[(size_t)k*n + i];
          s += t;
        }
        sh_S[r*18 + c] = s;
      } else {
        const int r = e - 171, br = r/6, rr = r%6;
        const double* yr = scr + (size_t)(MR_Y + r*6)*n;
        const int rows = br == 2 ? 3 : 2; const int ab = br == 0 ? MR_DA : (br == 1 ? MR_DB : MR_TH); const int b0 = br == 0 ? 0 : (br == 1 ? 2 : 4);
        for (int i = 0; i < n; i++) {
          double t = 0.0;
          for (int k = 0; k < rows; k++) t += scr[(size_t)(ab + k*6 + rr)*n + i]*scr[(size_t)(MR_B + b0 + k)*n + i];
          for (int k = 0; k < 6; k++) t -= yr[(size_t)k*n + i]*scr[(size_t)(MR_YL + k)*n + i];
          s += t;
        }
        sh_g[r] = s;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      // camera pose priors (J = I), damping, 18x18 Cholesky, step, candidate poses
      double r[6]; const double w2 = S.isig_prior*S.isig_prior;
      se3_local(sh_cur[0], prior_a, r); for (int k = 0; k < 6; k++) { sh_bpr[k] = r[k]*S.isig_prior; sh_S[k*18 + k] += w2; sh_g[k] += S.isig_prior*sh_bpr[k]; }
      se3_local(sh_cur[1], prior_b, r); for (int k = 0; k < 6; k++) { sh_bpr[6 + k] = r[k]*S.isig_prior; sh_S[(6 + k)*18 + 6 + k] += w2; sh_g[6 + k] += S.isig_prior*sh_bpr[6 + k]; }
      for (int k = 0; k < 18; k++) sh_S[k*18 + k] += lambda;
      const bool ok = chol_lower<18>(sh_S);
      if (ok) { chol_solve<18>(sh_S, sh_g, sh_dp); for (int v = 0; v < 3; v++) { Pose c; se3_retract(sh_cur[v], sh_dp + 6*v, c); sh_cand[v] = c; } }
      *sh_ok = ok ? 1 : 0;
    }
    __syncthreads();
    if (*sh_ok == 0) { __syncthreads(); return false; }
    for (int k = 0; k < 12; k++) old_lin += 0.5*sh_bpr[k]*sh_bpr[k];
    oldLin = old_lin;
    // ---- phase 3, a thread per tracklet: dl = L^-T (yl - Y^T dp), linear model at the step, candidate points
    double m[1] = { 0.0 };
    for (int i = threadIdx.x; i < n; i += STAR_THREADS) {
      TrackLin T; track_lin(S, f0 + i, Xa, Xb, H, K5, S.pt_cur + 6*(size_t)(f0 + i), T);
      const double* in = scr + i;
      double t[6], L[21];
      for (int e = 0; e < 21; e++) L[e] = in[(size_t)(MR_L + e)*n];
      for (int c = 0; c < 6; c++) { double s = in[(size_t)(MR_YL + c)*n]; for (int r = 0; r < 18; r++) s -= in[(size_t)(MR_Y + r*6 + c)*n]*sh_dp[r]; t[c] = s; }
      for (int c = 5; c >= 0; c--) { double s = t[c]; for (int k = c + 1; k < 6; k++) s -= L[k*(k + 1)/2 + c]*t[k]; t[c] = s/L[c*(c + 1)/2 + c]; }
      for (int k = 0; k < 7; k++) {
        double rr = -T.b[k];
        for (int c = 0; c < 6; c++) rr += T.P[k][c]*t[c];
        if (k < 2) { for (int c = 0; c < 6; c++) rr += T.Da[k*6 + c]*sh_dp[c]; }
        else if (k < 4) { for (int c = 0; c < 6; c++) rr += T.Db[(k - 2)*6 + c]*sh_dp[6 + c]; }
        else { for (int c = 0; c < 6; c++) rr += T.Th[(k - 4)*6 + c]*sh_dp[12 + c]; }
        m[0] += 0.5*rr*rr;
      }
      for (int c = 0; c < 6; c++) S.pt_cand[6*(size_t)(f0 + i) + c] = S.pt_cur[6*(size_t)(f0 + i) + c] + t[c];
    }
    block_sum<1>(m, red, sums);
    double new_lin = sums[0];
    for (int k = 0; k < 12; k++) { const double rr = S.isig_prior*sh_dp[k] - sh_bpr[k]; new_lin += 0.5*rr*rr; }
    newLin = new_lin;
    __syncthreads();
    nerr = error_at(sh_cand, S.pt_cand);
    return true;
  }
  __device__ void accept() {
    __syncthreads();
    if (threadIdx.x < 3) sh_cur[threadIdx.x] = sh_cand[threadIdx.x];
    for (int i = threadIdx.x; i < 6*n; i += STAR_THREADS) S.pt_cur[6*(size_t)f0 + i] = S.pt_cand[6*(size_t)f0 + i];
    __syncthreads();
  }
};

__global__ void __launch_bounds__(STAR_THREADS) motion_refine_kernel(MotionBatch S) {
  __shared__ double red[STAR_WARPS];
  __shared__ double sums[1];
  __shared__ double sh_S[18*18];
  __shared__ double sh_g[18], sh_dp[18], sh_bpr[12];
  __shared__ Pose sh_cur[3], sh_cand[3];
  __shared__ int sh_ok;
  const int pb = blockIdx.x;
  MotionProblem Q{ S, S.off[pb], S.off[pb + 1] - S.off[pb], {0, 0, 0, 0, 0}, Pose{}, Pose{}, S.scratch + (size_t)MR_SCR*(size_t)S.off[pb],
                   red, sums, sh_S, sh_g, sh_dp, sh_bpr, sh_cur, sh_cand, &sh_ok };
  for (int k = 0; k < 5; k++) Q.K5[k] = S.calib[5*pb + k];
  Pose H0;
  for (int k = 0; k < 9; k++) { Q.prior_a.R[k] = S.pose_a[12*pb + k]; Q.prior_b.R[k] = S.pose_b[12*pb + k]; H0.R[k] = S.motion0[12*pb + k]; }
  for (int k = 0; k < 3; k++) { Q.prior_a.t[k] = S.pose_a[12*pb + 9 + k]; Q.prior_b.t[k] = S.pose_b[12*pb + 9 + k]; H0.t[k] = S.motion0[12*pb + 9 + k]; }
  if (threadIdx.x == 0) { sh_cur[0] = Q.prior_a; sh_cur[1] = Q.prior_b; sh_cur[2] = H0; }
  for (int i = threadIdx.x; i < 6*Q.n; i += STAR_THREADS) S.pt_cur[6*(size_t)Q.f0 + i] = S.pt0[6*(size_t)Q.f0 + i];
  __syncthreads();
  const double err0 = Q.error_cur();
  double err = 0; int iterations = 0, inner = 0;
  run_lm(Q, S.prm, err, iterations, inner);
  __syncthreads();
  // Gaussian error of every motion factor at the result: what determineFactorOutliers<LandmarkMotionTernaryFactor> thresholds
  {
    const Pose Xa = sh_cur[0], Xb = sh_cur[1], H = sh_cur[2];
    for (int i = threadIdx.x; i < Q.n; i += STAR_THREADS) { double g; track_error(S, Q.f0 + i, Xa, Xb, H, Q.K5, S.pt_cur + 6*(size_t)(Q.f0 + i), &g); S.motion_err[Q.f0 + i] = g; }
  }
  if (threadIdx.x == 0) {
    for (int v = 0; v < 2; v++) { for (int k = 0; k < 9; k++) S.poses_out[24*pb + 12*v + k] = sh_cur[v].R[k]; for (int k = 0; k < 3; k++) S.poses_out[24*pb + 12*v + 9 + k] = sh_cur[v].t[k]; }
    for (int k = 0; k < 9; k++) S.motion_out[12*pb + k] = sh_cur[2].R[k];
    for (int k = 0; k < 3; k++) S.motion_out[12*pb + 9 + k] = sh_cur[2].t[k];
    S.err_before[pb] = err0; S.err_after[pb] = err; S.iterations[pb] = iterations; S.inner[pb] = inner;
  }
}

static StarContext g_star[64];
StarContext& star_context(int device) { return g_star[device]; }
int star_device_ready(int device) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return DYNOBA_ERR_CUDA;     // no CPU fallback
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) return DYNOBA_ERR_CUDA;
  if (device >= 64 || cudaSetDevice(device) != cudaSuccess) return DYNOBA_ERR_CUDA;
  StarContext& c = g_star[device];
  if (!c.stream && cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking) != cudaSuccess) { c.stream = nullptr; return DYNOBA_ERR_CUDA; }
  return DYNOBA_OK;
}

}  // namespace dynoba

using namespace dynoba;

extern "C" {

void dynoba_flow_pose_default_params(dynoba_flow_pose_params* p) {
  if (!p) return;
  p->flow_sigma = 10.0; p->flow_prior_sigma = 3.33; p->huber_k = 0.001;      // OpticalFlowAndPoseOptimizer::Params (MotionSolver.hpp:134-138)
  p->outlier_rounds = 4; p->outlier_threshold = 0.0;                          // outlier_reject = true: up to four rounds
  dynoba_lm_default_params(&p->lm); p->lm.max_iterations = 10;                // MotionSolver-inl.hpp:186
}

int dynoba_flow_pose_batch(int device, int32_t n_problems, const int32_t* offsets, const double* pose_init, const double* pose_prev,
                           const double* calib5, const double* kp_prev, const double* depth, const double* flow,
                           const dynoba_flow_pose_params* prm, double* pose_out, double* flow_out, uint8_t* inlier_out,
                           double* err_before, double* err_after, int32_t* iterations, int32_t* inner_iterations, int32_t* rounds) {
  if (n_problems == 0) return DYNOBA_OK;
  dynoba_flow_pose_params P; if (prm) P = *prm; else dynoba_flow_pose_default_params(&P);
  if (n_problems < 0 || !offsets || !pose_init || !pose_prev || !calib5 || !pose_out || !err_before || !err_after || !iterations || !inner_iterations ||
      !(P.flow_sigma > 0) || !(P.flow_prior_sigma > 0) || P.outlier_rounds < 0 || !lm_params_usable(P.lm)) return DYNOBA_ERR_BAD_ARG;
  const int total = offsets[n_problems];
  if (offsets[0] != 0 || total < 0 || (total > 0 && (!kp_prev || !depth || !flow || !flow_out))) return DYNOBA_ERR_BAD_ARG;
  for (int p = 0; p < n_problems; p++) if (offsets[p + 1] < offsets[p]) return DYNOBA_ERR_BAD_ARG;
  if (device < 0 || device >= 64) return DYNOBA_ERR_CUDA;
  std::lock_guard<std::mutex> lock(g_star[device].mu);
  int rc = star_device_ready(device); if (rc) return rc;
  StarContext& ctx = g_star[device];
  const size_t np = (size_t)n_problems, nt = (size_t)std::max(total, 1);
  DeviceBlock blk; FlowPoseBatch S{};
  int* d_off; double *d_pose0, *d_prev, *d_cal, *d_kp, *d_depth, *d_flow0;
  auto layout = [&]() {
    d_off = blk.take<int>(np + 1);
    d_pose0 = blk.take<double>(12*np); d_prev = blk.take<double>(12*np); d_cal = blk.take<double>(5*np);
    d_kp = blk.take<double>(2*nt); d_depth = blk.take<double>(nt); d_flow0 = blk.take<double>(2*nt);
    S.flow_cur = blk.take<double>(2*nt); S.flow_cand = blk.take<double>(2*nt);
    S.active = blk.take<unsigned char>(nt); S.outl = blk.take<unsigned char>(nt);
    S.pose_out = blk.take<double>(12*np); S.err_before = blk.take<double>(np); S.err_after = blk.take<double>(np);
    S.iterations = blk.take<int>(np); S.inner = blk.take<int>(np); S.rounds = blk.take<int>(np);
  };
  layout();
  if (!blk.allocate(ctx)) { cudaGetLastError(); return DYNOBA_ERR_CUDA; }
  layout();
  S.nprob = n_problems;
  cudaStream_t s = ctx.stream;
  cudaMemcpyAsync(d_off, offsets, (np + 1)*4, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_pose0, pose_init, 96*np, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_prev, pose_prev, 96*np, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_cal, calib5, 40*np, cudaMemcpyHostToDevice, s);
  if (total > 0) { cudaMemcpyAsync(d_kp, kp_prev, 16*(size_t)total, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_depth, depth, 8*(size_t)total, cudaMemcpyHostToDevice, s);
                   cudaMemcpyAsync(d_flow0, flow, 16*(size_t)total, cudaMemcpyHostToDevice, s); }
  S.off = d_off; S.pose0 = d_pose0; S.pose_prev = d_prev; S.calib = d_cal; S.kp = d_kp; S.depth = d_depth; S.flow0 = d_flow0;
  S.isig_flow = 1.0/P.flow_sigma; S.isig_prior = 1.0/P.flow_prior_sigma; S.huber_k = P.huber_k;
  S.outlier_rounds = P.outlier_rounds;
  S.outlier_thr = P.outlier_threshold > 0 ? P.outlier_threshold : 0.5*9.210340371976184;      // 0.5 chi2inv(0.99, 2) = -ln(0.01)
  S.prm = P.lm;
  flow_pose_kernel<<<n_problems, STAR_THREADS, 0, s>>>(S);
  cudaMemcpyAsync(pose_out, S.pose_out, 96*np, cudaMemcpyDeviceToHost, s);
  if (total > 0) cudaMemcpyAsync(flow_out, S.flow_cur, 16*(size_t)total, cudaMemcpyDeviceToHost, s);
  if (total > 0 && inlier_out) cudaMemcpyAsync(inlier_out, S.active, (size_t)total, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(err_before, S.err_before, 8*np, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(err_after, S.err_after, 8*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(iterations, S.iterations, 4*np, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(inner_iterations, S.inner, 4*np, cudaMemcpyDeviceToHost, s);
  if (rounds) cudaMemcpyAsync(rounds, S.rounds, 4*np, cudaMemcpyDeviceToHost, s);
  const cudaError_t e1 = cudaStreamSynchronize(s), e2 = cudaGetLastError();
  return (e1 == cudaSuccess && e2 == cudaSuccess) ? DYNOBA_OK : DYNOBA_ERR_CUDA;
}

void dynoba_motion_refine_default_params(dynoba_motion_refine_params* p) {
  if (!p) return;
  p->landmark_motion_sigma = 0.001; p->projection_sigma = 2.0; p->huber_k = 0.0001;   // MotionOnlyRefinementOptimizer::Params (MotionSolver.hpp:221-225)
  p->pose_prior_sigma = 0.00001;                                                       // MotionSolver-inl.hpp:326
  dynoba_lm_default_params(&p->lm); p->lm.max_iterations = 5;                          // :412
}

int dynoba_motion_refine_batch(int device, int32_t n_problems, const int32_t* offsets, const double* pose_prev, const double* pose_cur,
                               const double* motion_init, const double* calib5, const double* kp_prev, const double* kp_cur,
                               const double* points_init, const dynoba_motion_refine_params* prm, double* motion_out, double* poses_out,
                               double* points_out, double* motion_factor_error, double* err_before, double* err_after,
                               int32_t* iterations, int32_t* inner_iterations) {
  if (n_problems == 0) return DYNOBA_OK;
  dynoba_motion_refine_params P; if (prm) P = *prm; else dynoba_motion_refine_default_params(&P);
  if (n_problems < 0 || !offsets || !pose_prev || !pose_cur || !motion_init || !calib5 || !motion_out || !err_before || !err_after || !iterations ||
      !inner_iterations || !(P.landmark_motion_sigma > 0) || !(P.projection_sigma > 0) || !(P.pose_prior_sigma > 0) || !lm_params_usable(P.lm))
    return DYNOBA_ERR_BAD_ARG;
  const int total = offsets[n_problems];
  if (offsets[0] != 0 || total < 0 || (total > 0 && (!kp_prev || !kp_cur || !points_init))) return DYNOBA_ERR_BAD_ARG;
  for (int p = 0; p < n_problems; p++) if (offsets[p + 1] < offsets[p]) return DYNOBA_ERR_BAD_ARG;
  if (device < 0 || device >= 64) return DYNOBA_ERR_CUDA;
  std::lock_guard<std::mutex> lock(g_star[device].mu);
  int rc = star_device_ready(device); if (rc) return rc;
  StarContext& ctx = g_star[device];
  const size_t np = (size_t)n_problems, nt = (size_t)std::max(total, 1);
  DeviceBlock blk; MotionBatch S{};
  int* d_off; double *d_pa, *d_pb, *d_h, *d_cal, *d_ka, *d_kb, *d_pt0;
  auto layout = [&]() {
    d_off = blk.take<int>(np + 1);
    d_pa = blk.take<double>(12*np); d_pb = blk.take<double>(12*np); d_h = blk.take<double>(12*np); d_cal = blk.take<double>(5*np);
    d_ka = blk.take<double>(2*nt); d_kb = blk.take<double>(2*nt); d_pt0 = blk.take<double>(6*nt);
    S.pt_cur = blk.take<double>(6*nt); S.pt_cand = blk.take<double>(6*nt); S.motion_err = blk.take<double>(nt); S.scratch = blk.take<double>((size_t)MR_SCR*nt);
    S.motion_out = blk.take<double>(12*np); S.poses_out = blk.take<double>(24*np); S.err_before = blk.take<double>(np); S.err_after = blk.take<double>(np);
    S.iterations = blk.take<int>(np); S.inner = blk.take<int>(np);
  };
  layout();
  if (!blk.allocate(ctx)) { cudaGetLastError(); return DYNOBA_ERR_CUDA; }
  layout();
  S.nprob = n_problems;
  cudaStream_t s = ctx.stream;
  cudaMemcpyAsync(d_off, offsets, (np + 1)*4, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_pa, pose_prev, 96*np, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_pb, pose_cur, 96*np, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_h, motion_init, 96*np, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_cal, calib5, 40*np, cudaMemcpyHostToDevice, s);
  if (total > 0) { cudaMemcpyAsync(d_ka, kp_prev, 16*(size_t)total, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_kb, kp_cur, 16*(size_t)total, cudaMemcpyHostToDevice, s);
                   cudaMemcpyAsync(d_pt0, points_init, 48*(size_t)total, cudaMemcpyHostToDevice, s); }
  S.off = d_off; S.pose_a = d_pa; S.pose_b = d_pb; S.motion0 = d_h; S.calib = d_cal; S.kp_a = d_ka; S.kp_b = d_kb; S.pt0 = d_pt0;
  S.isig_proj = 1.0/P.projection_sigma; S.isig_motion = 1.0/P.landmark_motion_sigma; S.isig_prior = 1.0/P.pose_prior_sigma; S.huber_k = P.huber_k;
  S.prm = P.lm;
  motion_refine_kernel<<<n_problems, STAR_THREADS, 0, s>>>(S);
  cudaMemcpyAsync(motion_out, S.motion_out, 96*np, cudaMemcpyDeviceToHost, s);
  if (poses_out) cudaMemcpyAsync(poses_out, S.poses_out, 192*np, cudaMemcpyDeviceToHost, s);
  if (total > 0 && points_out) cudaMemcpyAsync(points_out, S.pt_cur, 48*(size_t)total, cudaMemcpyDeviceToHost, s);
  if (total > 0 && motion_factor_error) cudaMemcpyAsync(motion_factor_error, S.motion_err, 8*(size_t)total, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(err_before, S.err_before, 8*np, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(err_after, S.err_after, 8*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(iterations, S.iterations, 4*np, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(inner_iterations, S.inner, 4*np, cudaMemcpyDeviceToHost, s);
  const cudaError_t e1 = cudaStreamSynchronize(s), e2 = cudaGetLastError();
  return (e1 == cudaSuccess && e2 == cudaSuccess) ? DYNOBA_OK : DYNOBA_ERR_CUDA;
}

// frees the per-device workspace and stream the batch entry points (these two and dynoba_pnp_ransac_batch) keep between calls
int dynoba_batch_release(int device) {
  if (device < 0 || device >= 64) return DYNOBA_ERR_BAD_ARG;
  StarContext& c = g_star[device];
  std::lock_guard<std::mutex> lock(c.mu);
  if (!c.base && !c.stream) return DYNOBA_OK;
  if (cudaSetDevice(device) != cudaSuccess) return DYNOBA_ERR_CUDA;
  if (c.stream) { cudaStreamSynchronize(c.stream); cudaStreamDestroy(c.stream); c.stream = nullptr; }
  if (c.base) { cudaFree(c.base); c.base = nullptr; c.cap = 0; }
  return DYNOBA_OK;
}

}  // extern "C"
