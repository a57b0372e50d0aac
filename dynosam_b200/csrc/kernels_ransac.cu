// kernels_ransac.cu -- the front end's 3D-2D absolute-pose RANSAC for every problem of a frame (camera + objects) in ONE launch.
//
// EgoMotionSolver::geometricOutlierRejection3d2d (dynosam/src/frontend/vision/MotionSolver.cc:234-311) runs OpenGV's
// Ransac<AbsolutePoseSacProblem> with the KNEIP minimal solver once for the camera and once per object
// (ObjectMotionSovlerF2F::geometricOutlierRejection3d2d, :630-713).  Semantics: tests/pnp_oracle.py (steps 1-7, [OpenGV-ext]);
// every expression below evaluates the same IEEE operations in the same order as the oracle, which is why this translation
// unit is compiled with -fmad=false.
//
// One persistent CTA per problem.  The draws are a stateless stream (draw h of problem p is a function of (seed, p, h)), so
// the CTA evaluates them in chunks: one thread per draw builds its model (sampler, Kneip P3P, disambiguation), the warps count
// the inliers of every model of the chunk over the correspondences staged through shared memory in tiles, and thread 0
// replays OpenGV's sequential loop (Ransac::computeModel) over the chunk's counts.  The replay consumes a prefix of the stream
// and stops exactly where the sequential loop stops, so the results do not depend on the chunk size; the CTA goes on to the
// next chunk only while the loop has not ended.  A call is one launch whatever the iteration count.
#include <cfloat>
#include <climits>
#include <cmath>
#include <algorithm>
#include <mutex>
#include <vector>
#include "../../include/dynoba.h"
#include "internal.cuh"

namespace dynoba {

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS/32;
constexpr int RS_CHUNK = 256;          // draws per chunk at most (one per thread); chunks grow 32, 64, 128, 256, 256, ...
constexpr int RS_TILE = 256;           // correspondences per shared-memory tile
constexpr int RS_MIN_N = 5;            // MotionSolver.cc:241

struct RansacBatch {
  int nprob; const int* off;                      // [nprob + 1]
  const double* calib; const double* pts; const double* kp; const double* thr;     // [nprob][5], [total][3], [total][2], [nprob]
  int max_it, min_inl; double log1mp; unsigned long long seed;
  double* bear;                                   // [total][3] work
  double* pose_out; unsigned char* inl; int* n_inl; int* status; int* iters; int* skipped; int* best_h;
  int* hyp_counts;                                // [nprob][max_it + 1] or nullptr
};

// ---- step 4: sampler
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30))*0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27))*0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// the four draws of a partial Fisher-Yates over the identity permutation: step j swaps positions j and t; the permutation is
// kept as the list of writes (position, value), later writes override earlier ones (fully unrolled: registers only)
__device__ __forceinline__ void draw_indices(unsigned long long seed, int p, long long h, int n, int (&sel)[4]) {
  int pos[8], val[8];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const unsigned long long key = ((unsigned long long)p << 40) | ((unsigned long long)h << 2) | (unsigned long long)j;
    const unsigned long long r = splitmix64(seed + key);
    const int t = j + (int)(r % (unsigned long long)(n - j));
    int vt = t, vj = j;
#pragma unroll
    for (int s = 0; s < 2*j; s++) { if (pos[s] == t) vt = val[s]; if (pos[s] == j) vj = val[s]; }
    pos[2*j] = t; val[2*j] = vj; pos[2*j + 1] = j; val[2*j + 1] = vt;
    sel[j] = vt;
  }
}

// ---- step 3: score under the model M = (R row-major, C)
__device__ __forceinline__ double pnp_score(const double* M, double P0, double P1, double P2, double f0, double f1, double f2) {
  const double d0 = P0 - M[9], d1 = P1 - M[10], d2 = P2 - M[11];
  const double q0 = (M[0]*d0 + M[3]*d1) + M[6]*d2;
  const double q1 = (M[1]*d0 + M[4]*d1) + M[7]*d2;
  const double q2 = (M[2]*d0 + M[5]*d1) + M[8]*d2;
  const double nn = sqrt((q0*q0 + q1*q1) + q2*q2);
  const double dot = ((q0/nn)*f0 + (q1/nn)*f1) + (q2/nn)*f2;
  return 1.0 - dot;
}

// ---- step 5: Kneip P3P
struct V3 { double x, y, z; };
__device__ __forceinline__ V3 v3sub(V3 a, V3 b) { return V3{ a.x - b.x, a.y - b.y, a.z - b.z }; }
__device__ __forceinline__ V3 v3cross(V3 a, V3 b) { return V3{ a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x }; }
__device__ __forceinline__ double v3norm(V3 a) { return sqrt((a.x*a.x + a.y*a.y) + a.z*a.z); }
__device__ __forceinline__ V3 v3div(V3 a, double s) { return V3{ a.x/s, a.y/s, a.z/s }; }
__device__ __forceinline__ V3 rows_times(const V3* T, V3 v) {
  return V3{ (T[0].x*v.x + T[0].y*v.y) + T[0].z*v.z, (T[1].x*v.x + T[1].y*v.y) + T[1].z*v.z, (T[2].x*v.x + T[2].y*v.y) + T[2].z*v.z };
}
__device__ __forceinline__ double comp(V3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

// complex helpers (re, im), the oracle's _csqrt / _ccbrt / _cdiv
__device__ __forceinline__ void csqrt_(double ar, double ai, double& r, double& i) {
  if (ai == 0.0) { if (ar >= 0.0) { r = sqrt(ar); i = 0.0; } else { r = 0.0; i = sqrt(-ar); } return; }
  const double m = sqrt(ar*ar + ai*ai);
  const double t = sqrt((m + fabs(ar))*0.5);
  if (ar >= 0.0) { r = t; i = ai/(2.0*t); } else { r = fabs(ai)/(2.0*t); i = copysign(t, ai); }
}
__device__ __forceinline__ void ccbrt_(double ar, double ai, double& r, double& i) {
  if (ai == 0.0 && ar >= 0.0) { r = cbrt(ar); i = 0.0; return; }
  const double m = cbrt(sqrt(ar*ar + ai*ai));
  const double th = atan2(ai, ar)/3.0;
  r = m*cos(th); i = m*sin(th);
}
__device__ __forceinline__ void cdiv_(double ar, double ai, double br, double bi, double& r, double& i) {
  const double den = br*br + bi*bi;
  r = (ar*br + ai*bi)/den; i = (ai*br - ar*bi)/den;
}

__device__ __forceinline__ void solve_quartic(double A, double B, double C, double D, double E, double* roots) {
  const double A_pw2 = A*A, B_pw2 = B*B, A_pw3 = A_pw2*A, B_pw3 = B_pw2*B, A_pw4 = A_pw3*A, B_pw4 = B_pw3*B;
  const double alpha = (-3.0*B_pw2)/(8.0*A_pw2) + C/A;
  const double beta = (B_pw3/(8.0*A_pw3) - (B*C)/(2.0*A_pw2)) + D/A;
  const double gamma = (((-3.0*B_pw4)/(256.0*A_pw4) + (B_pw2*C)/(16.0*A_pw3)) - (B*D)/(4.0*A_pw2)) + E/A;
  const double alpha_pw2 = alpha*alpha, alpha_pw3 = alpha_pw2*alpha;
  const double P = -alpha_pw2/12.0 - gamma;
  const double Q = (-alpha_pw3/108.0 + alpha*gamma/3.0) - beta*beta/8.0;
  double sr, si; csqrt_(Q*Q/4.0 + P*P*P/27.0, 0.0, sr, si);
  const double Rr = -Q/2.0 + sr, Ri = si;
  double Ur, Ui; ccbrt_(Rr, Ri, Ur, Ui);
  double yr, yi;
  if (Ur == 0.0) { double cr, ci; ccbrt_(Q, 0.0, cr, ci); yr = -5.0*alpha/6.0 - cr; yi = -ci; }
  else { double qr, qi; cdiv_(P, 0.0, 3.0*Ur, 3.0*Ui, qr, qi); yr = (-5.0*alpha/6.0 - qr) + Ur; yi = -qi + Ui; }
  double wr, wi; csqrt_(alpha + 2.0*yr, 2.0*yi, wr, wi);
  double br_, bi_; cdiv_(2.0*beta, 0.0, wr, wi, br_, bi_);
  const double base = -B/(4.0*A);
  double s1r, s1i, s2r, s2i;
  csqrt_(-((3.0*alpha + 2.0*yr) + br_), -(2.0*yi + bi_), s1r, s1i);
  csqrt_(-((3.0*alpha + 2.0*yr) - br_), -(2.0*yi - bi_), s2r, s2i);
  roots[0] = base + 0.5*(wr + s1r); roots[1] = base + 0.5*(wr - s1r);
  roots[2] = base + 0.5*(-wr + s2r); roots[3] = base + 0.5*(-wr - s2r);
}

// The model of one draw: Kneip's four candidates from samples 0..2, the one of least score of sample 3 (strict <, from 1e6).
// false = skipped (collinear world triple, or no candidate wins).
__device__ __forceinline__ bool p3p_model(const V3* Pw, const V3* Fb, double* out) {
  V3 P1 = Pw[0], P2 = Pw[1]; const V3 P3 = Pw[2];
  if (v3norm(v3cross(v3sub(P2, P1), v3sub(P3, P1))) == 0.0) return false;
  V3 f1 = Fb[0], f2 = Fb[1]; const V3 f3o = Fb[2];
  V3 T[3];
  T[0] = f1; T[2] = v3div(v3cross(f1, f2), v3norm(v3cross(f1, f2))); T[1] = v3cross(T[2], T[0]);
  V3 f3 = rows_times(T, f3o);
  if (f3.z > 0.0) {
    f1 = Fb[1]; f2 = Fb[0];
    T[0] = f1; T[2] = v3div(v3cross(f1, f2), v3norm(v3cross(f1, f2))); T[1] = v3cross(T[2], T[0]);
    f3 = rows_times(T, f3o);
    P1 = Pw[1]; P2 = Pw[0];
  }
  V3 N[3];
  N[0] = v3sub(P2, P1); const double d_12 = v3norm(N[0]); N[0] = v3div(N[0], d_12);
  N[2] = v3cross(N[0], v3sub(P3, P1)); N[2] = v3div(N[2], v3norm(N[2]));
  N[1] = v3cross(N[2], N[0]);
  const V3 P3n = rows_times(N, v3sub(P3, P1));
  const double f_1 = f3.x/f3.z, f_2 = f3.y/f3.z;
  const double p_1 = P3n.x, p_2 = P3n.y;
  const double cos_beta = (f1.x*f2.x + f1.y*f2.y) + f1.z*f2.z;
  double b = 1.0/(1.0 - cos_beta*cos_beta) - 1.0;
  b = cos_beta < 0.0 ? -sqrt(b) : sqrt(b);
  const double f_1_pw2 = f_1*f_1, f_2_pw2 = f_2*f_2;
  const double p_1_pw2 = p_1*p_1, p_1_pw3 = p_1_pw2*p_1, p_1_pw4 = p_1_pw3*p_1;
  const double p_2_pw2 = p_2*p_2, p_2_pw3 = p_2_pw2*p_2, p_2_pw4 = p_2_pw3*p_2;
  const double d_12_pw2 = d_12*d_12, b_pw2 = b*b;
  // the same text as tests/pnp_oracle.py; + and - associate to the left in both languages
  const double F0 = -f_2_pw2*p_2_pw4 - p_2_pw4*f_1_pw2 - p_2_pw4;
  const double F1 = 2.0*p_2_pw3*d_12*b + 2.0*f_2_pw2*p_2_pw3*d_12*b - 2.0*f_2*p_2_pw3*f_1*d_12;
  const double F2 = (-f_2_pw2*p_2_pw2*p_1_pw2 - f_2_pw2*p_2_pw2*d_12_pw2*b_pw2 - f_2_pw2*p_2_pw2*d_12_pw2 + f_2_pw2*p_2_pw4 + p_2_pw4*f_1_pw2
          + 2.0*p_1*p_2_pw2*d_12 + 2.0*f_1*f_2*p_1*p_2_pw2*d_12*b - p_2_pw2*p_1_pw2*f_1_pw2 + 2.0*p_1*p_2_pw2*f_2_pw2*d_12
          - p_2_pw2*d_12_pw2*b_pw2 - 2.0*p_1_pw2*p_2_pw2);
  const double F3 = 2.0*p_1_pw2*p_2*d_12*b + 2.0*f_2*p_2_pw3*f_1*d_12 - 2.0*f_2_pw2*p_2_pw3*d_12*b - 2.0*p_1*p_2*d_12_pw2*b;
  const double F4 = (-2.0*f_2*p_2_pw2*f_1*p_1*d_12*b + f_2_pw2*p_2_pw2*d_12_pw2 + 2.0*p_1_pw3*d_12 - p_1_pw2*d_12_pw2
          + f_2_pw2*p_2_pw2*p_1_pw2 - p_1_pw4 - 2.0*f_2_pw2*p_2_pw2*p_1*d_12 + p_2_pw2*f_1_pw2*p_1_pw2
          + f_2_pw2*p_2_pw2*d_12_pw2*b_pw2);
  double roots[4];
  solve_quartic(F0, F1, F2, F3, F4, roots);
  double best = 1e6; bool found = false;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const double r = roots[q];
    const double cot_alpha = ((-f_1*p_1/f_2 - r*p_2) + d_12*b)/((-f_1*r*p_2/f_2 + p_1) - d_12);
    const double cos_theta = r;
    const double sin_theta = sqrt(1.0 - r*r);
    const double sin_alpha = sqrt(1.0/(cot_alpha*cot_alpha + 1.0));
    double cos_alpha = sqrt(1.0 - sin_alpha*sin_alpha);
    if (cot_alpha < 0.0) cos_alpha = -cos_alpha;
    const double g = sin_alpha*b + cos_alpha;
    const double Cv[3] = { d_12*cos_alpha*g, cos_theta*d_12*sin_alpha*g, sin_theta*d_12*sin_alpha*g };
    const double Rm[3][3] = { { -cos_alpha, -sin_alpha*cos_theta, -sin_alpha*sin_theta },
                              { sin_alpha, -cos_alpha*cos_theta, -cos_alpha*sin_theta },
                              { 0.0, -sin_theta, cos_theta } };
    double M[3][3], cand[12];
    for (int i = 0; i < 3; i++)
      for (int k = 0; k < 3; k++) M[i][k] = (comp(N[0], i)*Rm[k][0] + comp(N[1], i)*Rm[k][1]) + comp(N[2], i)*Rm[k][2];
    for (int i = 0; i < 3; i++)
      for (int k = 0; k < 3; k++) cand[3*i + k] = (M[i][0]*comp(T[0], k) + M[i][1]*comp(T[1], k)) + M[i][2]*comp(T[2], k);
    for (int i = 0; i < 3; i++) cand[9 + i] = comp(P1, i) + ((comp(N[0], i)*Cv[0] + comp(N[1], i)*Cv[1]) + comp(N[2], i)*Cv[2]);
    const double s = pnp_score(cand, Pw[3].x, Pw[3].y, Pw[3].z, Fb[3].x, Fb[3].y, Fb[3].z);
    if (s < best) { best = s; found = true; for (int e = 0; e < 12; e++) out[e] = cand[e]; }
  }
  return found;
}

__global__ void __launch_bounds__(RS_THREADS, 1) pnp_ransac_kernel(RansacBatch S) {
  __shared__ double sh_model[RS_CHUNK*12];
  __shared__ double sh_tile[6*RS_TILE];           // P (3) | f (3), entry-major
  __shared__ int sh_cnt[RS_CHUNK];                // inliers of each model of the chunk, -1 = skipped draw
  __shared__ double sh_best[12];
  __shared__ double sh_k;
  __shared__ int sh_it, sh_skipped, sh_best_cnt, sh_best_h, sh_done, sh_ninl;
  __shared__ long long sh_h0;
  const int pb = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int f0 = S.off[pb], n = S.off[pb + 1] - f0;
  const double* P = S.pts + 3*(size_t)f0;
  double* F = S.bear + 3*(size_t)f0;
  const double thr = S.thr[pb];
  // step 1: bearings (Cal3_S2 inverse in closed form)
  {
    const double fx = S.calib[5*pb], fy = S.calib[5*pb + 1], sk = S.calib[5*pb + 2], u0 = S.calib[5*pb + 3], v0 = S.calib[5*pb + 4];
    for (int i = t; i < n; i += RS_THREADS) {
      const double u = S.kp[2*(size_t)(f0 + i)], v = S.kp[2*(size_t)(f0 + i) + 1];
      const double y = (v - v0)/fy;
      const double x = ((u - u0) - sk*y)/fx;
      const double nrm = sqrt((x*x + y*y) + 1.0);
      F[3*(size_t)i] = x/nrm; F[3*(size_t)i + 1] = y/nrm; F[3*(size_t)i + 2] = 1.0/nrm;
    }
  }
  if (t == 0) { sh_it = 0; sh_skipped = 0; sh_best_cnt = -INT_MAX; sh_best_h = -1; sh_done = n < RS_MIN_N; sh_k = 1.0; sh_h0 = 0; sh_ninl = 0; }
  __syncthreads();
  const int max_skip = 10*S.max_it;
  for (int c = 0; !sh_done; c++) {
    const int nch = min(RS_CHUNK, 32 << min(c, 3));
    if (t < nch) {                                                    // one draw per thread
      int sel[4]; draw_indices(S.seed, pb, sh_h0 + t, n, sel);
      V3 Pw[4], Fb[4];
      for (int j = 0; j < 4; j++) {
        Pw[j] = V3{ P[3*(size_t)sel[j]], P[3*(size_t)sel[j] + 1], P[3*(size_t)sel[j] + 2] };
        Fb[j] = V3{ F[3*(size_t)sel[j]], F[3*(size_t)sel[j] + 1], F[3*(size_t)sel[j] + 2] };
      }
      sh_cnt[t] = p3p_model(Pw, Fb, sh_model + 12*t) ? 0 : -1;
    }
    for (int tile0 = 0; tile0 < n; tile0 += RS_TILE) {                 // inlier counts, correspondences tiled through shared memory
      const int tn = min(RS_TILE, n - tile0);
      __syncthreads();
      if (t < tn) for (int e = 0; e < 3; e++) { sh_tile[e*RS_TILE + t] = P[3*(size_t)(tile0 + t) + e]; sh_tile[(3 + e)*RS_TILE + t] = F[3*(size_t)(tile0 + t) + e]; }
      __syncthreads();
      for (int m = warp; m < nch; m += RS_WARPS) {
        if (sh_cnt[m] < 0) continue;
        double M[12];
        for (int e = 0; e < 12; e++) M[e] = sh_model[12*m + e];
        int cnt = 0;
        for (int j0 = 0; j0 < tn; j0 += 32) {
          const int j = j0 + lane;
          const bool in = j < tn && pnp_score(M, sh_tile[j], sh_tile[RS_TILE + j], sh_tile[2*RS_TILE + j],
                                              sh_tile[3*RS_TILE + j], sh_tile[4*RS_TILE + j], sh_tile[5*RS_TILE + j]) < thr;
          cnt += __popc(__ballot_sync(0xffffffffu, in));
        }
        if (lane == 0) sh_cnt[m] += cnt;
      }
    }
    __syncthreads();
    if (t == 0) {                                                     // step 6: OpenGV's sequential loop over this chunk's draws
      int it = sh_it, skipped = sh_skipped, best = sh_best_cnt, best_h = sh_best_h; double k = sh_k;
      bool done = false;
      for (int m = 0; m < nch; m++) {
        if (!(it < k && skipped < max_skip)) { done = true; break; }
        if (sh_cnt[m] < 0) { skipped++; continue; }
        const int cnt = sh_cnt[m];
        if (S.hyp_counts) S.hyp_counts[(size_t)pb*(S.max_it + 1) + it] = cnt;
        if (cnt > best) {
          best = cnt; best_h = (int)(sh_h0 + m);
          for (int e = 0; e < 12; e++) sh_best[e] = sh_model[12*m + e];
          const double w = (double)cnt/(double)n, w2 = w*w;
          const double pno = fmin(1.0 - DBL_EPSILON, fmax(DBL_EPSILON, 1.0 - w2*w2));
          k = S.log1mp/log(pno);
        }
        it++;
        if (it > S.max_it) { done = true; break; }
      }
      if (!(it < k && skipped < max_skip)) done = true;
      sh_it = it; sh_skipped = skipped; sh_best_cnt = best; sh_best_h = best_h; sh_k = k; sh_h0 += nch; sh_done = done;
    }
    __syncthreads();
  }
  // step 6 (end) and 7: the final inlier set under the best model
  const bool model = sh_best_h >= 0;
  for (int i = t; i < n; i += RS_THREADS) {
    const bool in = model && pnp_score(sh_best, P[3*(size_t)i], P[3*(size_t)i + 1], P[3*(size_t)i + 2], F[3*(size_t)i], F[3*(size_t)i + 1], F[3*(size_t)i + 2]) < thr;
    S.inl[f0 + i] = in ? 1 : 0;
    if (in) atomicAdd(&sh_ninl, 1);
  }
  __syncthreads();
  if (t == 0) {
    int st, ninl = sh_ninl;
    if (n < RS_MIN_N) st = DYNOBA_TRACK_FEW_MATCHES;
    else if (!model || (sh_it >= S.max_it && ninl == 0)) st = DYNOBA_TRACK_INVALID;
    else st = ninl >= S.min_inl ? DYNOBA_TRACK_VALID : DYNOBA_TRACK_FEW_MATCHES;
    const bool keep = model && st != DYNOBA_TRACK_INVALID;
    for (int e = 0; e < 12; e++) S.pose_out[12*pb + e] = keep ? sh_best[e] : ((e == 0 || e == 4 || e == 8) ? 1.0 : 0.0);
    S.status[pb] = st; S.n_inl[pb] = ninl; S.iters[pb] = sh_it; S.skipped[pb] = sh_skipped; S.best_h[pb] = model ? sh_best_h : -1;
  }
}

static bool all_finite(const double* a, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(a[i])) return false;
  return true;
}

}  // namespace dynoba

using namespace dynoba;

extern "C" {

void dynoba_pnp_ransac_default_params(dynoba_pnp_ransac_params* p) {
  if (!p) return;
  p->threshold_px = 1.0; p->max_iterations = 500; p->probability = 0.995;     // FrontendParams.yaml: ransac_threshold_pnp, _iterations, _probability
  p->min_inliers = 5;                                                          // MotionSolver.cc:299
  p->seed = DYNOBA_PNP_DEFAULT_SEED;
}

int dynoba_pnp_ransac_batch(int device, int32_t n_problems, const int32_t* offsets, const double* calib5, const double* points_world,
                            const double* keypoints, const dynoba_pnp_ransac_params* prm, double* pose_out, uint8_t* inlier_out,
                            int32_t* n_inliers, int32_t* status, int32_t* iterations, int32_t* skipped, int32_t* best_hypothesis,
                            int32_t* hyp_counts) {
  if (n_problems == 0) return DYNOBA_OK;
  dynoba_pnp_ransac_params P; if (prm) P = *prm; else dynoba_pnp_ransac_default_params(&P);
  if (n_problems < 0 || n_problems >= (1 << 24) || !offsets || !calib5 || !pose_out || !n_inliers || !status || !iterations || !skipped ||
      !best_hypothesis) return DYNOBA_ERR_BAD_ARG;
  if (!(P.threshold_px > 0) || !std::isfinite(P.threshold_px) || !(P.probability > 0 && P.probability < 1) || P.max_iterations < 1 ||
      P.max_iterations >= (1 << 24) || P.min_inliers < 0) return DYNOBA_ERR_BAD_ARG;
  const int total = offsets[n_problems];
  if (offsets[0] != 0 || total < 0 || (total > 0 && (!points_world || !keypoints || !inlier_out))) return DYNOBA_ERR_BAD_ARG;
  for (int p = 0; p < n_problems; p++) if (offsets[p + 1] < offsets[p]) return DYNOBA_ERR_BAD_ARG;
  if (!all_finite(calib5, 5*(size_t)n_problems) || !all_finite(points_world, 3*(size_t)total) || !all_finite(keypoints, 2*(size_t)total))
    return DYNOBA_ERR_BAD_ARG;
  std::vector<double> thr(n_problems);
  for (int p = 0; p < n_problems; p++) {
    const double fx = calib5[5*p], fy = calib5[5*p + 1];
    if (!(fx > 0) || !(fy > 0)) return DYNOBA_ERR_BAD_ARG;
    thr[p] = 1.0 - std::cos(std::atan(std::sqrt(2.0)*P.threshold_px/(0.5*(fx + fy))));     // MotionSolver.cc:269-274, host libm
  }
  if (device < 0 || device >= 64) return DYNOBA_ERR_CUDA;
  StarContext& ctx = star_context(device);
  std::lock_guard<std::mutex> lock(ctx.mu);
  int rc = star_device_ready(device); if (rc) return rc;
  const size_t np = (size_t)n_problems, nt = (size_t)std::max(total, 1), nh = np*(size_t)(P.max_iterations + 1);
  DeviceBlock blk; RansacBatch S{};
  int* d_off; double *d_cal, *d_pts, *d_kp, *d_thr;
  auto layout = [&]() {
    d_off = blk.take<int>(np + 1); d_cal = blk.take<double>(5*np); d_thr = blk.take<double>(np);
    d_pts = blk.take<double>(3*nt); d_kp = blk.take<double>(2*nt); S.bear = blk.take<double>(3*nt);
    S.pose_out = blk.take<double>(12*np); S.inl = blk.take<unsigned char>(nt);
    S.n_inl = blk.take<int>(np); S.status = blk.take<int>(np); S.iters = blk.take<int>(np); S.skipped = blk.take<int>(np); S.best_h = blk.take<int>(np);
    S.hyp_counts = hyp_counts ? blk.take<int>(nh) : nullptr;
  };
  layout();
  if (!blk.allocate(ctx)) { cudaGetLastError(); return DYNOBA_ERR_CUDA; }
  layout();
  S.nprob = n_problems; S.max_it = P.max_iterations; S.min_inl = P.min_inliers; S.seed = P.seed;
  S.log1mp = std::log(1.0 - P.probability);                          // host libm, as the threshold
  cudaStream_t s = ctx.stream;
  cudaMemcpyAsync(d_off, offsets, (np + 1)*4, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_cal, calib5, 40*np, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_thr, thr.data(), 8*np, cudaMemcpyHostToDevice, s);
  if (total > 0) { cudaMemcpyAsync(d_pts, points_world, 24*(size_t)total, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_kp, keypoints, 16*(size_t)total, cudaMemcpyHostToDevice, s); }
  if (S.hyp_counts) cudaMemsetAsync(S.hyp_counts, 0xff, 4*nh, s);   // -1 past the last evaluated model
  S.off = d_off; S.calib = d_cal; S.thr = d_thr; S.pts = d_pts; S.kp = d_kp;
  pnp_ransac_kernel<<<n_problems, RS_THREADS, 0, s>>>(S);
  cudaMemcpyAsync(pose_out, S.pose_out, 96*np, cudaMemcpyDeviceToHost, s);
  if (total > 0) cudaMemcpyAsync(inlier_out, S.inl, (size_t)total, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(n_inliers, S.n_inl, 4*np, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(status, S.status, 4*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(iterations, S.iters, 4*np, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(skipped, S.skipped, 4*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(best_hypothesis, S.best_h, 4*np, cudaMemcpyDeviceToHost, s);
  if (hyp_counts) cudaMemcpyAsync(hyp_counts, S.hyp_counts, 4*nh, cudaMemcpyDeviceToHost, s);
  const cudaError_t e1 = cudaStreamSynchronize(s), e2 = cudaGetLastError();
  return (e1 == cudaSuccess && e2 == cudaSuccess) ? DYNOBA_OK : DYNOBA_ERR_CUDA;
}

}  // extern "C"
