// kernels_srif.cu -- ObjectMotionSolverFilter's filter step (predict + robust update, srif.cuh) for every object of a frame in
// ONE launch.
//
// One CTA of SF_THREADS per object.  Thread 0 runs the 6x6 algebra (admission, key frame, reset, predict, the IRLS mean and
// camera, the outputs) on the state in shared memory; one thread per correspondence linearises, initialises points and
// weighs (srif_lin_one / srif_weight_one); the QR of the (3n + 6) x 7 stacked rows is a TSQR: warp w folds its contiguous
// chunk of correspondences, eight at a time, into a 7 x 7 triangle by Householder reflections across the warp (one row per
// lane), warp 0 starting from the prior rows [R0 | d0]; warp 0 then folds the SF_WARPS triangles, in warp order, into the
// new [R | d].  Every reduction is a fixed-order shuffle tree: no atomics, and a result does not depend on the batch around
// its object.
#include <cmath>
#include <mutex>
#include <vector>
#include "internal.cuh"
#include "landmark.cuh"
#include "srif.cuh"

namespace dynoba {

constexpr int SF_THREADS = 128;
constexpr int SF_WARPS = SF_THREADS/32;
constexpr int SF_BLOCK = 8;          // correspondences a warp folds per Householder pass: lanes 8..31 hold their 24 rows

struct SrifBatch {
  const int* off; const int* mode; const int* pnp;
  const double *Xp, *Xc, *K, *st_in;
  const double* z; const uint8_t* valid; const double* pc;
  double* m; uint8_t* has;
  double *lin, *e0, *rwe, *w;        // [total][21], [total] x 3: scratch
  double* st_out; int* status; uint8_t* solved; double *motion, *cov, *err, *before; int* counts;
  dynoba_object_srif_params P; double Rinv[9];
};

// QR of the 32 rows held one per lane (a[c] = column c) -> the 7 x 7 triangle in lanes 0..6, zeros below.  The reflectors
// are srif_fold's.
__device__ __forceinline__ void warp_householder(double (&a)[7], int lane) {
#pragma unroll
  for (int j = 0; j < 7; j++) {
    const double s = warp_sum(lane > j ? a[j]*a[j] : 0.0);
    const double alpha = __shfl_sync(0xffffffffu, a[j], j);
    if (s == 0.0) continue;
    const double nrm = sqrt(alpha*alpha + s), beta = alpha >= 0.0 ? -nrm : nrm;
    const double tau = (beta - alpha)/beta, v = lane == j ? 1.0 : (lane > j ? a[j]*(1.0/(alpha - beta)) : 0.0);
#pragma unroll
    for (int c = j + 1; c < 7; c++) {
      const double wc = warp_sum(v*a[c])*tau;
      a[c] -= v*wc;
    }
    if (lane == j) a[j] = beta;
    else if (lane > j) a[j] = 0.0;
  }
}

__global__ void __launch_bounds__(SF_THREADS) object_srif_kernel(SrifBatch S) {
  __shared__ double st[DYNOBA_SRIF_STATE];
  __shared__ double prior[42];
  __shared__ double cam[12], nad[36];
  __shared__ double tri[SF_WARPS][49];
  __shared__ int sh_status;
  const int ob = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int i0 = S.off[ob], n = S.off[ob + 1] - i0, mode = S.mode[ob];
  const double* K = S.K + 6*(size_t)ob;
  if (t == 0) {
    const int status = srif_admit(mode, n, S.P.min_new_inliers);
    for (int e = 0; e < DYNOBA_SRIF_STATE; e++) st[e] = S.st_in[DYNOBA_SRIF_STATE*(size_t)ob + e];
    double* before = S.before + 12*(size_t)ob;
    srif_eye(before);
    if (status == DYNOBA_SRIF_OK && mode != DYNOBA_SRIF_CONTINUE) {
      Pose Xp, Le; srif_pose_ld(S.Xp + 12*(size_t)ob, Xp);
      double sum[3] = { 0.0, 0.0, 0.0 };
      for (int i = 0; i < n; i++) for (int c = 0; c < 3; c++) sum[c] += S.pc[6*(size_t)(i0 + i) + c];
      srif_keyframe(Xp, sum, n, Le);
      if (mode == DYNOBA_SRIF_RESET) for (int e = 0; e < 12; e++) before[e] = st[SRIF_H + e];
      srif_reset(st, S.P.P0, Le);
    }
    sh_status = status;
    S.status[ob] = status;
  }
  __syncthreads();
  if (sh_status != DYNOBA_SRIF_OK) {
    for (int e = t; e < DYNOBA_SRIF_STATE; e += SF_THREADS) S.st_out[DYNOBA_SRIF_STATE*(size_t)ob + e] = st[e];
    for (int e = t; e < 36; e += SF_THREADS) {
      const int r = e % 12;
      S.motion[36*(size_t)ob + e] = (r == 0 || r == 4 || r == 8) ? 1.0 : 0.0;
      S.cov[36*(size_t)ob + e] = 0.0;
    }
    if (t == 0) {
      S.solved[ob] = 0; S.err[2*ob] = S.err[2*ob + 1] = 0.0;
      S.counts[3*ob] = S.counts[3*ob + 1] = S.counts[3*ob + 2] = 0;
    }
    return;
  }
  if (mode != DYNOBA_SRIF_CONTINUE) for (int i = t; i < n; i += SF_THREADS) S.has[i0 + i] = 0;
  int n_new = 0, n_clipped = 0;
  double err0 = 0.0, err1 = 0.0;
  for (int f = mode == DYNOBA_SRIF_CONTINUE ? 1 : 0; f < 2; f++) {
    const double* Xf = (f == 0 ? S.Xp : S.Xc) + 12*(size_t)ob;
    if (t == 0) {
      srif_predict(st, S.P.Q);
      Pose X, H, Le, C;
      srif_pose_ld(Xf, X); srif_pose_ld(st + SRIF_H, H); srif_pose_ld(st + SRIF_LE, Le);
      srif_pose_st(X, st + SRIF_XK);
      srif_camera(X, H, Le, C, nad);
      srif_pose_st(C, cam);
      for (int e = 0; e < 42; e++) prior[e] = st[e];
    }
    __syncthreads();
    {                                                                 // linearisation: one thread per correspondence
      Pose X, H, Le, C;
      srif_pose_ld(Xf, X); srif_pose_ld(st + SRIF_H, H); srif_pose_ld(st + SRIF_LE, Le); srif_pose_ld(cam, C);
      double nA[36];
      for (int e = 0; e < 36; e++) nA[e] = nad[e];
      for (int b = 0; b < n; b += SF_THREADS) {
        const int i = b + t;
        bool fresh = false;
        if (i < n) {
          const size_t g = (size_t)(i0 + i);
          fresh = srif_lin_one(X, H, Le, C, nA, K, S.Rinv, S.z + 6*g + 3*f, S.valid[2*g + f] != 0, S.pc + 6*g + 3*f,
                               S.m + 3*g, S.has + g, S.lin + SRIF_LIN*g, S.e0 + g);
          S.rwe[g] = 0.0;
        }
        n_new += __syncthreads_count(fresh);
      }
    }
    for (int it = 0; it < S.P.irls_iterations; it++) {
      if (t == 0) {
        Pose X, Hc, Le, C;
        srif_pose_ld(Xf, X); srif_mean(st, Hc); srif_pose_ld(st + SRIF_LE, Le);
        srif_camera(X, Hc, Le, C, nullptr);
        srif_pose_st(C, cam);
      }
      __syncthreads();
      {                                                               // weights: one thread per correspondence
        Pose C; srif_pose_ld(cam, C);
        n_clipped = 0;
        for (int b = 0; b < n; b += SF_THREADS) {
          const int i = b + t;
          bool clipped = false;
          if (i < n) {
            const size_t g = (size_t)(i0 + i);
            S.w[g] = srif_weight_one(C, K, S.Rinv, S.P.huber_k, S.z + 6*g + 3*f, S.valid[2*g + f] != 0, S.m + 3*g, S.rwe + g, &clipped);
          }
          n_clipped += __syncthreads_count(clipped);
        }
      }
      {                                                               // TSQR, stage 1: each warp's chunk -> tri[warp]
        double a[7];
#pragma unroll
        for (int c = 0; c < 7; c++) a[c] = (warp == 0 && lane < 6) ? (c < 6 ? prior[SRIF_R + 6*lane + c] : prior[SRIF_D + lane]) : 0.0;
        const int per = (n + SF_WARPS - 1)/SF_WARPS, c0 = min(n, warp*per), c1 = min(n, c0 + per);
        for (int b = c0; b < c1; b += SF_BLOCK) {
          if (lane >= 8) {
            const int j = lane - 8, ci = b + j/3, r = j % 3;
            double row[7] = { 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0 };
            if (ci < c1) {
              const size_t g = (size_t)(i0 + ci);
              const double wi = S.w[g];
              if (!(wi < SRIF_MIN_W)) srif_whiten_row(S.P.R_noise, wi, S.lin + SRIF_LIN*g, r, row);
            }
#pragma unroll
            for (int c = 0; c < 7; c++) a[c] = row[c];
          } else if (lane == 7) {
#pragma unroll
            for (int c = 0; c < 7; c++) a[c] = 0.0;
          }
          warp_householder(a, lane);
        }
        if (lane < 7) {
#pragma unroll
          for (int c = 0; c < 7; c++) tri[warp][7*lane + c] = a[c];
        }
      }
      __syncthreads();
      if (warp == 0) {                                                // stage 2: the warps' triangles, in warp order
        double a[7];
        const int wq = lane/7, r = lane % 7;
#pragma unroll
        for (int c = 0; c < 7; c++) a[c] = wq < SF_WARPS ? tri[wq][7*r + c] : 0.0;
        warp_householder(a, lane);
        if (lane < 6) {                                               // srif_take_row, with a[] kept in registers
          double dg = 0.0;
#pragma unroll
          for (int c = 0; c < 6; c++) if (c == lane) dg = a[c];
          const double sg = dg < 0.0 ? -1.0 : 1.0;
#pragma unroll
          for (int c = 0; c < 6; c++) st[SRIF_R + 6*lane + c] = c < lane ? 0.0 : sg*a[c];
          st[SRIF_D + lane] = sg*a[6];
        }
      }
      __syncthreads();
    }
    if (t == 0) {
      double s0 = 0.0, s1 = 0.0;
      for (int i = 0; i < n; i++) { const double e = S.e0[i0 + i], r = S.rwe[i0 + i]; s0 += e*e; s1 += r*r; }
      err0 = sqrt(s0); err1 = sqrt(s1);
    }
  }
  if (t == 0) {
    srif_outputs(st, S.motion + 36*(size_t)ob, S.cov + 36*(size_t)ob);
    for (int e = 0; e < DYNOBA_SRIF_STATE; e++) S.st_out[DYNOBA_SRIF_STATE*(size_t)ob + e] = st[e];
    S.solved[ob] = S.pnp[ob] == DYNOBA_TRACK_VALID;
    S.err[2*ob] = err0; S.err[2*ob + 1] = err1;
    S.counts[3*ob] = n_new; S.counts[3*ob + 1] = n - n_new; S.counts[3*ob + 2] = n_clipped;
  }
}

static bool finite_all(const double* a, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(a[i])) return false;
  return true;
}
static bool spd_host(const double* A, int N) {
  for (int i = 0; i < N; i++) for (int j = 0; j < i; j++) if (A[N*i + j] != A[N*j + i]) return false;
  double L[36];
  return N == 6 ? srif_chol<6>(A, L) : srif_chol<3>(A, L);
}

}  // namespace dynoba

using namespace dynoba;

extern "C" {

void dynoba_object_srif_default_params(dynoba_object_srif_params* p) {
  if (!p) return;
  for (int i = 0; i < 36; i++) { p->P0[i] = i % 7 == 0 ? 0.3 : 0.0; p->Q[i] = i % 7 == 0 ? 0.2 : 0.0; }   // MotionSolver.cc:1880-1886
  for (int i = 0; i < 9; i++) p->R_noise[i] = i % 4 == 0 ? 1.0 : 0.0;
  p->huber_k = 0.1;                                                                                    // kHuberKFilter, :1905
  p->irls_iterations = 2;                                                                              // :1940, :1964
  p->min_new_inliers = 4;                                                                              // :1888
}

int dynoba_object_srif_batch(int device, int32_t n_objects, const int32_t* offsets, const int32_t* mode,
                             const int32_t* pnp_status, const double* pose_prev, const double* pose_cur, const double* calib6,
                             const dynoba_object_srif_params* prm, const double* state_in, double* state_out,
                             const double* stereo, const uint8_t* stereo_valid, const double* points_cam, double* m_L,
                             uint8_t* has_point, int32_t* status, uint8_t* solved, double* motion_out, double* cov_out,
                             double* errors, double* before_reset, int32_t* counts) {
  if (n_objects == 0) return DYNOBA_OK;
  dynoba_object_srif_params P; if (prm) P = *prm; else dynoba_object_srif_default_params(&P);
  if (n_objects < 0 || n_objects >= (1 << 24) || !offsets || !mode || !pnp_status || !pose_prev || !pose_cur || !calib6 ||
      !state_in || !state_out || !status || !solved || !motion_out || !cov_out || !errors || !before_reset || !counts)
    return DYNOBA_ERR_BAD_ARG;
  if (!finite_all(P.P0, 36) || !finite_all(P.Q, 36) || !finite_all(P.R_noise, 9) || !spd_host(P.P0, 6) || !spd_host(P.Q, 6) ||
      !spd_host(P.R_noise, 3) || !(P.huber_k > 0) || !std::isfinite(P.huber_k) || P.irls_iterations < 1 || P.min_new_inliers < 0)
    return DYNOBA_ERR_BAD_ARG;
  const int total = offsets[n_objects];
  if (offsets[0] != 0 || total < 0 || total >= (1 << 28) || (total > 0 && (!stereo || !stereo_valid || !points_cam || !m_L || !has_point)))
    return DYNOBA_ERR_BAD_ARG;
  for (int o = 0; o < n_objects; o++) {
    if (offsets[o + 1] < offsets[o]) return DYNOBA_ERR_BAD_ARG;
    if (mode[o] != DYNOBA_SRIF_NEW && mode[o] != DYNOBA_SRIF_RESET && mode[o] != DYNOBA_SRIF_CONTINUE) return DYNOBA_ERR_BAD_ARG;
    const double* K = calib6 + 6*(size_t)o;
    if (!(K[0] > 0) || !(K[1] > 0) || !(K[5] > 0)) return DYNOBA_ERR_BAD_ARG;
  }
  const size_t no = (size_t)n_objects, nt = (size_t)total;
  if (!finite_all(pose_prev, 12*no) || !finite_all(pose_cur, 12*no) || !finite_all(calib6, 6*no) ||
      !finite_all(state_in, DYNOBA_SRIF_STATE*no) || !finite_all(points_cam, 6*nt) || !finite_all(m_L, 3*nt))
    return DYNOBA_ERR_BAD_ARG;
  for (size_t i = 0; i < nt; i++) {
    if (has_point[i] > 1 || stereo_valid[2*i] > 1 || stereo_valid[2*i + 1] > 1) return DYNOBA_ERR_BAD_ARG;
    for (int f = 0; f < 2; f++) if (stereo_valid[2*i + f] && !finite_all(stereo + 6*i + 3*f, 3)) return DYNOBA_ERR_BAD_ARG;
  }
  if (device < 0 || device >= 64) return DYNOBA_ERR_CUDA;
  StarContext& ctx = star_context(device);
  std::lock_guard<std::mutex> lock(ctx.mu);
  int rc = star_device_ready(device); if (rc) return rc;
  const size_t ntt = std::max<size_t>(nt, 1);
  DeviceBlock blk; SrifBatch S{};
  int *d_off, *d_mode, *d_pnp; double *d_Xp, *d_Xc, *d_K, *d_st, *d_z, *d_pc; uint8_t* d_valid;
  auto layout = [&]() {
    d_off = blk.take<int>(no + 1); d_mode = blk.take<int>(no); d_pnp = blk.take<int>(no);
    d_Xp = blk.take<double>(12*no); d_Xc = blk.take<double>(12*no); d_K = blk.take<double>(6*no); d_st = blk.take<double>(DYNOBA_SRIF_STATE*no);
    d_z = blk.take<double>(6*ntt); d_valid = blk.take<uint8_t>(2*ntt); d_pc = blk.take<double>(6*ntt);
    S.m = blk.take<double>(3*ntt); S.has = blk.take<uint8_t>(ntt);
    S.lin = blk.take<double>(SRIF_LIN*ntt); S.e0 = blk.take<double>(ntt); S.rwe = blk.take<double>(ntt); S.w = blk.take<double>(ntt);
    S.st_out = blk.take<double>(DYNOBA_SRIF_STATE*no); S.status = blk.take<int>(no); S.solved = blk.take<uint8_t>(no);
    S.motion = blk.take<double>(36*no); S.cov = blk.take<double>(36*no); S.err = blk.take<double>(2*no);
    S.before = blk.take<double>(12*no); S.counts = blk.take<int>(3*no);
  };
  layout();
  if (!blk.allocate(ctx)) { cudaGetLastError(); return DYNOBA_ERR_CUDA; }
  layout();
  S.off = d_off; S.mode = d_mode; S.pnp = d_pnp; S.Xp = d_Xp; S.Xc = d_Xc; S.K = d_K; S.st_in = d_st; S.z = d_z; S.valid = d_valid; S.pc = d_pc;
  S.P = P; srif_inv3(P.R_noise, S.Rinv);
  cudaStream_t s = ctx.stream;
  cudaMemcpyAsync(d_off, offsets, 4*(no + 1), cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_mode, mode, 4*no, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_pnp, pnp_status, 4*no, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_Xp, pose_prev, 96*no, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_Xc, pose_cur, 96*no, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_K, calib6, 48*no, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_st, state_in, 8*DYNOBA_SRIF_STATE*no, cudaMemcpyHostToDevice, s);
  if (nt > 0) {
    cudaMemcpyAsync(d_z, stereo, 48*nt, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(d_valid, stereo_valid, 2*nt, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_pc, points_cam, 48*nt, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(S.m, m_L, 24*nt, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(S.has, has_point, nt, cudaMemcpyHostToDevice, s);
  }
  object_srif_kernel<<<n_objects, SF_THREADS, 0, s>>>(S);
  cudaMemcpyAsync(state_out, S.st_out, 8*DYNOBA_SRIF_STATE*no, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(status, S.status, 4*no, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(solved, S.solved, no, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(motion_out, S.motion, 288*no, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(cov_out, S.cov, 288*no, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(errors, S.err, 16*no, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(before_reset, S.before, 96*no, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(counts, S.counts, 12*no, cudaMemcpyDeviceToHost, s);
  if (nt > 0) { cudaMemcpyAsync(m_L, S.m, 24*nt, cudaMemcpyDeviceToHost, s); cudaMemcpyAsync(has_point, S.has, nt, cudaMemcpyDeviceToHost, s); }
  const cudaError_t e1 = cudaStreamSynchronize(s), e2 = cudaGetLastError();
  return (e1 == cudaSuccess && e2 == cudaSuccess) ? DYNOBA_OK : DYNOBA_ERR_CUDA;
}

}  // extern "C"
