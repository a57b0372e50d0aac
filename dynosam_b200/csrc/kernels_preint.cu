// kernels_preint.cu -- dynoba_imu_preintegrate_batch: combined IMU preintegration (preint.cuh) of every frame interval of a
// batch in one launch, one warp per interval.
//
// The state chain (3x3 algebra, one sample after the other) is serial: lane 0 runs it and forms F's first nine rows and
// the injected noise Q of the step in shared memory.  The warp then shares F Sigma F^T + Q over its lanes through Sigma in
// shared memory (preint_cov_phase1 / 2; F's bias rows are the identity).  At the end lane 0 forms R (preint_sqrt_info)
// and the warp stores the record, Sigma and R.  A warp touches nothing but its own interval, so the results do not depend
// on how many intervals share a launch or a CTA.
#include <cstddef>
#include "internal.cuh"
#include "preint.cuh"

namespace dynoba {

constexpr int PI_WARPS = 4;                     // intervals per CTA

struct PreintBatch {
  const int* off; const double* stamps; const double* acc_gyr; const double* bias;
  double* rec; double* cov; double* R; int* status;
  int n;
  dynoba_imu_params prm;
};

// per warp: Sigma, Q (U of the final factorisation), A | B | C of the step, F9 | T (R of the final factorisation)
struct PreintStage { double S[PI_COV]; double Q[PI_COV]; double A[81], B[27], C[27]; double FT[2*PI_FR*PI_D]; };

__global__ void __launch_bounds__(PI_WARPS*32) preint_kernel(PreintBatch P) {
  __shared__ PreintStage st[PI_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = blockIdx.x*PI_WARPS + warp;
  if (p >= P.n) return;                         // whole warps only: the kernel has no CTA-wide barrier
  PreintStage& W = st[warp];
  double* F9 = W.FT; double* T = W.FT + PI_FR*PI_D;
  for (int e = lane; e < PI_COV; e += 32) W.S[e] = 0.0;
  double bh[6];
  for (int k = 0; k < 6; k++) bh[k] = P.bias ? P.bias[6*(size_t)p + k] : 0.0;
  PreintState s; preint_reset(s);
  const int m0 = P.off[p], m1 = P.off[p + 1];
  __syncwarp();
  for (int i = m0; i < m1 - 1; i++) {
    if (lane == 0) {
      const double dt = P.stamps[i + 1] - P.stamps[i];
      const double* z = P.acc_gyr + 6*(size_t)i;
      preint_step(P.prm, bh, z, z + 3, dt, s, W.A, W.B, W.C);
      preint_F(W.A, W.B, W.C, F9);
      preint_noise(P.prm, W.B, W.C, dt, W.Q);
    }
    __syncwarp();
    preint_cov_phase1(F9, W.S, T, lane, 32);
    __syncwarp();
    preint_cov_phase2(F9, T, W.Q, W.S, lane, 32);
    __syncwarp();
  }
  if (lane == 0) {
    preint_record(s, bh, P.prm.n_gravity, P.rec + PI_REC*(size_t)p);
    P.status[p] = preint_sqrt_info(W.S, W.Q, W.FT);
  }
  __syncwarp();
  for (int e = lane; e < PI_COV; e += 32) { P.cov[PI_COV*(size_t)p + e] = W.S[e]; P.R[PI_COV*(size_t)p + e] = W.FT[e]; }
}

// the parameter check below reads every field before the flag as one array of doubles
static_assert(offsetof(dynoba_imu_params, has_body_P_sensor) == 96*sizeof(double), "dynoba_imu_params: 96 doubles, then the flag");

static bool finite_all(const double* a, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(a[i])) return false;
  return true;
}

}  // namespace dynoba

using namespace dynoba;

extern "C" {

void dynoba_imu_default_params(dynoba_imu_params* p) {
  if (!p) return;
  *p = dynoba_imu_params{};
  // [GTSAM-ext navigation/CombinedImuFactor.h PreintegrationCombinedParams, ImuFactor.h PreintegrationParams,
  // PreintegratedRotation.h]: accelerometer, gyroscope, integration, biasAcc, biasOmega covariances and biasAccOmegaInt
  // all default to the identity; body_P_sensor is unset
  for (int i = 0; i < 3; i++) {
    const int d = 4*i;
    p->accelerometer_cov[d] = p->gyroscope_cov[d] = p->integration_cov[d] = 1.0;
    p->bias_acc_cov[d] = p->bias_omega_cov[d] = 1.0;
  }
  for (int i = 0; i < 6; i++) p->bias_acc_omega_int[7*i] = 1.0;
  for (int i = 0; i < 3; i++) p->body_P_sensor[4*i] = 1.0;
}

int dynoba_imu_preintegrate_batch(int device, const dynoba_imu_params* params, int32_t n_intervals, const int32_t* offsets,
                                  const double* stamps, const double* acc_gyr, const double* bias_hat, double* record,
                                  double* cov, double* sqrt_info, int32_t* status) {
  if (n_intervals == 0) return DYNOBA_OK;
  if (n_intervals < 0 || n_intervals >= (1 << 24) || !params || !offsets || !stamps || !acc_gyr || !record || !cov ||
      !sqrt_info || !status) return DYNOBA_ERR_BAD_ARG;
  const dynoba_imu_params& P = *params;
  if (!finite_all(&P.n_gravity[0], offsetof(dynoba_imu_params, has_body_P_sensor)/sizeof(double))) return DYNOBA_ERR_BAD_ARG;
  if (P.has_body_P_sensor != 0 && P.has_body_P_sensor != 1) return DYNOBA_ERR_BAD_ARG;
  if (P.has_body_P_sensor) {                     // a rotation: R R^T = I to 1e-9, det > 0
    const double* R = P.body_P_sensor;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
      const double d = R[3*i]*R[3*j] + R[3*i + 1]*R[3*j + 1] + R[3*i + 2]*R[3*j + 2] - (i == j ? 1.0 : 0.0);
      if (!(std::fabs(d) <= 1e-9)) return DYNOBA_ERR_BAD_ARG;
    }
    const double det = R[0]*(R[4]*R[8] - R[5]*R[7]) - R[1]*(R[3]*R[8] - R[5]*R[6]) + R[2]*(R[3]*R[7] - R[4]*R[6]);
    if (!(det > 0)) return DYNOBA_ERR_BAD_ARG;
  }
  if (offsets[0] != 0) return DYNOBA_ERR_BAD_ARG;
  for (int p = 0; p < n_intervals; p++) {
    const int m0 = offsets[p], m1 = offsets[p + 1];
    if (m1 < m0 || m1 - m0 < 2) return DYNOBA_ERR_BAD_ARG;
    for (int i = m0; i < m1; i++) if (!std::isfinite(stamps[i])) return DYNOBA_ERR_BAD_ARG;
    for (int i = m0; i < m1 - 1; i++) {
      const double dt = stamps[i + 1] - stamps[i];
      if (!(dt > 0.0) || !std::isfinite(dt)) return DYNOBA_ERR_BAD_ARG;
      if (!finite_all(acc_gyr + 6*(size_t)i, 6)) return DYNOBA_ERR_BAD_ARG;
    }
  }
  if (bias_hat && !finite_all(bias_hat, 6*(size_t)n_intervals)) return DYNOBA_ERR_BAD_ARG;
  if (device < 0 || device >= 64) return DYNOBA_ERR_CUDA;
  StarContext& ctx = star_context(device);
  std::lock_guard<std::mutex> lock(ctx.mu);
  int rc = star_device_ready(device); if (rc) return rc;
  const size_t np = (size_t)n_intervals, nt = (size_t)offsets[n_intervals];
  DeviceBlock blk; PreintBatch S{};
  int* d_off; double *d_st, *d_ag, *d_bh;
  auto layout = [&]() {
    d_off = blk.take<int>(np + 1); d_st = blk.take<double>(nt); d_ag = blk.take<double>(6*nt);
    d_bh = bias_hat ? blk.take<double>(6*np) : nullptr;
    S.rec = blk.take<double>(PI_REC*np); S.cov = blk.take<double>(PI_COV*np); S.R = blk.take<double>(PI_COV*np);
    S.status = blk.take<int>(np);
  };
  layout();
  if (!blk.allocate(ctx)) { cudaGetLastError(); return DYNOBA_ERR_CUDA; }
  layout();
  cudaStream_t s = ctx.stream;
  cudaMemcpyAsync(d_off, offsets, 4*(np + 1), cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_st, stamps, 8*nt, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(d_ag, acc_gyr, 48*nt, cudaMemcpyHostToDevice, s);
  if (bias_hat) cudaMemcpyAsync(d_bh, bias_hat, 48*np, cudaMemcpyHostToDevice, s);
  S.off = d_off; S.stamps = d_st; S.acc_gyr = d_ag; S.bias = d_bh; S.n = n_intervals; S.prm = P;
  preint_kernel<<<(n_intervals + PI_WARPS - 1)/PI_WARPS, PI_WARPS*32, 0, s>>>(S);
  cudaMemcpyAsync(record, S.rec, 8*PI_REC*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(cov, S.cov, 8*PI_COV*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(sqrt_info, S.R, 8*PI_COV*np, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(status, S.status, 4*np, cudaMemcpyDeviceToHost, s);
  const cudaError_t e1 = cudaStreamSynchronize(s), e2 = cudaGetLastError();
  return (e1 == cudaSuccess && e2 == cudaSuccess) ? DYNOBA_OK : DYNOBA_ERR_CUDA;
}

}  // extern "C"
