// preint_host.cu -- the combined IMU preintegration of dynosam_b200/csrc/preint.cuh compiled for the host, so that
// tests/test_preint.py can run it on a machine without a GPU and tools/preint_bench.py can time it on one CPU thread.
// The interval loop is kernels_preint.cu's with one lane: the same functions in the same order.
#include "preint.cuh"

using namespace dynoba;

extern "C" {
// every interval of a batch, the arguments of dynoba_imu_preintegrate_batch (no validation: the tests pass valid input)
void host_preint_batch(const dynoba_imu_params* P, int n, const int* off, const double* stamps, const double* acc_gyr,
                       const double* bias_hat, double* rec, double* cov, double* R, int* status) {
  double S[PI_COV], Q[PI_COV], A[81], B[27], C[27], FT[2*PI_FR*PI_D];
  for (int p = 0; p < n; p++) {
    double bh[6];
    for (int k = 0; k < 6; k++) bh[k] = bias_hat ? bias_hat[6*p + k] : 0.0;
    for (int e = 0; e < PI_COV; e++) S[e] = 0.0;
    PreintState s; preint_reset(s);
    for (int i = off[p]; i < off[p + 1] - 1; i++) {
      const double dt = stamps[i + 1] - stamps[i];
      preint_step(*P, bh, acc_gyr + 6*i, acc_gyr + 6*i + 3, dt, s, A, B, C);
      preint_F(A, B, C, FT);
      preint_noise(*P, B, C, dt, Q);
      preint_cov_phase1(FT, S, FT + PI_FR*PI_D, 0, 1);
      preint_cov_phase2(FT, FT + PI_FR*PI_D, Q, S, 0, 1);
    }
    preint_record(s, bh, P->n_gravity, rec + PI_REC*p);
    status[p] = preint_sqrt_info(S, Q, FT);
    for (int e = 0; e < PI_COV; e++) { cov[PI_COV*p + e] = S[e]; R[PI_COV*p + e] = FT[e]; }
  }
}
// one step from a record-shaped state (the first 70 doubles of a record; its biasHat is the step's): the new record, A[81],
// B[27], C[27], F9[135] and Q[225]
void host_preint_step(const dynoba_imu_params* P, const double* z_in, const double* acc, const double* omega, double dt,
                      double* z_out, double* A, double* B, double* C, double* F9, double* Q) {
  PreintState s;
  for (int i = 0; i < 9; i++) { s.R[i] = z_in[i]; s.JRw[i] = z_in[22 + i]; s.JPa[i] = z_in[31 + i]; s.JPw[i] = z_in[40 + i];
                                s.JVa[i] = z_in[49 + i]; s.JVw[i] = z_in[58 + i]; }
  for (int k = 0; k < 3; k++) { s.p[k] = z_in[9 + k]; s.v[k] = z_in[12 + k]; }
  s.T = z_in[15];
  preint_step(*P, z_in + 16, acc, omega, dt, s, A, B, C);
  preint_F(A, B, C, F9);
  preint_noise(*P, B, C, dt, Q);
  preint_record(s, z_in + 16, z_in + 67, z_out);
}
// PreintegrationBase::predict: Xj[12] (R row-major | t), vj[3]
void host_preint_predict(const double* z, const double* Xi, const double* vi, const double* bi, double* Xj, double* vj) {
  Pose I, J;
  for (int i = 0; i < 9; i++) I.R[i] = Xi[i];
  for (int i = 0; i < 3; i++) I.t[i] = Xi[9 + i];
  preint_predict(z, I, vi, bi, J, vj);
  for (int i = 0; i < 9; i++) Xj[i] = J.R[i];
  for (int i = 0; i < 3; i++) Xj[9 + i] = J.t[i];
}
}
