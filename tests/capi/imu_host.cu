// imu_host.cu -- the CombinedImuFactor evaluation of dynosam_b200/csrc/imu.cuh compiled for the host, so that
// tests/test_imu_cases.py can run it on a machine without a GPU (imu.cuh and se3.cuh are __host__ __device__).
// Poses are 12 doubles, R row-major | t; the record is the 70 doubles of include/dynoba.h.
#include "imu.cuh"

using namespace dynoba;

static Pose load(const double* p) {
  Pose P;
  for (int i = 0; i < 9; i++) P.R[i] = p[i];
  for (int i = 0; i < 3; i++) P.t[i] = p[9 + i];
  return P;
}

extern "C" {
// r[15] and J[15 x 30] (row-major) of one factor
void host_imu_eval(const double* Xi, const double* vi, const double* Xj, const double* vj, const double* bi, const double* bj,
                   const double* z, double* rJ) {
  imu_eval(load(Xi), vi, load(Xj), vj, bi, bj, z, rJ, rJ + IMU_D);
}
// r[15] alone (the error sweep's path: J == nullptr)
void host_imu_residual(const double* Xi, const double* vi, const double* Xj, const double* vj, const double* bi, const double* bj,
                       const double* z, double* r) {
  imu_eval(load(Xi), vi, load(Xj), vj, bi, bj, z, r, nullptr);
}
void host_so3_jr(const double* x, double* J) { so3_jr(x, J); }
void host_so3_jr_inv(const double* x, double* J) { so3_jr_inv(x, J); }
}
