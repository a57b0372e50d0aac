// se3_host.cu -- the SE(3) maps of dynosam_b200/csrc/se3.cuh compiled for the host, so that tests/test_factor_cases.py can
// run them on a machine without a GPU (se3.cuh is __host__ __device__ throughout).  Poses are 12 doubles, R row-major | t.
#include "se3.cuh"

using namespace dynoba;

static Pose load(const double* p) {
  Pose P;
  for (int i = 0; i < 9; i++) P.R[i] = p[i];
  for (int i = 0; i < 3; i++) P.t[i] = p[9 + i];
  return P;
}
static void store(const Pose& P, double* p) {
  for (int i = 0; i < 9; i++) p[i] = P.R[i];
  for (int i = 0; i < 3; i++) p[9 + i] = P.t[i];
}

extern "C" {
void host_so3_expmap(const double* w, double* R) { so3_expmap(w, R); }
void host_so3_logmap(const double* R, double* w) { so3_logmap(R, w); }
void host_se3_expmap(const double* xi, double* p) { Pose P; se3_expmap(xi, P); store(P, p); }
void host_se3_logmap(const double* p, double* xi) { se3_logmap(load(p), xi); }
void host_se3_retract(const double* p, const double* xi, double* o) { Pose O; se3_retract(load(p), xi, O); store(O, o); }
void host_se3_local(const double* a, const double* b, double* xi) { se3_local(load(a), load(b), xi); }
void host_se3_adjoint(const double* p, double* Ad) { se3_adjoint(load(p), Ad); }
}
