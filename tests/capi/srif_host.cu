// srif_host.cu -- the object-motion filter step of dynosam_b200/csrc/srif.cuh compiled for the host, so that tests/test_srif.py
// can run it on a machine without a GPU and tools/srif_bench.py can time it on one CPU thread.  The object loop runs
// srif_object_seq, the sequential statement kernels_srif.cu parallelises.
#include <vector>
#include "srif.cuh"

using namespace dynoba;

extern "C" {
// every object of a batch, the arguments of dynoba_object_srif_batch (no validation: the tests pass valid input)
void host_srif_batch(int n_objects, const int* off, const int* mode, const int* pnp_status, const double* pose_prev,
                     const double* pose_cur, const double* calib6, const dynoba_object_srif_params* P, const double* state_in,
                     double* state_out, const double* stereo, const uint8_t* stereo_valid, const double* points_cam, double* m_L,
                     uint8_t* has_point, int* status, uint8_t* solved, double* motion_out, double* cov_out, double* errors,
                     double* before_reset, int* counts) {
  double Rinv[9]; srif_inv3(P->R_noise, Rinv);
  for (int o = 0; o < n_objects; o++) {
    const int i0 = off[o], n = off[o + 1] - i0;
    std::vector<double> lin(SRIF_LIN*(size_t)(n + 1)), e0(n + 1), rwe(n + 1);
    SrifObject ob{ mode[o], n, pnp_status[o], pose_prev + 12*o, pose_cur + 12*o, calib6 + 6*o, stereo + 6*(size_t)i0,
                   stereo_valid + 2*(size_t)i0, points_cam + 6*(size_t)i0, m_L + 3*(size_t)i0, has_point + i0 };
    SrifOut out;
    srif_object_seq(state_in + DYNOBA_SRIF_STATE*(size_t)o, state_out + DYNOBA_SRIF_STATE*(size_t)o, ob, *P, Rinv, lin.data(),
                    e0.data(), rwe.data(), out);
    status[o] = out.status; solved[o] = (uint8_t)out.solved;
    for (int e = 0; e < 36; e++) { motion_out[36*o + e] = out.motion[e]; cov_out[36*o + e] = out.cov[e]; }
    for (int e = 0; e < 12; e++) before_reset[12*o + e] = out.before[e];
    errors[2*o] = out.error; errors[2*o + 1] = out.rerror;
    counts[3*o] = out.n_new; counts[3*o + 1] = out.status == DYNOBA_SRIF_OK ? n - out.n_new : 0; counts[3*o + 2] = out.n_clipped;
  }
}
// the Huber weight of a residual y (e = sqrt(y^T Rinv y)): returns w, writes e and whether the weight was clipped
double host_srif_huber(const double* y, const double* Rinv, double k, double* e, int* clipped) {
  *e = srif_mahal(y, Rinv);
  bool c; const double w = srif_huber(*e, k, &c);
  *clipped = c;
  return w;
}
}
