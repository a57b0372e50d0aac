/* Plain-C consumer of libdynoba through include/dynoba.h (no ctypes, no C++): what a cgo / FFI binding would link.
 * Builds a small static graph -- two camera poses (prior + odometry) observing eight points with PoseToPoint factors --
 * runs the Levenberg-Marquardt call and checks that the error went down.
 * Exit code 0 = optimised on the GPU, 3 = no usable device (DYNOBA_ERR_CUDA from dynoba_create: there is no CPU path),
 * anything else = failure.  tests/test_host.py expects 3 on a box without a GPU, tests/test_gpu_parity.py expects 0. */
#include <stdio.h>
#include <stdlib.h>
#include "dynoba.h"

#define CK(call) do { int st_ = (call); if (st_ != DYNOBA_OK) { fprintf(stderr, "%s -> %s: %s\n", #call, dynoba_status_string(st_), dynoba_last_error(h)); return 1; } } while (0)

int main(void) {
  dynoba_handle h = NULL;
  int st = dynoba_create(0, &h);
  if (st == DYNOBA_ERR_CUDA) { printf("no usable sm_90 device: %s\n", dynoba_status_string(st)); return 3; }
  if (st != DYNOBA_OK) return 1;
  /* poses: R row-major | t.  pose 1 starts 0.3 m off its true place (1, 0, 0) */
  double poses[2][12] = { {1,0,0, 0,1,0, 0,0,1, 0,0,0}, {1,0,0, 0,1,0, 0,0,1, 1.3,0.1,-0.1} };
  double points[8][3], z[16][3]; int32_t idx[16][2];
  for (int i = 0; i < 8; i++) {
    const double p[3] = { -2.0 + 0.6*i, 0.5*((i % 3) - 1), 6.0 + (i % 4) };
    for (int k = 0; k < 3; k++) points[i][k] = p[k] + 0.05*((i + k) % 3 - 1);            /* perturbed initial value */
    for (int c = 0; c < 2; c++) {                                                          /* z = R^T (p - t), R = I */
      idx[2*i + c][0] = c; idx[2*i + c][1] = i;
      z[2*i + c][0] = p[0] - (c ? 1.0 : 0.0); z[2*i + c][1] = p[1]; z[2*i + c][2] = p[2];
    }
  }
  CK(dynoba_set_variables(h, DYNOBA_POSE6, 2, NULL, &poses[0][0]));
  CK(dynoba_set_variables(h, DYNOBA_POINT3, 8, NULL, &points[0][0]));
  const double sig_pt = 0.1; const double sig6[6] = {1e-3, 1e-3, 1e-3, 1e-3, 1e-3, 1e-3}, sig_od[6] = {0.05, 0.05, 0.05, 0.1, 0.1, 0.1};
  const double prior[12] = {1,0,0, 0,1,0, 0,0,1, 0,0,0}, odom[12] = {1,0,0, 0,1,0, 0,0,1, 1,0,0};
  const int32_t i0 = 0, i01[2] = {0, 1};
  CK(dynoba_add_factors(h, DYNOBA_POSE2POINT3, 16, &idx[0][0], &z[0][0], &sig_pt, 1, 1, 0.0, NULL));
  CK(dynoba_add_factors(h, DYNOBA_PRIOR6, 1, &i0, prior, sig6, 6, 1, 0.0, NULL));
  CK(dynoba_add_factors(h, DYNOBA_BETWEEN6, 1, i01, odom, sig_od, 6, 1, 0.0, NULL));
  double e0 = 0.0; CK(dynoba_error(h, &e0));
  dynoba_lm_params prm; dynoba_lm_default_params(&prm);
  dynoba_lm_stats stats;
  CK(dynoba_optimize(h, &prm, &stats));
  double out[2][12]; CK(dynoba_get_variables(h, DYNOBA_POSE6, 2, &out[0][0]));
  printf("chi2 %.6g -> %.6g in %d iterations (%d damped solves, %lld kernel launches); pose 1 t = (%.4f %.4f %.4f)\n",
         e0, stats.error_final, stats.iterations, stats.inner_iterations, (long long)stats.kernel_launches, out[1][9], out[1][10], out[1][11]);
  const int ok = stats.error_final < 1e-3*e0 && stats.kernel_launches > 0 && out[1][9] > 0.99 && out[1][9] < 1.01;
  dynoba_destroy(h);
  return ok ? 0 : 2;
}
