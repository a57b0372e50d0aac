/* Plain-C consumer of the batched per-object refinement (dynoba_flow_pose_batch, include/dynoba.h) -- what a cgo / FFI
 * binding of the front end would link.  One object: the previous camera at the origin, the camera moved 0.5 m forward, six
 * features with exact measured flows, an initial pose 0.1 m off.
 * Exit code 0 = refined on the GPU (error went down), 3 = no usable device (DYNOBA_ERR_CUDA: there is no CPU path),
 * anything else = failure. */
#include <stdio.h>
#include "dynoba.h"

int main(void) {
  const int32_t off[2] = {0, 6};
  const double I12[12] = {1,0,0, 0,1,0, 0,0,1, 0,0,0}, guess[12] = {1,0,0, 0,1,0, 0,0,1, 0.05,0.0,0.4}, K5[5] = {700, 700, 0, 600, 180};
  double kp[6][2], depth[6], flow[6][2];
  for (int i = 0; i < 6; i++) {
    kp[i][0] = 300.0 + 100.0*i; kp[i][1] = 100.0 + 30.0*(i % 3); depth[i] = 8.0 + i;
    const double x = (kp[i][0] - K5[3])/K5[0]*depth[i], y = (kp[i][1] - K5[4])/K5[1]*depth[i], zc = depth[i] - 0.5;     /* in the moved camera */
    flow[i][0] = K5[0]*x/zc + K5[3] - kp[i][0]; flow[i][1] = K5[1]*y/zc + K5[4] - kp[i][1];
  }
  dynoba_flow_pose_params fp; dynoba_flow_pose_default_params(&fp);
  double pose_out[12], flow_out[6][2], eb = 0.0, ea = 0.0; uint8_t inl[6]; int32_t its = 0, inner = 0, rounds = 0;
  const int st = dynoba_flow_pose_batch(0, 1, off, guess, I12, K5, &kp[0][0], depth, &flow[0][0], &fp, pose_out, &flow_out[0][0], inl, &eb, &ea, &its, &inner, &rounds);
  if (st == DYNOBA_ERR_CUDA) { printf("no usable sm_90 device: %s\n", dynoba_status_string(st)); return 3; }
  if (st != DYNOBA_OK) { fprintf(stderr, "dynoba_flow_pose_batch -> %s\n", dynoba_status_string(st)); return 1; }
  printf("flow+pose: error %.6g -> %.6g in %d iterations, t_z %.4f\n", eb, ea, (int)its, pose_out[11]);
  dynoba_batch_release(0);
  return (ea <= eb && its >= 1) ? 0 : 2;
}
