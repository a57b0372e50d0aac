// builder.cu -- SURVEY.md 8f-3: graph construction straight into the flat SoA blocks of the C ABI.
//
// The reference walks its Map (frames -> observed tracklets / objects) and allocates one heap factor per observation
// (Formulation<MAP>::updateStaticObservations / updateDynamicObservations, dynosam/include/dynosam/backend/
// Formulation-impl.hpp:552-897; the hybrid rules in src/backend/rgbd/HybridEstimator.cc:573-830), only for the solver to
// walk them again.  This builder takes the same information -- per frame: camera pose estimate, odometry, static and
// dynamic point observations, front-end object motions -- and applies the formulation's topology rules once, emitting the
// variable arrays and one homogeneous block per factor type, ready for dynoba_set_variables / dynoba_add_factors:
//   * camera chain: PriorFactor(X_first, sigma 1e-6) + BetweenFactor odometry (VisionImuBackendModule.hpp:168-243)
//   * static points: added once seen min_static_obs times, initial value X_k z of the first observation, one
//     PoseToPointFactor per observation (Formulation-impl.hpp:145-212)
//   * HYBRID: object key-frame e = first frame of a visibility segment (a new key-frame once the object was unseen for more
//     than keyframe_gap frames, HybridEstimator.cc:985-998); motion variable e_H_k per (object, frame); one m_L per tracklet
//     initialised by HybridObjectMotion::projectToObject3 at its first observation; HybridMotionFactor(X_k, e_H_k, m_L; z, L_e);
//     PriorFactor(H_e = I, 1e-6) at the key-frame (:744-746); three-motion HybridSmoothingFactor inside a segment (:800-802);
//     L_e = centroid of the key-frame's points with identity rotation unless given (:867-875).
//   * WCME (formulation 1; WorldMotionEstimator.cc:151-351): one point per (tracklet, frame) initialised X_k z, a PoseToPointFactor
//     per observation, LandmarkMotionTernaryFactor(m_prev, m_k, H_k) between consecutive observations of a tracklet, a motion
//     variable H_k per (object, frame that closes a pair) initialised with the front end's translation and IDENTITY rotation
//     (:297-303), BetweenFactor(H_k-1, H_k, I) smoothing between consecutive frames (:309-349).
//   * WCPE (formulation 2; WorldPoseEstimator.cc:89-315): the same points, LandmarkMotionPoseFactor(m_prev, m_k, L_prev, L_k), an
//     object pose L_k per (object, frame) initialised motion * L_k-1 when the front end gave a motion and L_k-1 exists, else the
//     centroid of the object's points at k with identity rotation (:205-232), LandmarkPoseSmoothingFactor over three consecutive
//     frames (:259-306); no prior on the object poses.
//   * IMU (dynoba_builder_set_imu; RegularBackendModule.cc:528-570, VisionImuBackendModule.hpp:114-290): when any frame has
//     a preintegrated measurement, every frame after the first must have one and frame ids must be consecutive.  Velocity
//     and bias variables V_k, b_k per frame; V_0 = 0, b_0 = 0 with PriorFactor<Vector3> (sigma 1e-5) and
//     PriorFactor<ConstantBias> (sigma 0.1 x3, 0.01 x3); for k >= 1 (X_k, V_k) = predict(X_k-1, V_k-1, b_k-1) (the
//     preintegrated measurement of frame k), b_k = b_k-1, CombinedImuFactor(X_k-1, V_k-1, X_k, V_k, b_k-1, b_k) in place of
//     the odometry BetweenFactor, and the predicted X_k stands for the front end's pose everywhere: as the initial value of
//     the camera pose and of every point (and key-frame centroid) initialised from frame k.  The first frame keeps its pose.
// Host code only (no kernel): it lives in libdynoba.so because its output is the library's input.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/dynoba.h"
#include "se3.cuh"
#include "preint.cuh"
#include "triangulate.cuh"

using namespace dynoba;

namespace {

struct Obs { int32_t frame; int64_t tracklet; int32_t object; double z[3]; };
struct Block { int type = 0; std::vector<int32_t> idx, aux; std::vector<double> meas, sigma; int sigma_dim = 1; bool bcast = true; double k = 0; bool has_aux = false;
               int64_t sigma_count = 1;       // 1: one sigma for the block; n: one per factor (COMBINED_IMU15's R)
               int64_t n() const { static const int ar[14] = {1, 2, 2, 2, 3, 3, 3, 4, 3, 3, 2, 1, 1, 6}; return (int64_t)idx.size()/ar[type]; } };
struct ImuMeas { double z[70]; double R[225]; };

Pose pose_from(const double* p) { Pose P; for (int i = 0; i < 9; i++) P.R[i] = p[i]; for (int i = 0; i < 3; i++) P.t[i] = p[9 + i]; return P; }
void pose_to(const Pose& P, double* p) { for (int i = 0; i < 9; i++) p[i] = P.R[i]; for (int i = 0; i < 3; i++) p[9 + i] = P.t[i]; }
Pose identity_pose() { Pose P; for (int i = 0; i < 9; i++) P.R[i] = (i % 4 == 0) ? 1.0 : 0.0; P.t[0] = P.t[1] = P.t[2] = 0.0; return P; }
uint64_t sym(char c, uint64_t j) { return ((uint64_t)(unsigned char)c << 56) | j; }
uint64_t labeled(char c, uint64_t label, uint64_t j) { return ((uint64_t)(unsigned char)c << 56) | (label << 48) | j; }
uint64_t cantor(uint64_t k1, uint64_t k2) { return (k1 + k2)*(k1 + k2 + 1)/2 + k2; }

}  // namespace

struct dynoba_builder {
  dynoba_builder_params prm; std::string err; bool finalized = false;
  std::map<int32_t, std::pair<Pose, bool>> frames;             // frame -> (camera pose estimate, has odometry)
  std::map<int32_t, Pose> odom;                                  // frame -> relative pose from the previous frame
  std::vector<Obs> stat, dyn;
  std::map<std::pair<int32_t, int32_t>, Pose> motion_init, keyframe_pose;    // (object, frame)
  std::map<int32_t, ImuMeas> imu;                                // frame -> preintegrated measurement from the previous frame
  // STEREO_PROJECTION static landmarks (dynoba_builder_set_static_stereo): (frame, tracklet, uL uR v) per observation
  bool stereo = false; double calib6[6] = {}; double sigma_px = 0; int stereo_device = -1;
  std::vector<Obs> stereo_obs;
  int64_t st_added = 0, st_failed[4] = {}, st_never = 0;
  // products
  std::vector<double> pose, point, aux; std::vector<int32_t> order; std::vector<uint64_t> pose_keys, point_keys;
  std::vector<double> vel, bias; std::vector<int32_t> nav_order; std::vector<uint64_t> vel_keys, bias_keys;
  std::vector<Block> blocks;
};

#define BARG(cond, msg) do { if (!(cond)) { if (b) b->err = msg; return DYNOBA_ERR_BAD_ARG; } } while (0)

extern "C" {

void dynoba_builder_default_params(dynoba_builder_params* p) {
  p->min_static_obs = 2; p->min_dynamic_obs = 3; p->keyframe_gap = 2;       // params: min_static_observations, min_dynamic_observations
  p->sigma_static = 0.2; p->sigma_dynamic = 0.2; p->huber_k = 1e-4;           // BackendDefinitions.cc:124-196 flag defaults
  const double od[6] = {0.02, 0.02, 0.02, 0.01, 0.01, 0.01}, sm[6] = {0.01, 0.01, 0.01, 0.1, 0.1, 0.1};
  for (int i = 0; i < 6; i++) { p->odometry_sigma[i] = od[i]; p->smoothing_sigma[i] = sm[i]; }
  p->prior_sigma = 1e-6;
  p->formulation = DYNOBA_FORMULATION_HYBRID; p->sigma_motion = 0.01;         // motion_ternary_factor_noise_sigma
  p->backtrack = 1;
}
int dynoba_builder_create(const dynoba_builder_params* p, dynoba_builder_handle* out) {
  if (!out) return DYNOBA_ERR_BAD_ARG;
  dynoba_builder* b = new dynoba_builder();
  if (p) b->prm = *p; else dynoba_builder_default_params(&b->prm);
  *out = b; return DYNOBA_OK;
}
int dynoba_builder_destroy(dynoba_builder_handle b) { if (!b) return DYNOBA_ERR_BAD_ARG; delete b; return DYNOBA_OK; }
const char* dynoba_builder_last_error(dynoba_builder_handle b) { return b ? b->err.c_str() : "null builder"; }

int dynoba_builder_add_frame(dynoba_builder_handle b, int32_t frame, const double* X, const double* odom_from_prev) {
  BARG(b && X && frame >= 0, "bad frame");
  b->frames[frame] = { pose_from(X), odom_from_prev != nullptr };
  if (odom_from_prev) b->odom[frame] = pose_from(odom_from_prev);
  b->finalized = false; return DYNOBA_OK;
}
int dynoba_builder_add_static(dynoba_builder_handle b, int32_t frame, int64_t n, const int64_t* tracklet, const double* z) {
  BARG(b && n >= 0 && (n == 0 || (tracklet && z)), "bad static observations");
  BARG(!b->stereo, "static landmarks use the stereo formulation: add them with dynoba_builder_add_static_stereo");
  for (int64_t i = 0; i < n; i++) b->stat.push_back(Obs{ frame, tracklet[i], 0, { z[3*i], z[3*i + 1], z[3*i + 2] } });
  b->finalized = false; return DYNOBA_OK;
}
int dynoba_builder_add_dynamic(dynoba_builder_handle b, int32_t frame, int64_t n, const int64_t* tracklet, const int32_t* object, const double* z) {
  BARG(b && n >= 0 && (n == 0 || (tracklet && object && z)), "bad dynamic observations");
  for (int64_t i = 0; i < n; i++) { BARG(object[i] > 0, "object ids start at 1 (0 is the background)"); b->dyn.push_back(Obs{ frame, tracklet[i], object[i], { z[3*i], z[3*i + 1], z[3*i + 2] } }); }
  b->finalized = false; return DYNOBA_OK;
}
int dynoba_builder_set_motion_init(dynoba_builder_handle b, int32_t object, int32_t frame, const double* H) {
  BARG(b && H, "null"); b->motion_init[{object, frame}] = pose_from(H); b->finalized = false; return DYNOBA_OK;
}
int dynoba_builder_set_keyframe_pose(dynoba_builder_handle b, int32_t object, int32_t keyframe, const double* L_e) {
  BARG(b && L_e, "null"); b->keyframe_pose[{object, keyframe}] = pose_from(L_e); b->finalized = false; return DYNOBA_OK;
}

int dynoba_builder_set_imu(dynoba_builder_handle b, int32_t frame, const double* record, const double* sqrt_info) {
  BARG(b && record && sqrt_info && frame >= 0, "bad IMU measurement");
  for (int i = 0; i < 70; i++) BARG(std::isfinite(record[i]), "IMU record not finite");
  BARG(record[15] > 0.0, "IMU record with deltaTij <= 0");
  for (int i = 0; i < 225; i++) BARG(std::isfinite(sqrt_info[i]), "IMU square-root information not finite");
  for (int i = 0; i < 15; i++) BARG(sqrt_info[16*i] > 0.0, "IMU square-root information with a non-positive diagonal");
  ImuMeas& m = b->imu[frame];
  std::copy(record, record + 70, m.z); std::copy(sqrt_info, sqrt_info + 225, m.R);
  b->finalized = false; return DYNOBA_OK;
}

int dynoba_builder_set_static_stereo(dynoba_builder_handle b, const double* calib6, double sigma_px, int device) {
  BARG(b && calib6, "null");
  BARG(b->stat.empty(), "point-to-point static observations were added already");
  for (int i = 0; i < 6; i++) BARG(std::isfinite(calib6[i]), "calibration not finite");
  BARG(calib6[0] > 0.0 && calib6[1] > 0.0 && calib6[5] > 0.0, "fx, fy and the baseline must be positive");
  BARG(std::isfinite(sigma_px) && sigma_px > 0.0, "sigma_px must be positive and finite");
  b->stereo = true; std::copy(calib6, calib6 + 6, b->calib6); b->sigma_px = sigma_px; b->stereo_device = device;
  b->finalized = false; return DYNOBA_OK;
}
int dynoba_builder_add_static_stereo(dynoba_builder_handle b, int32_t frame, int64_t n, const int64_t* tracklet, const double* stereo) {
  BARG(b && n >= 0 && (n == 0 || (tracklet && stereo)), "bad static stereo observations");
  BARG(b->stereo, "select the stereo formulation first (dynoba_builder_set_static_stereo)");
  for (int64_t i = 0; i < n; i++)
    BARG(std::isfinite(stereo[3*i]) && std::isfinite(stereo[3*i + 2]) && (std::isfinite(stereo[3*i + 1]) || std::isnan(stereo[3*i + 1])),
         "a stereo measurement needs finite uL and v, and a finite or NaN uR");
  for (int64_t i = 0; i < n; i++) b->stereo_obs.push_back(Obs{ frame, tracklet[i], 0, { stereo[3*i], stereo[3*i + 1], stereo[3*i + 2] } });
  b->finalized = false; return DYNOBA_OK;
}
int dynoba_builder_static_stereo_stats(dynoba_builder_handle b, int64_t* added, int64_t* failed, int64_t* never_added) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  if (added) *added = b->st_added;
  if (failed) std::copy(b->st_failed, b->st_failed + 4, failed);
  if (never_added) *never_added = b->st_never;
  return DYNOBA_OK;
}

// STEREO_PROJECTION static landmarks (Formulation-impl.hpp:258-411): attempts in rounds by observation index, one batched
// triangulation per round (dynoba_triangulate_batch on stereo_device, or the host build of triangulate.cuh), then the
// landmarks, their initial values and the STEREO3 block
static int stereo_landmarks(dynoba_builder* b, const std::map<int32_t, int32_t>& cam_index) {
  b->st_added = b->st_never = 0; std::fill(b->st_failed, b->st_failed + 4, 0);
  auto by_frame = [](const Obs& a, const Obs& c) { return a.frame < c.frame; };
  std::stable_sort(b->stereo_obs.begin(), b->stereo_obs.end(), by_frame);
  std::map<int64_t, size_t> slot; std::vector<int64_t> tid; std::vector<std::vector<size_t>> tracks;   // first-appearance order
  size_t longest = 0;
  for (size_t i = 0; i < b->stereo_obs.size(); i++) {
    const Obs& o = b->stereo_obs[i];
    BARG(cam_index.count(o.frame), "static observation in an unknown frame");
    auto it = slot.find(o.tracklet);
    if (it == slot.end()) { it = slot.emplace(o.tracklet, tracks.size()).first; tid.push_back(o.tracklet); tracks.emplace_back(); }
    auto& t = tracks[it->second];
    BARG(t.empty() || b->stereo_obs[t.back()].frame < o.frame, "a static tracklet is observed twice in one frame");
    t.push_back(i); longest = std::max(longest, t.size());
  }
  const double* K = b->calib6; const double base = K[5];
  auto disparity_ok = [](const Obs& o) { return o.z[0] - o.z[1] > 0.5; };      // false for a NaN uR
  std::vector<int> added_at(tracks.size(), -1); std::vector<double> point(3*tracks.size());
  std::vector<int32_t> off, st; std::vector<double> poses, kp, cal, pt; std::vector<size_t> which;
  for (size_t r = 0; r < longest; r++) {
    off.assign(1, 0); poses.clear(); kp.clear(); cal.clear(); which.clear();
    for (size_t ti = 0; ti < tracks.size(); ti++) {
      if (added_at[ti] >= 0 || tracks[ti].size() <= r) continue;
      for (size_t j = 0; j <= r; j++) {
        const Obs& o = b->stereo_obs[tracks[ti][j]];
        const Pose& X = b->frames.at(o.frame).first;                  // hasInitialSensorPose: the add_frame pose
        double p[12]; pose_to(X, p);
        poses.insert(poses.end(), p, p + 12); kp.push_back(o.z[0]); kp.push_back(o.z[2]);
        if (!std::isnan(o.z[1])) {                                     // right camera X * (I, (b, 0, 0))
          for (int k = 0; k < 3; k++) p[9 + k] = X.t[k] + base*X.R[3*k];
          poses.insert(poses.end(), p, p + 12); kp.push_back(o.z[1]); kp.push_back(o.z[2]);
        }
      }
      off.push_back((int32_t)(poses.size()/12)); cal.insert(cal.end(), K, K + 5); which.push_back(ti);
    }
    if (which.empty()) continue;
    const int32_t np = (int32_t)which.size();
    st.assign(np, 0); pt.assign(3*(size_t)np, 0.0);
    if (b->stereo_device >= 0) {
      const int rc = dynoba_triangulate_batch(b->stereo_device, np, off.data(), poses.data(), kp.data(), cal.data(), 1.0, 3.0,
                                              pt.data(), st.data(), nullptr, nullptr);
      if (rc) { b->err = "dynoba_triangulate_batch failed"; return rc; }
    } else {
      std::vector<double> A;
      for (int32_t p = 0; p < np; p++) {
        const int m = off[p + 1] - off[p]; A.resize(8*(size_t)m);
        TriHostLanes lanes; TriOut o;
        tri_solve(m, poses.data() + 12*(size_t)off[p], kp.data() + 2*(size_t)off[p], K, 1.0, 3.0, A.data(), lanes, o);
        st[p] = o.status; for (int k = 0; k < 3; k++) pt[3*(size_t)p + k] = o.point[k];
      }
    }
    for (int32_t p = 0; p < np; p++) {
      const size_t ti = which[p];
      if (st[p] != DYNOBA_TRI_OK) { b->st_failed[st[p]]++; continue; }
      int good = 0;
      for (size_t j = 0; j <= r; j++) good += disparity_ok(b->stereo_obs[tracks[ti][j]]);
      if (good < 2) { b->st_failed[DYNOBA_TRI_OK]++; continue; }
      added_at[ti] = (int)r; for (int k = 0; k < 3; k++) point[3*ti + k] = pt[3*(size_t)p + k];
    }
  }
  Block blk; blk.type = DYNOBA_STEREO3; blk.sigma.assign(3, b->sigma_px); blk.sigma_dim = 3; blk.k = b->prm.huber_k;
  for (size_t ti = 0; ti < tracks.size(); ti++) {
    if (added_at[ti] < 0) { b->st_never++; continue; }
    b->st_added++;
    const int32_t pi = (int32_t)(b->point.size()/3);
    b->point.insert(b->point.end(), &point[3*ti], &point[3*ti] + 3); b->point_keys.push_back(sym('l', (uint64_t)tid[ti]));
    for (size_t j = 0; j < tracks[ti].size(); j++) {
      const Obs& o = b->stereo_obs[tracks[ti][j]];
      // at the attempt that added it: the observations with disparity > 0.5; afterwards every one with a right key-point
      if ((int)j <= added_at[ti] ? !disparity_ok(o) : std::isnan(o.z[1])) continue;
      blk.idx.push_back(cam_index.at(o.frame)); blk.idx.push_back(pi); blk.meas.insert(blk.meas.end(), o.z, o.z + 3);
    }
  }
  if (blk.n()) b->blocks.push_back(std::move(blk));
  return DYNOBA_OK;
}

int dynoba_builder_finalize(dynoba_builder_handle b) {
  BARG(b, "null builder");
  if (b->finalized) return DYNOBA_OK;
  const dynoba_builder_params& P = b->prm;
  b->pose.clear(); b->point.clear(); b->aux.clear(); b->order.clear(); b->pose_keys.clear(); b->point_keys.clear(); b->blocks.clear();
  b->vel.clear(); b->bias.clear(); b->nav_order.clear(); b->vel_keys.clear(); b->bias_keys.clear();
  BARG(!b->frames.empty(), "no frames");
  // ---- initial camera poses: the front end's, or with IMU the prediction chain from the first frame
  std::map<int32_t, Pose> X0;
  for (auto& kv : b->frames) X0[kv.first] = kv.second.first;
  const bool imu = !b->imu.empty();
  if (imu) {
    for (auto& kv : b->imu) BARG(b->frames.count(kv.first), "IMU measurement on a frame that was not added");
    int32_t prev = -1; Pose X; double v[3] = {0, 0, 0}; const double bz[6] = {0, 0, 0, 0, 0, 0};
    for (auto& kv : b->frames) {
      const int32_t f = kv.first;
      if (prev < 0) X = kv.second.first;
      else {
        BARG(f == prev + 1, "frame ids are not consecutive while IMU is present");
        auto it = b->imu.find(f);
        BARG(it != b->imu.end(), "IMU measurements on some frames but not on others");
        Pose Xn; double vn[3];
        preint_predict(it->second.z, X, v, bz, Xn, vn);             // b_k-1 = b_0 = 0
        X = Xn; for (int a = 0; a < 3; a++) v[a] = vn[a];
        X0[f] = X;
      }
      b->vel.insert(b->vel.end(), v, v + 3); b->bias.insert(b->bias.end(), bz, bz + 6);
      b->nav_order.push_back(f); b->vel_keys.push_back(sym('V', (uint64_t)f)); b->bias_keys.push_back(sym('b', (uint64_t)f));
      prev = f;
    }
  }
  // ---- camera poses, in frame order
  std::map<int32_t, int32_t> cam_index;
  for (auto& kv : b->frames) {
    cam_index[kv.first] = (int32_t)cam_index.size();
    double p[12]; pose_to(X0[kv.first], p); b->pose.insert(b->pose.end(), p, p + 12);
    b->order.push_back(kv.first); b->pose_keys.push_back(sym('X', (uint64_t)kv.first));
  }
  auto cam = [&](int32_t f) -> int32_t { auto it = cam_index.find(f); return it == cam_index.end() ? -1 : it->second; };
  // ---- static landmarks: tracklets in order of first appearance (frame-major, insertion order inside a frame)
  auto by_frame = [](const Obs& a, const Obs& c) { return a.frame < c.frame; };
  std::stable_sort(b->stat.begin(), b->stat.end(), by_frame);
  std::stable_sort(b->dyn.begin(), b->dyn.end(), by_frame);
  // ---- which observations enter the graph.  A tracklet needs min_*_obs observations.  With backtrack (the batch graph of
  // SURVEY 8d; UpdateObservationParams::do_backtrack = true, ParallelHybridBackendModule.cc:427) all of them are added; without
  // (RegularBackendModule.cc:139,197) the tracklet enters at the frame its count reaches the minimum and only what that update
  // adds is kept: static -- that frame's observation on (Formulation-impl.hpp:194-199); dynamic -- the pair (previous, that
  // frame) on (:703-720), i.e. the first min_dynamic_obs - 2 observations never enter.
  std::vector<Obs> stat, dyn;
  {
    std::map<std::pair<int32_t, int64_t>, int> count, seen;
    for (auto& o : b->stat) count[{0, o.tracklet}]++;
    for (auto& o : b->dyn) count[{o.object, o.tracklet}]++;
    const int min_dyn = P.formulation == DYNOBA_FORMULATION_HYBRID ? P.min_dynamic_obs : std::max(P.min_dynamic_obs, 2);   // a motion factor needs a pair
    const int start_s = P.backtrack ? 0 : std::max(P.min_static_obs - 1, 0), start_d = P.backtrack ? 0 : std::max(min_dyn - 2, 0);
    for (auto& o : b->stat) if (count[{0, o.tracklet}] >= P.min_static_obs && seen[{0, o.tracklet}]++ >= start_s) stat.push_back(o);
    for (auto& o : b->dyn) if (count[{o.object, o.tracklet}] >= min_dyn && seen[{o.object, o.tracklet}]++ >= start_d) dyn.push_back(o);
  }
  // ---- static landmarks: tracklets in order of first appearance (frame-major, insertion order inside a frame)
  if (b->stereo) { int rc = stereo_landmarks(b, cam_index); if (rc) return rc; }
  else {
    std::map<int64_t, std::vector<size_t>> tracks; std::vector<int64_t> first_seen;
    for (size_t i = 0; i < stat.size(); i++) { BARG(cam(stat[i].frame) >= 0, "static observation in an unknown frame");
      auto& t = tracks[stat[i].tracklet]; if (t.empty()) first_seen.push_back(stat[i].tracklet); t.push_back(i); }
    Block blk; blk.type = DYNOBA_POSE2POINT3; blk.sigma = { P.sigma_static }; blk.k = P.huber_k;
    for (int64_t tid : first_seen) {
      auto& t = tracks[tid];
      const int32_t pi = (int32_t)(b->point.size()/3);
      const Obs& o0 = stat[t[0]];
      double w[3]; se3_transform_from(X0[o0.frame], o0.z, w);          // initial value: X_k z of the first observation that enters
      b->point.insert(b->point.end(), w, w + 3); b->point_keys.push_back(sym('l', (uint64_t)tid));
      for (size_t i : t) { const Obs& o = stat[i]; blk.idx.push_back(cam(o.frame)); blk.idx.push_back(pi); blk.meas.insert(blk.meas.end(), o.z, o.z + 3); }
    }
    if (blk.n()) b->blocks.push_back(std::move(blk));
  }
  if (P.formulation != DYNOBA_FORMULATION_HYBRID) {
    // ---- world-centric formulations: a point per (tracklet, observation), chained by motion factors
    BARG(P.formulation == DYNOBA_FORMULATION_WCME || P.formulation == DYNOBA_FORMULATION_WCPE, "unknown formulation");
    const bool wcpe = P.formulation == DYNOBA_FORMULATION_WCPE;
    const int32_t n_cam = (int32_t)cam_index.size();
    std::map<std::pair<int32_t, int64_t>, std::vector<size_t>> tracks; std::vector<std::pair<int32_t, int64_t>> first_seen;
    for (size_t i = 0; i < dyn.size(); i++) { BARG(cam(dyn[i].frame) >= 0, "dynamic observation in an unknown frame");
      auto key = std::make_pair(dyn[i].object, dyn[i].tracklet);
      auto& t = tracks[key]; if (t.empty()) first_seen.push_back(key); t.push_back(i); }
    std::stable_sort(first_seen.begin(), first_seen.end(), [](const std::pair<int32_t, int64_t>& a, const std::pair<int32_t, int64_t>& c) { return a.first < c.first; });
    // (object, frame) -> pose-like variable: WCME the frame that closes a pair, WCPE every observed frame of a kept tracklet
    std::map<std::pair<int32_t, int32_t>, int32_t> var_index;
    std::map<std::pair<int32_t, int32_t>, std::pair<std::array<double, 3>, int>> centroid;     // world points of the kept tracklets
    for (auto& key : first_seen) {
      auto& t = tracks[key];
      for (size_t k = 0; k < t.size(); k++) { const Obs& o = dyn[t[k]];
        if (k > 0) BARG(o.frame > dyn[t[k-1]].frame, "a tracklet is observed twice in one frame");
        if (wcpe || k > 0) var_index[{o.object, o.frame}] = -1;
        double w[3]; se3_transform_from(X0[o.frame], o.z, w);
        auto& c = centroid[{o.object, o.frame}]; for (int a = 0; a < 3; a++) c.first[a] += w[a]; c.second++; }
    }
    for (auto& kv : var_index) {                                       // std::map order: object-major, frames ascending
      const int32_t obj = kv.first.first, fr = kv.first.second;
      kv.second = (int32_t)(b->pose.size()/12);
      Pose V = identity_pose();
      auto mi = b->motion_init.find({obj, fr});
      if (!wcpe) { if (mi != b->motion_init.end()) for (int a = 0; a < 3; a++) V.t[a] = mi->second.t[a]; }
      else {
        auto given = b->keyframe_pose.find({obj, fr}); auto prev = var_index.find({obj, fr - 1});
        if (given != b->keyframe_pose.end()) V = given->second;
        else if (mi != b->motion_init.end() && prev != var_index.end() && prev->second >= 0) se3_compose(mi->second, pose_from(&b->pose[(size_t)12*prev->second]), V);
        else { auto& c = centroid[{obj, fr}]; for (int a = 0; a < 3; a++) V.t[a] = c.first[a]/std::max(c.second, 1); }
      }
      double p[12]; pose_to(V, p); b->pose.insert(b->pose.end(), p, p + 12);
      b->order.push_back(fr); b->pose_keys.push_back(labeled(wcpe ? 'L' : 'H', (uint64_t)('0' + obj), (uint64_t)fr));
    }
    Block ptp; ptp.type = DYNOBA_POSE2POINT3; ptp.sigma = { P.sigma_dynamic }; ptp.k = P.huber_k;
    Block mot; mot.type = wcpe ? DYNOBA_MOTIONPOSE3 : DYNOBA_TERNARY3; mot.sigma = { P.sigma_motion }; mot.k = P.huber_k;
    for (auto& key : first_seen) {
      auto& t = tracks[key];
      for (size_t k = 0; k < t.size(); k++) { const Obs& o = dyn[t[k]];
        const int32_t pi = (int32_t)(b->point.size()/3);
        double w[3]; se3_transform_from(X0[o.frame], o.z, w);                 // X_k z (dynamicPointUpdateCallback)
        b->point.insert(b->point.end(), w, w + 3); b->point_keys.push_back(sym('m', cantor((uint64_t)o.tracklet, (uint64_t)o.frame)));
        ptp.idx.push_back(cam(o.frame)); ptp.idx.push_back(pi); ptp.meas.insert(ptp.meas.end(), o.z, o.z + 3);
        if (k > 0) { mot.idx.push_back(pi - 1); mot.idx.push_back(pi);
          if (wcpe) mot.idx.push_back(var_index[{o.object, dyn[t[k-1]].frame}]);
          mot.idx.push_back(var_index[{o.object, o.frame}]); }
      }
    }
    if (ptp.n()) b->blocks.push_back(std::move(ptp));
    if (mot.n()) b->blocks.push_back(std::move(mot));
    Block sm; sm.type = wcpe ? DYNOBA_SMOOTH_POSE6 : DYNOBA_BETWEEN6; sm.sigma.assign(P.smoothing_sigma, P.smoothing_sigma + 6); sm.sigma_dim = 6;
    const Pose I = identity_pose(); double pi12[12]; pose_to(I, pi12);
    for (auto& kv : var_index) {
      const int32_t obj = kv.first.first, fr = kv.first.second;
      auto p1 = var_index.find({obj, fr - 1}), p2 = var_index.find({obj, fr - 2});
      if (!wcpe) { if (p1 != var_index.end()) { sm.idx.push_back(p1->second); sm.idx.push_back(kv.second); sm.meas.insert(sm.meas.end(), pi12, pi12 + 12); } }
      else if (p1 != var_index.end() && p2 != var_index.end()) { sm.idx.push_back(p2->second); sm.idx.push_back(p1->second); sm.idx.push_back(kv.second); }
    }
    if (sm.n()) b->blocks.push_back(std::move(sm));
  } else {
  // ---- dynamic: objects -> visibility segments (key-frames) -> motion variables
  const int32_t n_cam = (int32_t)cam_index.size();
  std::map<int32_t, std::vector<int32_t>> obj_frames;                  // object -> sorted frames it is observed in
  for (auto& o : dyn) { BARG(cam(o.frame) >= 0, "dynamic observation in an unknown frame"); obj_frames[o.object].push_back(o.frame); }
  struct Seg { int32_t object, keyframe, aux; };
  std::map<std::pair<int32_t, int32_t>, int32_t> motion_index;         // (object, frame) -> pose index
  std::map<std::pair<int32_t, int32_t>, int32_t> seg_of;               // (object, frame) -> segment
  std::vector<Seg> segs; std::vector<std::vector<int32_t>> seg_motions;
  for (auto& kv : obj_frames) {
    auto& fr = kv.second; std::sort(fr.begin(), fr.end()); fr.erase(std::unique(fr.begin(), fr.end()), fr.end());
    for (size_t i = 0; i < fr.size(); i++) {
      if (i == 0 || fr[i] - fr[i-1] > P.keyframe_gap) { segs.push_back(Seg{ kv.first, fr[i], -1 }); seg_motions.emplace_back(); }
      const int32_t pi = n_cam + (int32_t)motion_index.size();
      motion_index[{kv.first, fr[i]}] = pi; seg_of[{kv.first, fr[i]}] = (int32_t)segs.size() - 1; seg_motions.back().push_back(pi);
      Pose H = identity_pose();                                        // key-frame motion starts at its prior; others at the front end's estimate
      if (fr[i] != segs.back().keyframe) { auto it = b->motion_init.find({kv.first, fr[i]}); if (it != b->motion_init.end()) H = it->second; }
      double p[12]; pose_to(H, p); b->pose.insert(b->pose.end(), p, p + 12);
      b->order.push_back(fr[i]); b->pose_keys.push_back(labeled('H', (uint64_t)('0' + kv.first), (uint64_t)fr[i]));
    }
  }
  // ---- dynamic tracklets (object-major, then first appearance), key-frame poses, hybrid factors
  {
    std::map<std::pair<int32_t, int64_t>, std::vector<size_t>> tracks; std::vector<std::pair<int32_t, int64_t>> first_seen;
    for (size_t i = 0; i < dyn.size(); i++) { auto key = std::make_pair(dyn[i].object, dyn[i].tracklet);
      auto& t = tracks[key]; if (t.empty()) first_seen.push_back(key); t.push_back(i); }
    std::stable_sort(first_seen.begin(), first_seen.end(), [](const std::pair<int32_t, int64_t>& a, const std::pair<int32_t, int64_t>& c) { return a.first < c.first; });
    // L_e per segment: given, or the centroid of the key-frame's world points with identity rotation
    for (size_t s = 0; s < segs.size(); s++) {
      Pose Le; auto it = b->keyframe_pose.find({segs[s].object, segs[s].keyframe});
      if (it != b->keyframe_pose.end()) Le = it->second;
      else {
        Le = identity_pose(); double c[3] = {0, 0, 0}; int cnt = 0;
        for (auto& o : dyn) if (o.object == segs[s].object && o.frame == segs[s].keyframe) { double w[3]; se3_transform_from(X0[o.frame], o.z, w); for (int k = 0; k < 3; k++) c[k] += w[k]; cnt++; }
        for (int k = 0; k < 3; k++) Le.t[k] = cnt ? c[k]/cnt : 0.0;
      }
      segs[s].aux = (int32_t)(b->aux.size()/12); double p[12]; pose_to(Le, p); b->aux.insert(b->aux.end(), p, p + 12);
    }
    Block blk; blk.type = DYNOBA_HYBRID3; blk.sigma = { P.sigma_dynamic }; blk.k = P.huber_k; blk.has_aux = true;
    for (auto& key : first_seen) {
      auto& t = tracks[key];
      const Obs& o0 = dyn[t[0]];
      const int32_t s0 = seg_of[{o0.object, o0.frame}];
      // every observation of a tracklet refers to the key-frame of its FIRST observation (a tracklet does not outlive a segment)
      bool one_segment = true; for (size_t i : t) one_segment = one_segment && seg_of[{dyn[i].object, dyn[i].frame}] == s0;
      BARG(one_segment, "a dynamic tracklet spans two key-frame segments of its object");
      const int32_t pi = (int32_t)(b->point.size()/3);
      // m_L = L_e^-1 (e_H_k)^-1 X_k z at the first observation (HybridObjectMotion::projectToObject3)
      const Pose Le = pose_from(&b->aux[(size_t)12*segs[s0].aux]); const Pose E = pose_from(&b->pose[(size_t)12*motion_index[{o0.object, o0.frame}]]);
      double w[3], q[3], m[3]; se3_transform_from(X0[o0.frame], o0.z, w); se3_transform_to(E, w, q); se3_transform_to(Le, q, m);
      b->point.insert(b->point.end(), m, m + 3); b->point_keys.push_back(sym('m', cantor((uint64_t)key.second, 0)));
      for (size_t i : t) { const Obs& o = dyn[i];
        blk.idx.push_back(cam(o.frame)); blk.idx.push_back(motion_index[{o.object, o.frame}]); blk.idx.push_back(pi);
        blk.meas.insert(blk.meas.end(), o.z, o.z + 3); blk.aux.push_back(segs[s0].aux); }
    }
    if (blk.n()) b->blocks.push_back(std::move(blk));
    // priors on the key-frame motions, three-motion smoothing inside a segment
    Block pr; pr.type = DYNOBA_PRIOR6; pr.sigma.assign(6, P.prior_sigma); pr.sigma_dim = 6;
    Block sm; sm.type = DYNOBA_SMOOTH_HYBRID6; sm.sigma.assign(P.smoothing_sigma, P.smoothing_sigma + 6); sm.sigma_dim = 6; sm.has_aux = true;
    const Pose I = identity_pose(); double pi12[12]; pose_to(I, pi12);
    for (size_t s = 0; s < segs.size(); s++) {
      pr.idx.push_back(seg_motions[s][0]); pr.meas.insert(pr.meas.end(), pi12, pi12 + 12);
      for (size_t i = 0; i + 2 < seg_motions[s].size(); i++) { sm.idx.push_back(seg_motions[s][i]); sm.idx.push_back(seg_motions[s][i + 1]); sm.idx.push_back(seg_motions[s][i + 2]); sm.aux.push_back(segs[s].aux); }
    }
    if (pr.n()) b->blocks.push_back(std::move(pr));
    if (sm.n()) b->blocks.push_back(std::move(sm));
  }
  }
  // ---- camera chain
  {
    Block pr; pr.type = DYNOBA_PRIOR6; pr.sigma.assign(6, P.prior_sigma); pr.sigma_dim = 6;
    pr.idx.push_back(0); pr.meas.insert(pr.meas.end(), b->pose.begin(), b->pose.begin() + 12);      // prior = the first frame's pose
    b->blocks.push_back(std::move(pr));
    Block od; od.type = DYNOBA_BETWEEN6; od.sigma.assign(P.odometry_sigma, P.odometry_sigma + 6); od.sigma_dim = 6;
    int32_t prev = -1;
    for (auto& kv : b->frames) {
      if (prev >= 0 && kv.second.second && !imu) { od.idx.push_back(cam(prev)); od.idx.push_back(cam(kv.first)); double p[12]; pose_to(b->odom[kv.first], p); od.meas.insert(od.meas.end(), p, p + 12); }
      prev = kv.first;
    }
    if (od.n()) b->blocks.push_back(std::move(od));
  }
  // ---- IMU chain: priors on V_0, b_0 and one CombinedImuFactor per later frame (velocity / bias index = camera index)
  if (imu) {
    Block pv; pv.type = DYNOBA_PRIOR_VEL3; pv.sigma = { 1e-5 }; pv.idx.push_back(0); pv.meas.assign(3, 0.0);
    Block pb; pb.type = DYNOBA_PRIOR_BIAS6; pb.sigma = { 0.1, 0.1, 0.1, 0.01, 0.01, 0.01 }; pb.sigma_dim = 6; pb.idx.push_back(0); pb.meas.assign(6, 0.0);
    b->blocks.push_back(std::move(pv)); b->blocks.push_back(std::move(pb));
    Block im; im.type = DYNOBA_COMBINED_IMU15; im.sigma_dim = 225;
    int32_t k = 0;
    for (auto& kv : b->frames) {
      if (k > 0) {
        const int32_t q[6] = { k - 1, k - 1, k, k, k - 1, k };
        const ImuMeas& m = b->imu[kv.first];
        im.idx.insert(im.idx.end(), q, q + 6); im.meas.insert(im.meas.end(), m.z, m.z + 70); im.sigma.insert(im.sigma.end(), m.R, m.R + 225);
      }
      k++;
    }
    im.sigma_count = im.n();
    if (im.n()) b->blocks.push_back(std::move(im));
  }
  b->finalized = true;
  return DYNOBA_OK;
}

int dynoba_builder_counts(dynoba_builder_handle b, int64_t* n_pose, int64_t* n_point, int64_t* n_aux, int32_t* n_blocks) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  if (n_pose) *n_pose = (int64_t)b->pose.size()/12; if (n_point) *n_point = (int64_t)b->point.size()/3; if (n_aux) *n_aux = (int64_t)b->aux.size()/12;
  if (n_blocks) *n_blocks = (int32_t)b->blocks.size();
  return DYNOBA_OK;
}
int dynoba_builder_get_variables(dynoba_builder_handle b, double* pose, double* point, double* aux, int32_t* pose_order, uint64_t* pose_keys, uint64_t* point_keys) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  if (pose) std::copy(b->pose.begin(), b->pose.end(), pose); if (point) std::copy(b->point.begin(), b->point.end(), point);
  if (aux) std::copy(b->aux.begin(), b->aux.end(), aux); if (pose_order) std::copy(b->order.begin(), b->order.end(), pose_order);
  if (pose_keys) std::copy(b->pose_keys.begin(), b->pose_keys.end(), pose_keys); if (point_keys) std::copy(b->point_keys.begin(), b->point_keys.end(), point_keys);
  return DYNOBA_OK;
}
int dynoba_builder_block_info(dynoba_builder_handle b, int32_t bi, int32_t* type, int64_t* n, int32_t* sigma_dim, int64_t* sigma_count, double* robust_k, int32_t* has_aux) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  BARG(bi >= 0 && bi < (int32_t)b->blocks.size(), "bad block index");
  const Block& k = b->blocks[bi];
  if (type) *type = k.type; if (n) *n = k.n(); if (sigma_dim) *sigma_dim = k.sigma_dim; if (sigma_count) *sigma_count = k.sigma_count;
  if (robust_k) *robust_k = k.k; if (has_aux) *has_aux = k.has_aux ? 1 : 0;
  return DYNOBA_OK;
}
int dynoba_builder_get_block(dynoba_builder_handle b, int32_t bi, int32_t* idx, double* meas, double* sigma, int32_t* aux) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  BARG(bi >= 0 && bi < (int32_t)b->blocks.size(), "bad block index");
  const Block& k = b->blocks[bi];
  if (idx) std::copy(k.idx.begin(), k.idx.end(), idx); if (meas) std::copy(k.meas.begin(), k.meas.end(), meas);
  if (sigma) std::copy(k.sigma.begin(), k.sigma.end(), sigma); if (aux) std::copy(k.aux.begin(), k.aux.end(), aux);
  return DYNOBA_OK;
}
// hands everything to a solver handle: the calls a flattening adapter would make, without the factor objects in between
int dynoba_builder_emit(dynoba_builder_handle b, dynoba_handle h) {
  BARG(b && h, "null"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  if ((rc = dynoba_set_variables(h, DYNOBA_POSE6, (int64_t)b->pose.size()/12, b->pose_keys.data(), b->pose.data()))) return rc;
  if ((rc = dynoba_set_variables(h, DYNOBA_POINT3, (int64_t)b->point.size()/3, b->point_keys.data(), b->point.data()))) return rc;
  if (!b->aux.empty() && (rc = dynoba_set_aux_poses(h, (int64_t)b->aux.size()/12, b->aux.data()))) return rc;
  if (b->stereo && (rc = dynoba_set_calibration(h, b->calib6))) return rc;
  const int64_t nn = (int64_t)b->nav_order.size();
  if (nn) {
    if ((rc = dynoba_set_variables(h, DYNOBA_VEL3, nn, b->vel_keys.data(), b->vel.data()))) return rc;
    if ((rc = dynoba_set_variables(h, DYNOBA_BIAS6, nn, b->bias_keys.data(), b->bias.data()))) return rc;
  }
  for (auto& k : b->blocks)
    if ((rc = dynoba_add_factors(h, k.type, k.n(), k.idx.data(), k.meas.empty() ? nullptr : k.meas.data(), k.sigma.data(), k.sigma_dim, k.sigma_count, k.k, k.has_aux ? k.aux.data() : nullptr))) return rc;
  if ((rc = dynoba_set_pose_order(h, (int64_t)b->order.size(), b->order.data()))) return rc;
  if (nn) {
    if ((rc = dynoba_set_variable_order(h, DYNOBA_VEL3, nn, b->nav_order.data()))) return rc;
    if ((rc = dynoba_set_variable_order(h, DYNOBA_BIAS6, nn, b->nav_order.data()))) return rc;
  }
  return DYNOBA_OK;
}
int dynoba_builder_nav_counts(dynoba_builder_handle b, int64_t* n_vel, int64_t* n_bias) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  if (n_vel) *n_vel = (int64_t)b->vel.size()/3; if (n_bias) *n_bias = (int64_t)b->bias.size()/6;
  return DYNOBA_OK;
}
int dynoba_builder_get_nav_variables(dynoba_builder_handle b, double* vel, double* bias, int32_t* vel_order, int32_t* bias_order,
                                     uint64_t* vel_keys, uint64_t* bias_keys) {
  BARG(b, "null builder"); int rc = dynoba_builder_finalize(b); if (rc) return rc;
  if (vel) std::copy(b->vel.begin(), b->vel.end(), vel); if (bias) std::copy(b->bias.begin(), b->bias.end(), bias);
  if (vel_order) std::copy(b->nav_order.begin(), b->nav_order.end(), vel_order);
  if (bias_order) std::copy(b->nav_order.begin(), b->nav_order.end(), bias_order);
  if (vel_keys) std::copy(b->vel_keys.begin(), b->vel_keys.end(), vel_keys); if (bias_keys) std::copy(b->bias_keys.begin(), b->bias_keys.end(), bias_keys);
  return DYNOBA_OK;
}

}  // extern "C"
