"""ctypes binding of libdynofront.so (include/dynofront.h): dense-flow tracking / mask propagation / pyramidal KLT.
Mirrors the reference's FeatureTracker entry points (dynosam/src/frontend/vision/FeatureTracker.cc).  No CPU fallback."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdynofront.so")
EXPORTS = ["dynofront_create", "dynofront_destroy", "dynofront_last_error", "dynofront_set_frame", "dynofront_track_dynamic",
           "dynofront_sample_candidates", "dynofront_propagate_mask", "dynofront_klt_track", "dynofront_klt_track_fb",
           "dynofront_klt_last_min_eig", "dynofront_stereo_track", "dynofront_track_static_flow", "dynofront_next_frame", "dynofront_pin_host", "dynofront_unpin_host",
           "dynofront_get_motion_mask", "dynofront_get_pyramid_level", "dynofront_anms_range_tree", "dynofront_sample_dynamic",
           "dynofront_detect_static", "dynofront_detect_last_stages", "dynofront_set_depth", "dynofront_update_depths",
           "dynofront_back_project", "dynofront_dense_cloud", "dynofront_homography_default_params", "dynofront_find_homography_batch",
           "dynofront_homography_last_trace", "dynofront_homography_record_counts", "dynofront_klt_track_points",
           "dynofront_klt_dynamic_default_params", "dynofront_track_dynamic_klt", "dynofront_fundamental_default_params",
           "dynofront_find_fundamental_batch", "dynofront_fundamental_last_trace", "dynofront_fundamental_record", "dynofront_set_right",
           "dynofront_stereo_match", "dynofront_object_boundary"]


class TrackParamsC(C.Structure):
    _fields_ = [("max_dynamic_feature_age", C.c_int32), ("min_distance", C.c_int32), ("shrink_row", C.c_int32), ("shrink_col", C.c_int32)]


@dataclass
class TrackParams:
    max_dynamic_feature_age: int = 20
    min_distance: int = 2
    shrink_row: int = 0
    shrink_col: int = 0

    def c(self):
        return TrackParamsC(self.max_dynamic_feature_age, self.min_distance, self.shrink_row, self.shrink_col)


class KltFbParamsC(C.Structure):
    _fields_ = [("win", C.c_int32), ("max_level", C.c_int32), ("max_count", C.c_int32), ("epsilon", C.c_double),
                ("win_back", C.c_int32), ("max_level_back", C.c_int32), ("max_count_back", C.c_int32), ("epsilon_back", C.c_double),
                ("use_initial_flow", C.c_int32), ("min_eig_threshold", C.c_double), ("max_fb_distance", C.c_double),
                ("check_static", C.c_int32), ("max_feature_track_age", C.c_int32), ("track", TrackParamsC)]


class DetectParamsC(C.Structure):
    _fields_ = [("use_clahe", C.c_int32), ("use_anms", C.c_int32), ("use_subpix", C.c_int32), ("max_corners", C.c_int32),
                ("quality_level", C.c_double), ("block_size", C.c_int32), ("use_harris", C.c_int32), ("min_distance", C.c_int32),
                ("max_features", C.c_int32), ("subpix_win", C.c_int32), ("subpix_max_iter", C.c_int32), ("subpix_eps", C.c_double),
                ("track", TrackParamsC)]


@dataclass
class DetectParams:
    """KltFeatureTracker::detectFeatures parameters: TrackerParams defaults, params/FrontendParams.yaml where it sets them."""
    use_clahe: bool = True
    use_anms: bool = True
    use_subpix: bool = True
    max_corners: int = 1000          # max_nr_keypoints_before_anms
    quality_level: float = 0.001
    block_size: int = 3
    use_harris: bool = False
    min_distance: int = 15           # min_distance_btw_tracked_and_detected_static_features
    max_features: int = 800          # max_features_per_frame
    subpix_win: int = 5
    subpix_max_iter: int = 40
    subpix_eps: float = 0.001
    shrink_row: int = 0
    shrink_col: int = 0

    def c(self):
        return DetectParamsC(int(self.use_clahe), int(self.use_anms), int(self.use_subpix), self.max_corners, float(self.quality_level), self.block_size,
                             int(self.use_harris), self.min_distance, self.max_features, self.subpix_win, self.subpix_max_iter, float(self.subpix_eps),
                             TrackParamsC(0, 0, self.shrink_row, self.shrink_col))


class HomographyParamsC(C.Structure):
    _fields_ = [("threshold_px", C.c_double), ("confidence", C.c_double), ("max_iters", C.c_int32), ("refine", C.c_int32)]


@dataclass
class HomographyParams:
    """cv::findHomography(src, dst, RANSAC, threshold_px, mask, max_iters, confidence) as geometricVerification calls it;
    refine=False returns the RANSAC model and mask instead of the refined ones."""
    threshold_px: float = 5.0
    confidence: float = 0.995
    max_iters: int = 2000
    refine: bool = True

    def c(self):
        return HomographyParamsC(float(self.threshold_px), float(self.confidence), int(self.max_iters), int(bool(self.refine)))


HOM_OK, HOM_TOO_FEW, HOM_FOUR_POINT, HOM_RANSAC_FAILED = 0, 1, 2, 3     # dynofront_find_homography_batch status


class FundamentalParamsC(C.Structure):
    _fields_ = [("threshold_px", C.c_double), ("confidence", C.c_double), ("max_iters", C.c_int32)]


@dataclass
class FundamentalParams:
    """cv::findFundamentalMat(p1, p2, FM_RANSAC, threshold_px, confidence, max_iters) as stereoTrack calls it"""
    threshold_px: float = 1.0
    confidence: float = 0.99
    max_iters: int = 1000

    def c(self):
        return FundamentalParamsC(float(self.threshold_px), float(self.confidence), int(self.max_iters))


FUND_OK, FUND_LMEDS, FUND_SEVEN_POINT, FUND_TOO_FEW, FUND_FAILED = 0, 1, 2, 3, 4     # dynofront_find_fundamental_batch status
STEREO_UNTOUCHED, STEREO_MATCHED, STEREO_LOST, STEREO_EPIPOLAR, STEREO_DISPARITY = 0, 1, 2, 3, 4   # dynofront_stereo_match per-feature state


class KltDynamicParamsC(C.Structure):
    _fields_ = [("win", C.c_int32), ("max_level", C.c_int32), ("max_count", C.c_int32), ("epsilon", C.c_double), ("min_eig_threshold", C.c_double),
                ("track", TrackParamsC), ("max_features", C.c_int32), ("quality_level", C.c_double), ("age_buffer", C.c_int32),
                ("min_tracks", C.c_int32), ("min_iou", C.c_double)]


@dataclass
class KltDynamicParams:
    """FeatureTracker::trackDynamicKLT + requiresSampling parameters: the LK criteria of the reference's CPU call
    (FeatureTracker.cc:625-639) and params/FrontendParams.yaml."""
    win: int = 21
    max_level: int = 3
    max_count: int = 30
    epsilon: float = 0.03
    min_eig_threshold: float = 1e-4
    max_dynamic_feature_age: int = 20
    min_distance: int = 2              # min_distance_btw_tracked_and_detected_dynamic_features
    shrink_row: int = 0
    shrink_col: int = 0
    max_features: int = 200            # max_dynamic_features_per_frame
    quality_level: float = 0.01
    age_buffer: int = 3                # dynamic_feature_age_buffer
    min_tracks: int = 20               # min_dynamic_tracks
    min_iou: float = 0.1               # min_dynamic_mask_iou

    def c(self):
        return KltDynamicParamsC(self.win, self.max_level, self.max_count, float(self.epsilon), float(self.min_eig_threshold),
                                 TrackParamsC(self.max_dynamic_feature_age, self.min_distance, self.shrink_row, self.shrink_col),
                                 self.max_features, float(self.quality_level), self.age_buffer, self.min_tracks, float(self.min_iou))


class ObjectStatusC(C.Structure):
    _fields_ = [(f, C.c_int32) for f in ("object_id", "exists", "num_previous_track", "num_track", "num_outside_shrunken_image",
                                         "num_tracked_with_different_label", "num_tracked_with_background_label", "object_new",
                                         "object_resampled", "sampled", "num_sampled")]


OBJECT_STATUS_FIELDS = [f for f, _ in ObjectStatusC._fields_]
DKLT_TRACKED, DKLT_MASKED, DKLT_REJECTED, DKLT_OUTSIDE, DKLT_LOST = 1, 2, 3, 4, 5     # dynofront_track_dynamic_klt per-feature state


_LIB = None


def load():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it first (__graft_entry__.build()); there is no CPU fallback")
        L = C.CDLL(LIB_PATH)
        L.dynofront_last_error.restype = C.c_char_p
        L.dynofront_last_error.argtypes = [C.c_void_p]
        L.dynofront_create.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.dynofront_destroy.argtypes = [C.c_void_p]
        L.dynofront_set_frame.argtypes = [C.c_void_p] + [C.c_void_p]*3
        L.dynofront_track_dynamic.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p]*4 + [C.POINTER(TrackParamsC), C.POINTER(C.c_int64)] + [C.c_void_p]*8
        L.dynofront_sample_candidates.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(TrackParamsC)] + [C.c_void_p]*4 + [C.c_int64]
        L.dynofront_propagate_mask.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p]*4 + [C.POINTER(TrackParamsC), C.c_int32, C.c_void_p]
        L.dynofront_klt_track.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_double, C.POINTER(C.c_float)]
        L.dynofront_klt_track_fb.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.POINTER(KltFbParamsC), C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.dynofront_stereo_track.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]
        L.dynofront_set_right.argtypes = [C.c_void_p, C.c_void_p]
        L.dynofront_stereo_match.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_double, C.c_double,
                                             C.POINTER(FundamentalParamsC), C.POINTER(C.c_int32)] + [C.c_void_p]*6 + [C.POINTER(C.c_int32)]*4 + \
                                            [C.POINTER(C.c_float)]
        L.dynofront_klt_last_min_eig.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.dynofront_track_static_flow.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                                  C.POINTER(C.c_int64)] + [C.c_void_p]*8 + [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.dynofront_next_frame.argtypes = [C.c_void_p] + [C.c_void_p]*4
        L.dynofront_pin_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.dynofront_unpin_host.argtypes = [C.c_void_p, C.c_void_p]
        L.dynofront_get_motion_mask.argtypes = [C.c_void_p, C.c_void_p]
        L.dynofront_object_boundary.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32)] + [C.c_void_p]*4 + [C.POINTER(C.c_float)]
        L.dynofront_anms_range_tree.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p]*4 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]
        L.dynofront_sample_dynamic.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(TrackParamsC), C.POINTER(C.c_int64),
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p]*5 + [C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.dynofront_detect_static.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(DetectParamsC), C.POINTER(C.c_int64), C.c_int32,
                                              C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.dynofront_detect_last_stages.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
        L.dynofront_set_depth.argtypes = [C.c_void_p, C.c_void_p]
        L.dynofront_update_depths.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p,
                                              C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.dynofront_back_project.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p]*5 + [C.c_double, C.c_int32, C.c_void_p, C.c_int32] + [C.c_void_p]*4 + \
                                            [C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.dynofront_dense_cloud.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double] + [C.c_void_p]*4 + [C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.dynofront_homography_default_params.argtypes = [C.POINTER(HomographyParamsC)]
        L.dynofront_homography_default_params.restype = None
        L.dynofront_find_homography_batch.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(HomographyParamsC)] + \
                                                     [C.c_void_p]*5 + [C.POINTER(C.c_float)]
        L.dynofront_homography_last_trace.argtypes = [C.c_void_p] + [C.c_void_p]*4 + [C.c_int32, C.c_void_p, C.POINTER(C.c_int32)]
        L.dynofront_homography_record_counts.argtypes = [C.c_void_p, C.c_int32]
        L.dynofront_fundamental_default_params.argtypes = [C.POINTER(FundamentalParamsC)]
        L.dynofront_fundamental_default_params.restype = None
        L.dynofront_find_fundamental_batch.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(FundamentalParamsC)] + \
                                                      [C.c_void_p]*6 + [C.POINTER(C.c_float)]
        L.dynofront_fundamental_last_trace.argtypes = [C.c_void_p] + [C.c_void_p]*5 + [C.c_int32, C.c_void_p, C.POINTER(C.c_int32)]
        L.dynofront_fundamental_record.argtypes = [C.c_void_p, C.c_int32]
        L.dynofront_klt_track_points.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.POINTER(KltFbParamsC), C.POINTER(HomographyParamsC)] + [C.c_void_p]*4 + \
                                                [C.POINTER(C.c_int32)]*4 + [C.POINTER(C.c_float)]
        L.dynofront_klt_dynamic_default_params.argtypes = [C.POINTER(KltDynamicParamsC)]
        L.dynofront_klt_dynamic_default_params.restype = None
        L.dynofront_track_dynamic_klt.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p]*4 + [C.c_int32, C.c_void_p, C.c_void_p,
                                                  C.POINTER(KltDynamicParamsC), C.POINTER(C.c_int64)] + [C.c_void_p]*4 + [C.c_int32] + \
                                                 [C.c_void_p]*5 + [C.POINTER(C.c_int32), C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p,
                                                  C.POINTER(C.c_float)]
        L.dynofront_get_pyramid_level.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class FrontendError(RuntimeError):
    pass


def builder_measurements(bp, tracklet, object_id):
    """Turns FeatureTrackerGPU.back_project output into graph-builder arguments: the measurements that have a point, split into
    static (object 0) and dynamic ones.  tracklet / object_id are per input feature.  Returns ((tracklet, z), (tracklet, object,
    z)) for dynoba_builder_add_static / dynoba_builder_add_dynamic (dynosam_b200.builder.GraphBuilder.add_static / add_dynamic)."""
    idx = np.asarray(bp["index"]); z = np.asarray(bp["point"]).reshape(-1, 3)
    has = ~np.isnan(z[:, 2]); idx = idx[has]; z = z[has]
    tid = np.asarray(tracklet, np.int64)[idx]; obj = np.asarray(object_id, np.int32)[idx]
    st = obj == 0
    return (tid[st], z[st]), (tid[~st], obj[~st], z[~st])


def pnp_correspondences(tracklet_prev, usable_prev, label_prev, bp_prev, tracklet_cur, usable_cur, label_cur, kp_cur, calib5):
    """The 3D-2D problems of a frame for binding.pnp_ransac_batch: what Frame::getCorrespondences gathers for
    EgoMotionSolver::geometricOutlierRejection3d2d (camera, label 0) and for every object (Frame-inl.hpp:38-64,
    VisionTools.cc:75-98).  Frame k's features are visited in container order; a feature enters when it is usable, its tracklet
    is in frame k-1, usable there with the same label.  Its reference is the world point of the k-1 feature, from
    FeatureTrackerGPU.back_project(..., X_world=pose_k-1) of frame k-1 (bp_prev: index / point); a feature without one raises
    ValueError, as the reference throws when the previous feature has no depth (Frame.cc:280-285).  Returns the camera problem
    first, then one problem per object in ascending label: dicts with label, tracklet [m], points [m,3], kp [m,2], calib [5]."""
    t0 = np.asarray(tracklet_prev, np.int64); u0 = np.asarray(usable_prev, bool); l0 = np.asarray(label_prev, np.int64)
    t1 = np.asarray(tracklet_cur, np.int64); u1 = np.asarray(usable_cur, bool); l1 = np.asarray(label_cur, np.int64)
    kp = np.asarray(kp_cur, np.float64).reshape(-1, 2)
    pw = np.full((len(t0), 3), np.nan)
    pw[np.asarray(bp_prev["index"], np.int64)] = np.asarray(bp_prev["point"], np.float64).reshape(-1, 3)
    order = np.argsort(t0, kind="stable")
    j = np.searchsorted(t0[order], t1).clip(0, max(len(t0) - 1, 0))
    j = order[j] if len(t0) else np.zeros(len(t1), np.int64)
    take = u1 & (t0[j] == t1) & u0[j] & (l0[j] == l1) if len(t0) else np.zeros(len(t1), bool)
    if np.isnan(pw[j[take]]).any():
        raise ValueError("pnp_correspondences: a previous feature has no world point (no depth)")
    cal = np.asarray(calib5, np.float64).reshape(5)
    out = []
    for lab in [0] + sorted(set(int(x) for x in l1[take]) - {0}):
        s = take & (l1 == lab)
        out.append(dict(label=lab, tracklet=t1[s], points=pw[j[s]], kp=kp[s], calib=cal.copy()))
    return out


class FeatureTrackerGPU:
    """One handle per camera stream (image size fixed at construction)."""

    def __init__(self, width, height, device=0):
        self.lib = load(); self.W, self.H = int(width), int(height)
        self.h = C.c_void_p()
        st = self.lib.dynofront_create(device, self.W, self.H, C.byref(self.h))
        if st != 0:
            raise FrontendError(f"dynofront_create failed ({st}): no sm_90 CUDA device; libdynofront has no CPU path")

    def _ck(self, st):
        if st != 0:
            raise FrontendError(f"libdynofront status {st}: {self.lib.dynofront_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            self.lib.dynofront_destroy(self.h); self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_frame(self, flow, motion_mask, detection_mask=None):
        flow = np.ascontiguousarray(flow, dtype=np.float32); motion_mask = np.ascontiguousarray(motion_mask, dtype=np.int32)
        det = None if detection_mask is None else np.ascontiguousarray(detection_mask, dtype=np.uint8)
        self._ck(self.lib.dynofront_set_frame(self.h, _p(flow), _p(motion_mask), _p(det)))

    # ---- streaming mode (resident frames)
    def pin(self, arr):
        """register a C-contiguous numpy array as pinned host memory (asynchronous uploads); keep it alive until unpin"""
        self._ck(self.lib.dynofront_pin_host(self.h, _p(arr), arr.nbytes))

    def unpin(self, arr):
        self._ck(self.lib.dynofront_unpin_host(self.h, _p(arr)))

    def next_frame(self, gray, flow, motion_mask, detection_mask=None):
        """arrays must already be C-contiguous uint8 / float32 / int32 (no conversion copies on the streaming path)"""
        assert gray.dtype == np.uint8 and flow.dtype == np.float32 and motion_mask.dtype == np.int32
        assert gray.flags.c_contiguous and flow.flags.c_contiguous and motion_mask.flags.c_contiguous
        self._ck(self.lib.dynofront_next_frame(self.h, _p(gray), _p(flow), _p(motion_mask), _p(detection_mask)))

    def propagate_mask_resident(self, prev_pred_kp, prev_label, prm: TrackParams, min_votes=150):
        kp = np.ascontiguousarray(prev_pred_kp, dtype=np.float64).reshape(-1, 2); lab = np.ascontiguousarray(prev_label, dtype=np.int32)
        pc = prm.c()
        self._ck(self.lib.dynofront_propagate_mask(self.h, kp.shape[0], _p(kp), _p(lab), None, None, C.byref(pc), int(min_votes), None))

    def motion_mask(self):
        out = np.zeros((self.H, self.W), np.int32)
        self._ck(self.lib.dynofront_get_motion_mask(self.h, _p(out)))
        return out

    def object_boundary(self, thickness=-1, want_mask=False, capacity=255):
        """FeatureTracker::objectDetection with a provided mask (dynofront_object_boundary): computeObjectMaskBoundaryMask on the
        current motion mask as uploaded.  thickness < 0: the reference's scaled value for the frame size.  The boundary mask becomes
        the current frame's (as if uploaded through next_frame).  Returns (objects [n] ascending, bb [n][4], inner_bb [n][4], and
        with want_mask the boundary mask u8[H][W], else None); capacity limits the rows returned."""
        cap = int(capacity)
        objs = np.zeros(max(cap, 1), np.int32); bb = np.zeros((max(cap, 1), 4), np.int32); ib = np.zeros((max(cap, 1), 4), np.int32)
        mask = np.zeros((self.H, self.W), np.uint8) if want_mask else None
        n = C.c_int32(); ms = C.c_float()
        self._ck(self.lib.dynofront_object_boundary(self.h, int(thickness), cap, C.byref(n), _p(objs), _p(bb), _p(ib), _p(mask), C.byref(ms)))
        self.last_ms = ms.value; self.last_n_objects = n.value
        s = min(n.value, cap)
        return objs[:s], bb[:s], ib[:s], mask

    def track_dynamic(self, prev_pred_kp, prev_label, prev_age, prev_tracklet, prm: TrackParams, next_tracklet_id: int, want_masks=True):
        kp = np.ascontiguousarray(prev_pred_kp, dtype=np.float64).reshape(-1, 2); n = kp.shape[0]
        lab = np.ascontiguousarray(prev_label, dtype=np.int32); age = np.ascontiguousarray(prev_age, dtype=np.int32)
        tid = np.ascontiguousarray(prev_tracklet, dtype=np.int64)
        acc = np.zeros(n, np.uint8); pk = np.zeros((n, 2)); fl = np.zeros((n, 2)); oage = np.zeros(n, np.int32)
        otid = np.zeros(n, np.int64); olab = np.zeros(n, np.int32)
        det = np.zeros((self.H, self.W), np.uint8) if want_masks else None
        trk = np.zeros((self.H, self.W), np.uint8) if want_masks else None
        nid = C.c_int64(int(next_tracklet_id)); pc = prm.c()
        self._ck(self.lib.dynofront_track_dynamic(self.h, n, _p(kp), _p(lab), _p(age), _p(tid), C.byref(pc), C.byref(nid), _p(acc), _p(pk), _p(fl),
                                                  _p(oage), _p(otid), _p(olab), _p(det), _p(trk)))
        return acc, pk, fl, oage, otid, olab, nid.value, det, trk

    def sample_candidates(self, objects, prm: TrackParams, capacity=None):
        objs = np.ascontiguousarray(objects, dtype=np.int32); n = objs.shape[0]
        cap = int(capacity if capacity is not None else self.W*self.H)
        counts = np.zeros(n, np.int32); offs = np.zeros(n, np.int32); zero = np.zeros(n, np.int32); idx = np.empty(cap, np.int32)
        pc = prm.c()
        self._ck(self.lib.dynofront_sample_candidates(self.h, n, _p(objs), C.byref(pc), _p(counts), _p(offs), _p(zero), _p(idx), cap))
        return {int(o): idx[offs[i]:offs[i] + counts[i]].copy() for i, o in enumerate(objs)}, {int(o): int(zero[i]) for i, o in enumerate(objs)}

    def anms_range_tree(self, lists, k_needed, tolerance, cols=None, rows=None):
        """Range-tree ANMS (suppressNonMax, response-0 key-points) on several integer key-point lists in one launch.
        lists: sequence of [n_l, 2] (col, row) arrays; k_needed / tolerance: one value per list (or a scalar).
        Returns one int32 array per list: indices of the selected key-points, in selection order."""
        lists = [np.ascontiguousarray(a, dtype=np.int32).reshape(-1, 2) for a in lists]; m = len(lists)
        offs = np.zeros(m + 1, np.int32); offs[1:] = np.cumsum([len(a) for a in lists])
        xy = np.ascontiguousarray(np.concatenate(lists) if m else np.zeros((0, 2), np.int32), dtype=np.int32)
        k = np.ascontiguousarray(np.broadcast_to(np.asarray(k_needed, np.int32), (m,)))
        tol = np.ascontiguousarray(np.broadcast_to(np.asarray(tolerance, np.float32), (m,)))
        sel = np.zeros(max(int(offs[-1]), 1), np.int32); nsel = np.zeros(max(m, 1), np.int32); ms = C.c_float()
        self._ck(self.lib.dynofront_anms_range_tree(self.h, m, _p(offs), _p(xy), _p(k), _p(tol), int(cols or self.W), int(rows or self.H),
                                                    _p(sel), _p(nsel), C.byref(ms)))
        self.last_ms = ms.value
        return [sel[offs[l]:offs[l] + nsel[l]].copy() for l in range(m)]

    def sample_dynamic(self, objects, num_track, prm: TrackParams, next_tracklet_id: int, max_features=200, capacity=None):
        """FeatureTracker::sampleDynamic on the device: candidate scan, range-tree ANMS per object, new features.  Uses the
        detection mask left by track_dynamic (or the uploaded one).  Returns a dict: per object counts / num_sampled /
        zero_flow, per feature keypoint / flow / predicted / tracklet / label (packed object after object), next_tracklet_id."""
        objs = np.ascontiguousarray(objects, dtype=np.int32); n = objs.shape[0]
        ntr = np.ascontiguousarray(np.broadcast_to(np.asarray(num_track, np.int32), (n,)))
        cap = int(capacity if capacity is not None else n*max(int(max_features), 1)*2 + 64)
        counts = np.zeros(n, np.int32); ns = np.zeros(n, np.int32); zero = np.zeros(n, np.int32)
        kp = np.zeros((cap, 2)); fl = np.zeros((cap, 2)); pk = np.zeros((cap, 2)); tid = np.zeros(cap, np.int64); lab = np.zeros(cap, np.int32)
        nid = C.c_int64(int(next_tracklet_id)); nf = C.c_int32(); ms = C.c_float(); pc = prm.c()
        self._ck(self.lib.dynofront_sample_dynamic(self.h, n, _p(objs), _p(ntr), int(max_features), C.byref(pc), C.byref(nid), _p(counts), _p(ns),
                                                   _p(zero), cap, _p(kp), _p(fl), _p(pk), _p(tid), _p(lab), C.byref(nf), C.byref(ms)))
        self.last_ms = ms.value
        if nf.value > cap:                                        # more than the guess: run again with room for all
            return self.sample_dynamic(objects, num_track, prm, next_tracklet_id, max_features, nf.value)
        s = nf.value
        return dict(counts=counts, num_sampled=ns, zero_flow=zero, keypoint=kp[:s], flow=fl[:s], predicted=pk[:s], tracklet=tid[:s], label=lab[:s],
                    next_tracklet_id=nid.value)

    def detect_static(self, gray, cur_kp, prm: DetectParams, next_tracklet_id: int, capacity=None):
        """KltFeatureTracker::detectFeatures on the device: detection mask, CLAHE, good-features-to-track, range-tree ANMS,
        cornerSubPix and the new static features.  gray=None: the resident current frame of next_frame.  Uses the motion mask
        and boundary mask of the current frame.  Returns (keypoints [n][2], tracklet ids, next_tracklet_id, n_corners)."""
        g = None if gray is None else np.ascontiguousarray(gray, dtype=np.uint8)
        kp = np.ascontiguousarray(cur_kp, dtype=np.float64).reshape(-1, 2); n = kp.shape[0]
        cap = int(capacity if capacity is not None else max(prm.max_features, 1) + 64)
        out = np.zeros((cap, 2)); tid = np.zeros(cap, np.int64)
        nid = C.c_int64(int(next_tracklet_id)); nf = C.c_int32(); nc = C.c_int32(); ms = C.c_float(); pc = prm.c()
        self._ck(self.lib.dynofront_detect_static(self.h, _p(g), n, _p(kp), C.byref(pc), C.byref(nid), cap, _p(out), _p(tid), C.byref(nf), C.byref(nc),
                                                  C.byref(ms)))
        self.last_ms = ms.value
        if nf.value > cap:                                        # more than the guess: run again with room for all
            return self.detect_static(gray, cur_kp, prm, next_tracklet_id, nf.value)
        return out[:nf.value], tid[:nf.value], nid.value, nc.value

    def detect_stages(self):
        """the last detect_static's CLAHE image, minimum-eigenvalue image and GFTT corners before ANMS ([n][2] x, y)"""
        nc = C.c_int32()
        self._ck(self.lib.dynofront_detect_last_stages(self.h, None, None, None, C.byref(nc)))
        cl = np.zeros((self.H, self.W), np.uint8); eig = np.zeros((self.H, self.W), np.float32); xy = np.zeros((max(nc.value, 1), 2), np.int32)
        self._ck(self.lib.dynofront_detect_last_stages(self.h, _p(cl), _p(eig), _p(xy), C.byref(nc)))
        return cl, eig, xy[:nc.value]

    def propagate_mask(self, prev_pred_kp, prev_label, prev_mask, prev_flow, current_mask, prm: TrackParams, min_votes=150):
        kp = np.ascontiguousarray(prev_pred_kp, dtype=np.float64).reshape(-1, 2)
        lab = np.ascontiguousarray(prev_label, dtype=np.int32)
        pm = np.ascontiguousarray(prev_mask, dtype=np.int32); pf = np.ascontiguousarray(prev_flow, dtype=np.float32)
        cur = np.ascontiguousarray(current_mask, dtype=np.int32).copy(); pc = prm.c()
        self._ck(self.lib.dynofront_propagate_mask(self.h, kp.shape[0], _p(kp), _p(lab), _p(pm), _p(pf), C.byref(pc), int(min_votes), _p(cur)))
        return cur

    def klt_track(self, prev_gray, cur_gray, prev_pts, win=21, max_level=3, max_count=30, eps=0.03, initial=None, min_eig=1e-4):
        """cv::calcOpticalFlowPyrLK(prev, cur, prevPts, nextPts, status, err, (win,win), maxLevel, (EPS|COUNT, max_count, eps))."""
        pg = np.ascontiguousarray(prev_gray, dtype=np.uint8); cg = np.ascontiguousarray(cur_gray, dtype=np.uint8)
        p0 = np.ascontiguousarray(prev_pts, dtype=np.float32).reshape(-1, 2); n = p0.shape[0]
        nxt = np.ascontiguousarray(initial, dtype=np.float32).reshape(-1, 2).copy() if initial is not None else np.zeros((n, 2), np.float32)
        st = np.zeros(n, np.uint8); err = np.zeros(n, np.float32); ms = C.c_float()
        self._ck(self.lib.dynofront_klt_track(self.h, _p(pg), _p(cg), n, _p(p0), _p(nxt), _p(st), _p(err), win, max_level, max_count, float(eps),
                                              1 if initial is not None else 0, float(min_eig), C.byref(ms)))
        self.last_ms = ms.value
        return nxt, st, err

    def klt_track_fb(self, prev_gray, cur_gray, prev_pts, prm: TrackParams | None = None, prev_age=None, max_feature_track_age=25,
                     win=21, max_level=3, max_count=30, eps=0.03, initial=None, min_eig=1e-4, max_fb_distance=0.5):
        """KltFeatureTracker::trackPoints in one call: forward LK, backward LK (21x21, 5 levels, OpenCV default criteria), the
        round-trip test and -- when prev_age is given -- the label / border / age checks.  Returns (next, status, back, keep)."""
        pg = None if prev_gray is None else np.ascontiguousarray(prev_gray, dtype=np.uint8)     # None, None: the resident frame pair
        cg = None if cur_gray is None else np.ascontiguousarray(cur_gray, dtype=np.uint8)
        p0 = np.ascontiguousarray(prev_pts, dtype=np.float32).reshape(-1, 2); n = p0.shape[0]
        nxt = np.ascontiguousarray(initial, dtype=np.float32).reshape(-1, 2).copy() if initial is not None else np.zeros((n, 2), np.float32)
        st = np.zeros(n, np.uint8); back = np.zeros((n, 2), np.float32); keep = np.zeros(n, np.uint8); ms = C.c_float()
        check = prev_age is not None
        age = np.ascontiguousarray(prev_age, dtype=np.int32) if check else None
        pc = KltFbParamsC(win, max_level, max_count, float(eps), 21, 5, 30, 0.01, 1 if initial is not None else 0, float(min_eig), float(max_fb_distance),
                          1 if check else 0, int(max_feature_track_age), (prm or TrackParams()).c())
        ns = C.c_int32(); nk = C.c_int32()
        self._ck(self.lib.dynofront_klt_track_fb(self.h, _p(pg), _p(cg), n, _p(p0), _p(nxt), _p(st), _p(back), C.byref(pc), _p(age), _p(keep),
                                                 C.byref(ns), C.byref(nk), C.byref(ms)))
        self.last_ms = ms.value; self.last_counts = (ns.value, nk.value)
        return nxt, st, back, (keep if check else None)

    def klt_track_points(self, prev_gray, cur_gray, prev_pts, prm: TrackParams | None = None, prev_age=None, max_feature_track_age=25,
                         hom: HomographyParams | None = None, win=21, max_level=3, max_count=30, eps=0.03, initial=None, min_eig=1e-4,
                         max_fb_distance=0.5):
        """KltFeatureTracker::trackPoints steps 1-4 in one call: klt_track_fb's stages, then cv::findHomography(RANSAC) over the
        points that passed the round trip, in order, then the checks.  Returns (next, status, verified, keep, H); keep is None
        without prev_age, H is None when the homography has none.  self.last_counts = (n_status, n_verified, n_keep),
        self.last_hom_status = the homography's HOM_* status."""
        pg = None if prev_gray is None else np.ascontiguousarray(prev_gray, dtype=np.uint8)     # None, None: the resident frame pair
        cg = None if cur_gray is None else np.ascontiguousarray(cur_gray, dtype=np.uint8)
        p0 = np.ascontiguousarray(prev_pts, dtype=np.float32).reshape(-1, 2); n = p0.shape[0]
        nxt = np.ascontiguousarray(initial, dtype=np.float32).reshape(-1, 2).copy() if initial is not None else np.zeros((n, 2), np.float32)
        st = np.zeros(n, np.uint8); ver = np.zeros(n, np.uint8); keep = np.zeros(n, np.uint8); H = np.zeros(9); ms = C.c_float()
        check = prev_age is not None
        age = np.ascontiguousarray(prev_age, dtype=np.int32) if check else None
        pc = KltFbParamsC(win, max_level, max_count, float(eps), 21, 5, 30, 0.01, 1 if initial is not None else 0, float(min_eig), float(max_fb_distance),
                          1 if check else 0, int(max_feature_track_age), (prm or TrackParams()).c())
        hc = (hom or HomographyParams()).c()
        hs = C.c_int32(); ns = C.c_int32(); nv = C.c_int32(); nk = C.c_int32()
        self._ck(self.lib.dynofront_klt_track_points(self.h, _p(pg), _p(cg), n, _p(p0), _p(nxt), _p(st), C.byref(pc), C.byref(hc), _p(age), _p(ver),
                                                     _p(keep), _p(H), C.byref(hs), C.byref(ns), C.byref(nv), C.byref(nk), C.byref(ms)))
        self.last_ms = ms.value; self.last_counts = (ns.value, nv.value, nk.value); self.last_hom_status = hs.value
        return nxt, st, ver, (keep if check else None), (H.reshape(3, 3) if hs.value in (HOM_OK, HOM_FOUR_POINT) and H.any() else None)

    def track_dynamic_klt(self, prev_gray, cur_gray, prev_kp, prev_label, prev_age, prev_tracklet, objects, inner_bb, next_tracklet_id: int,
                          prm: KltDynamicParams | None = None, want_masks=True, capacity=None):
        """FeatureTracker::trackDynamicKLT with requiresSampling in one call (dynofront_track_dynamic_klt).  prev_gray = cur_gray =
        None: the resident frame pair of next_frame.  prev_kp [n][2] (float32, as toOpenCV gives it), labels, ages, tracklet ids of
        the previous usable dynamic features; objects / inner_bb [m][4] (x, y, w, h) from the object boundary mask.  Uses the motion
        mask and boundary mask of the current frame.  Returns a dict: per previous feature lk_pts, lk_status, state (DKLT_*),
        tracked, measured_flow; the output features keypoint / age / tracklet / label / source (tracked ones first, by ascending
        label, then the new ones in objects order); status (a dict of arrays over [label 0] + objects, OBJECT_STATUS_FIELDS);
        n_outside_image, next_tracklet_id and, with want_masks, detection_mask / tracking_mask."""
        pg = None if prev_gray is None else np.ascontiguousarray(prev_gray, dtype=np.uint8)
        cg = None if cur_gray is None else np.ascontiguousarray(cur_gray, dtype=np.uint8)
        kp = np.ascontiguousarray(prev_kp, dtype=np.float32).reshape(-1, 2); n = kp.shape[0]
        lab = np.ascontiguousarray(prev_label, dtype=np.int32).reshape(n); age = np.ascontiguousarray(prev_age, dtype=np.int32).reshape(n)
        tid = np.ascontiguousarray(prev_tracklet, dtype=np.int64).reshape(n)
        objs = np.ascontiguousarray(objects, dtype=np.int32).reshape(-1); m = objs.shape[0]
        bb = np.ascontiguousarray(inner_bb, dtype=np.int32).reshape(m, 4)
        p = prm or KltDynamicParams()
        cap = int(capacity if capacity is not None else n + m*max(p.max_features, 1))
        lk = np.zeros((n, 2), np.float32); st = np.zeros(n, np.uint8); state = np.zeros(n, np.uint8); fl = np.zeros((n, 2))
        okp = np.zeros((max(cap, 1), 2)); oage = np.zeros(max(cap, 1), np.int32); otid = np.zeros(max(cap, 1), np.int64)
        olab = np.zeros(max(cap, 1), np.int32); osrc = np.zeros(max(cap, 1), np.int32)
        rows = (ObjectStatusC*(m + 1))()
        det = np.zeros((self.H, self.W), np.uint8) if want_masks else None
        trk = np.zeros((self.H, self.W), np.uint8) if want_masks else None
        nid = C.c_int64(int(next_tracklet_id)); nf = C.c_int32(); no = C.c_int32(); ms = C.c_float(); pc = p.c()
        self._ck(self.lib.dynofront_track_dynamic_klt(self.h, _p(pg), _p(cg), n, _p(kp), _p(lab), _p(age), _p(tid), m, _p(objs), _p(bb), C.byref(pc),
                                                      C.byref(nid), _p(lk), _p(st), _p(state), _p(fl), cap, _p(okp), _p(oage), _p(otid), _p(olab),
                                                      _p(osrc), C.byref(nf), C.cast(rows, C.c_void_p), C.byref(no), _p(det), _p(trk), C.byref(ms)))
        self.last_ms = ms.value
        if nf.value > cap:                                        # more than the guess: the call is not repeatable (ids), so refuse
            raise FrontendError(f"track_dynamic_klt: {nf.value} features exceed capacity {cap}")
        s = nf.value
        status = {f: np.array([getattr(r, f) for r in rows], np.int32) for f in OBJECT_STATUS_FIELDS}
        return dict(lk_pts=lk, lk_status=st, state=state, tracked=(state == DKLT_TRACKED).astype(np.uint8), measured_flow=fl, keypoint=okp[:s],
                    age=oage[:s], tracklet=otid[:s], label=olab[:s], source=osrc[:s], status=status, n_outside_image=no.value,
                    next_tracklet_id=nid.value, detection_mask=det, tracking_mask=trk)

    def find_homography_batch(self, problems, prm: HomographyParams | None = None):
        """cv::findHomography(src, dst, RANSAC, ...) on every problem in one launch.  problems: sequence of (src [n][2], dst [n][2]).
        Returns a dict: H [P][3][3] (0 where there is none), masks (one u8 array per problem), n_inliers, status, iterations."""
        srcs = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 2) for a, _ in problems]
        dsts = [np.ascontiguousarray(b, dtype=np.float32).reshape(-1, 2) for _, b in problems]
        P = len(srcs)
        off = np.zeros(P + 1, np.int32); off[1:] = np.cumsum([len(a) for a in srcs])
        src = np.ascontiguousarray(np.concatenate(srcs) if P else np.zeros((0, 2), np.float32))
        dst = np.ascontiguousarray(np.concatenate(dsts) if P else np.zeros((0, 2), np.float32))
        if src.shape != dst.shape:
            raise ValueError("find_homography_batch: src and dst of a problem must have the same length")
        H = np.zeros((max(P, 1), 9)); mask = np.zeros(max(int(off[-1]), 1), np.uint8)
        ninl = np.zeros(max(P, 1), np.int32); st = np.zeros(max(P, 1), np.int32); it = np.zeros(max(P, 1), np.int32); ms = C.c_float()
        pc = (prm or HomographyParams()).c()
        self._ck(self.lib.dynofront_find_homography_batch(self.h, P, _p(off), _p(src), _p(dst), C.byref(pc), _p(H), _p(mask), _p(ninl), _p(st), _p(it),
                                                          C.byref(ms)))
        self.last_ms = ms.value
        return dict(H=H[:P].reshape(P, 3, 3), masks=[mask[off[p]:off[p + 1]].copy() for p in range(P)], n_inliers=ninl[:P], status=st[:P],
                    iterations=it[:P])

    def homography_record_counts(self, counts_cap):
        """record the inlier count of each of the first counts_cap iterations in the following calls (0: none, the default)"""
        self._ck(self.lib.dynofront_homography_record_counts(self.h, int(counts_cap)))

    def homography_trace(self, counts_cap=0):
        """the draw trace of the last find_homography_batch / klt_track_points: status, groups, rejected, best (iteration of the
        best model) per problem, and counts [P][counts_cap] (inlier count per iteration as recorded after
        homography_record_counts; -1 without a model, past the end or not recorded)"""
        npb = C.c_int32()
        self._ck(self.lib.dynofront_homography_last_trace(self.h, None, None, None, None, 0, None, C.byref(npb)))
        P = npb.value; m = max(P, 1)
        st = np.zeros(m, np.int32); g = np.zeros(m, np.int32); rj = np.zeros(m, np.int32); b = np.zeros(m, np.int32)
        cnt = np.zeros((m, max(counts_cap, 1)), np.int32)
        self._ck(self.lib.dynofront_homography_last_trace(self.h, _p(st), _p(g), _p(rj), _p(b), int(counts_cap), _p(cnt) if counts_cap else None,
                                                          C.byref(npb)))
        return dict(status=st[:P], groups=g[:P], rejected=rj[:P], best=b[:P], counts=cnt[:P, :counts_cap])

    def find_fundamental_batch(self, problems, prm: FundamentalParams | None = None):
        """cv::findFundamentalMat(p1, p2, FM_RANSAC, ...) on every problem in one launch.  problems: sequence of (p1 [n][2],
        p2 [n][2]).  Returns a dict: F [P][3][3][3] (up to 3 models, 0 past n_models), n_models, masks (one u8 array per problem),
        n_inliers, status (FUND_*), iterations."""
        p1s = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 2) for a, _ in problems]
        p2s = [np.ascontiguousarray(b, dtype=np.float32).reshape(-1, 2) for _, b in problems]
        if any(a.shape != b.shape for a, b in zip(p1s, p2s)):
            raise ValueError("find_fundamental_batch: p1 and p2 of a problem must have the same length")
        P = len(p1s)
        off = np.zeros(P + 1, np.int32); off[1:] = np.cumsum([len(a) for a in p1s])
        p1 = np.ascontiguousarray(np.concatenate(p1s) if P else np.zeros((0, 2), np.float32))
        p2 = np.ascontiguousarray(np.concatenate(p2s) if P else np.zeros((0, 2), np.float32))
        m = max(P, 1)
        F = np.zeros((m, 27)); mask = np.zeros(max(int(off[-1]), 1), np.uint8)
        nm = np.zeros(m, np.int32); ninl = np.zeros(m, np.int32); st = np.zeros(m, np.int32); it = np.zeros(m, np.int32); ms = C.c_float()
        pc = (prm or FundamentalParams()).c()
        self._ck(self.lib.dynofront_find_fundamental_batch(self.h, P, _p(off), _p(p1), _p(p2), C.byref(pc), _p(F), _p(nm), _p(mask), _p(ninl),
                                                           _p(st), _p(it), C.byref(ms)))
        self.last_ms = ms.value
        return dict(F=F[:P].reshape(P, 3, 3, 3), n_models=nm[:P], masks=[mask[off[p]:off[p + 1]].copy() for p in range(P)],
                    n_inliers=ninl[:P], status=st[:P], iterations=it[:P])

    def fundamental_record(self, iters_cap):
        """record (models, scores) of each of the first iters_cap iterations in the following calls (0: none, the default)"""
        self._ck(self.lib.dynofront_fundamental_record(self.h, int(iters_cap)))

    def fundamental_trace(self, iters_cap=0):
        """the draw trace of the last find_fundamental_batch: groups, rejected, best (iteration), best_root, success per problem,
        and record [P][iters_cap][4] = (models of the draw, score of root 0, 1, 2) as recorded after fundamental_record (NaN
        where nothing was recorded; the score is the inlier count under RANSAC, the median error under LMedS)"""
        npb = C.c_int32()
        self._ck(self.lib.dynofront_fundamental_last_trace(self.h, None, None, None, None, None, 0, None, C.byref(npb)))
        P = npb.value; m = max(P, 1)
        a = [np.zeros(m, np.int32) for _ in range(5)]
        rec = np.zeros((m, max(iters_cap, 1), 4), np.float32)
        self._ck(self.lib.dynofront_fundamental_last_trace(self.h, *[_p(x) for x in a], int(iters_cap), _p(rec) if iters_cap else None,
                                                           C.byref(npb)))
        return dict(groups=a[0][:P], rejected=a[1][:P], best=a[2][:P], best_root=a[3][:P], success=a[4][:P], record=rec[:P, :iters_cap])

    def stereo_track(self, left_gray, right_gray, left_pts, fx, baseline):
        """FeatureTracker::stereoTrack without its RANSAC: (right_pts, status, depth, valid)"""
        lg = np.ascontiguousarray(left_gray, dtype=np.uint8); rg = np.ascontiguousarray(right_gray, dtype=np.uint8)
        p0 = np.ascontiguousarray(left_pts, dtype=np.float32).reshape(-1, 2); n = p0.shape[0]
        rp = np.zeros((n, 2), np.float32); st = np.zeros(n, np.uint8); depth = np.zeros(n); valid = np.zeros(n, np.uint8); ms = C.c_float()
        self._ck(self.lib.dynofront_stereo_track(self.h, _p(lg), _p(rg), n, _p(p0), _p(rp), _p(st), float(fx), float(baseline), _p(depth), _p(valid), C.byref(ms)))
        self.last_ms = ms.value
        return rp, st, depth, valid

    def set_right(self, right):
        """upload the current frame's right image (uint8 [H][W]) and build its pyramid; call after next_frame, which marks it
        stale.  A C-contiguous uint8 array is passed as is (pin it for an asynchronous copy and keep it untouched until the next call)."""
        r = np.ascontiguousarray(right, dtype=np.uint8)
        assert r.shape == (self.H, self.W)
        self._keep_right = r                                     # the copy may still be in flight when this returns
        self._ck(self.lib.dynofront_set_right(self.h, _p(r)))

    def stereo_match(self, left_pts, fx, baseline, prm: FundamentalParams | None = None, left=None, right=None):
        """FeatureTracker::stereoTrack in one call (dynofront_stereo_match): LK left -> right, cv::findFundamentalMat(FM_RANSAC)
        over the LK-good points, the disparity test.  left = right = None: the resident current frame of next_frame and the
        right image of set_right.  left_pts [n][2]: the usable static features in container order.  Returns a dict: matched (the
        reference's return value), per point state (STEREO_*), depth and right_u (NaN unless MATCHED), right_pts / lk_status (the
        LK result), F [3][3], fund_status (FUND_*, -1 when the RANSAC did not run), n_tracked, n_inliers, n_stereo."""
        lg = None if left is None else np.ascontiguousarray(left, dtype=np.uint8)
        rg = None if right is None else np.ascontiguousarray(right, dtype=np.uint8)
        p0 = np.ascontiguousarray(left_pts, dtype=np.float32).reshape(-1, 2); n = p0.shape[0]
        state = np.zeros(n, np.uint8); depth = np.zeros(n); ru = np.zeros(n); rp = np.zeros((n, 2), np.float32); st = np.zeros(n, np.uint8)
        F = np.zeros(9); mt = C.c_int32(); fs = C.c_int32(); nt = C.c_int32(); ni = C.c_int32(); ns = C.c_int32(); ms = C.c_float()
        pc = (prm or FundamentalParams()).c()
        self._ck(self.lib.dynofront_stereo_match(self.h, _p(lg), _p(rg), n, _p(p0), float(fx), float(baseline), C.byref(pc), C.byref(mt), _p(state),
                                                 _p(depth), _p(ru), _p(rp), _p(st), _p(F), C.byref(fs), C.byref(nt), C.byref(ni), C.byref(ns),
                                                 C.byref(ms)))
        self.last_ms = ms.value
        return dict(matched=bool(mt.value), state=state, depth=depth, right_u=ru, right_pts=rp, lk_status=st, F=F.reshape(3, 3),
                    fund_status=fs.value, n_tracked=nt.value, n_inliers=ni.value, n_stereo=ns.value)

    # ---- depth and back-projection
    def set_depth(self, depth):
        """upload the current frame's depth image (float64 [H][W]); call after set_frame / next_frame, which mark it stale.
        A C-contiguous float64 array is passed as is (pin it for an asynchronous copy and keep it untouched until the next call)."""
        d = np.ascontiguousarray(depth, dtype=np.float64)
        assert d.shape == (self.H, self.W)
        self._keep_depth = d                                     # the copy may still be in flight when this returns
        self._ck(self.lib.dynofront_set_depth(self.h, _p(d)))

    def update_depths(self, kp, label, max_background_depth=200.0, max_object_depth=30.0):
        """Frame::updateDepths on features kp[n][2] with labels (0 = static): returns (depth, valid, n_invalid, n_outside)"""
        k = np.ascontiguousarray(kp, dtype=np.float64).reshape(-1, 2); n = k.shape[0]
        lab = np.ascontiguousarray(np.broadcast_to(np.asarray(label, np.int32), (n,)))
        d = np.zeros(n); v = np.zeros(n, np.uint8); ni = C.c_int32(); no = C.c_int32(); ms = C.c_float()
        self._ck(self.lib.dynofront_update_depths(self.h, n, _p(k), _p(lab), float(max_background_depth), float(max_object_depth), _p(d), _p(v),
                                                  C.byref(ni), C.byref(no), C.byref(ms)))
        self.last_ms = ms.value
        return d, v, ni.value, no.value

    def back_project(self, kp, depth, usable, calib5, baseline=0.0, rgbd=False, right_u=None, X_world=None, capacity=None):
        """fillOutputPacketWithTracks per feature: returns a dict with index [m], point [m][3], stereo [m][3] (uL, uR, v),
        outlier [n] and m (the first min(m, capacity) rows are filled when a capacity is given)"""
        k = np.ascontiguousarray(kp, dtype=np.float64).reshape(-1, 2); n = k.shape[0]
        d = np.ascontiguousarray(depth, dtype=np.float64); u = np.ascontiguousarray(usable, dtype=np.uint8)
        r = None if right_u is None else np.ascontiguousarray(right_u, dtype=np.float64)
        X = None if X_world is None else np.ascontiguousarray(X_world, dtype=np.float64).reshape(12)
        cal = np.ascontiguousarray(calib5, dtype=np.float64).reshape(5)
        cap = int(n if capacity is None else capacity)
        idx = np.zeros(max(cap, 1), np.int32); pt = np.zeros((max(cap, 1), 3)); st = np.zeros((max(cap, 1), 3)); out = np.zeros(n, np.uint8)
        m = C.c_int32(); ms = C.c_float()
        self._ck(self.lib.dynofront_back_project(self.h, n, _p(k), _p(d), _p(u), _p(r), _p(cal), float(baseline), int(bool(rgbd)), _p(X), cap, _p(idx),
                                                 _p(pt), _p(st), _p(out), C.byref(m), C.byref(ms)))
        self.last_ms = ms.value
        s = min(m.value, cap)
        return dict(index=idx[:s], point=pt[:s], stereo=st[:s], outlier=out, m=m.value)

    def dense_cloud(self, calib5, max_background_depth=200.0, max_object_depth=30.0):
        """Frame::projectToDenseCloud on the resident depth / motion mask / boundary mask: (xyz f32[H][W][3], rgb u8[H][W][3],
        label u32[H][W], valid u8[H][W], n_valid)"""
        cal = np.ascontiguousarray(calib5, dtype=np.float64).reshape(5)
        xyz = np.zeros((self.H, self.W, 3), np.float32); rgb = np.zeros((self.H, self.W, 3), np.uint8)
        lab = np.zeros((self.H, self.W), np.uint32); val = np.zeros((self.H, self.W), np.uint8); nv = C.c_int32(); ms = C.c_float()
        self._ck(self.lib.dynofront_dense_cloud(self.h, _p(cal), float(max_background_depth), float(max_object_depth), _p(xyz), _p(rgb), _p(lab), _p(val),
                                                C.byref(nv), C.byref(ms)))
        self.last_ms = ms.value
        return xyz, rgb, lab, val, nv.value

    def klt_last_min_eig(self, n):
        out = np.zeros((n, 2), np.float32)
        self._ck(self.lib.dynofront_klt_last_min_eig(self.h, n, _p(out)))
        return out

    def track_static_flow(self, prev_pred_kp, prev_age, prev_usable, det_xy, cell_size, max_features, next_tracklet_id):
        """ExternalFlowFeatureTracker::trackStatic on the frame given to set_frame.  Returns a dict of per-feature arrays."""
        kp = np.ascontiguousarray(prev_pred_kp, dtype=np.float64).reshape(-1, 2); n = kp.shape[0]
        age = np.ascontiguousarray(prev_age, dtype=np.int32); use = np.ascontiguousarray(prev_usable, dtype=np.uint8)
        det = np.ascontiguousarray(det_xy, dtype=np.int32).reshape(-1, 2); m = det.shape[0]
        acc = np.zeros(n, np.uint8); fl = np.zeros((n, 2)); pk = np.zeros((n, 2)); oage = np.zeros(n, np.int32)
        dacc = np.zeros(m, np.uint8); dfl = np.zeros((m, 2)); dpk = np.zeros((m, 2)); dtid = np.zeros(m, np.int64)
        nid = C.c_int64(int(next_tracklet_id)); nt = C.c_int32(); nd = C.c_int32()
        self._ck(self.lib.dynofront_track_static_flow(self.h, n, _p(kp), _p(age), _p(use), m, _p(det), int(cell_size), int(max_features), C.byref(nid),
                                                      _p(acc), _p(fl), _p(pk), _p(oage), _p(dacc), _p(dfl), _p(dpk), _p(dtid), C.byref(nt), C.byref(nd)))
        return dict(acc=acc, flow=fl, pred=pk, age=oage, det_acc=dacc, det_flow=dfl, det_pred=dpk, det_tracklet=dtid,
                    next_tracklet_id=nid.value, n_tracked=nt.value, n_detected=nd.value)

    def pyramid_level(self, which, level):
        w = C.c_int32(); h = C.c_int32()
        self._ck(self.lib.dynofront_get_pyramid_level(self.h, which, level, C.byref(w), C.byref(h), None, None))
        img = np.zeros((h.value, w.value), np.uint8); der = np.zeros((h.value, w.value, 2), np.int16)
        self._ck(self.lib.dynofront_get_pyramid_level(self.h, which, level, C.byref(w), C.byref(h), _p(img), _p(der)))
        return img, der
