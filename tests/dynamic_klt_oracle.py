"""CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT) for FeatureTracker::trackDynamicKLT on the device.

Literal Python restatement of
  * FeatureTracker::trackDynamicKLT   dynosam/src/frontend/vision/FeatureTracker.cc:596-862 (after the LK call, whose
    output is an input here: the device's own LK result, so that LK rounding is kept apart)
  * FeatureTracker::requiresSampling  FeatureTracker.cc:1018-1149
  * utils::calculateIoU               dynosam_common/src/utils/OpenCVUtils.cc:87-102 (cv::Rect operator& of OpenCV 4)
with cv2.circle on a copy of the mask, cv2.goodFeaturesToTrack per object, selection_oracle.anms_range_tree and
cv2.boundingRect.  Where the reference is undefined or unordered the device's definitions are restated: an LK point whose
truncated pixel is outside the image is dropped and counted apart, and the new features come object by object in the given
objects order.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

import selection_oracle as SO

TRACKED, MASKED, REJECTED, OUTSIDE, LOST = 1, 2, 3, 4, 5         # dynofront_track_dynamic_klt per-feature state
STATUS_FIELDS = ["object_id", "exists", "num_previous_track", "num_track", "num_outside_shrunken_image", "num_tracked_with_different_label",
                 "num_tracked_with_background_label", "object_new", "object_resampled", "sampled", "num_sampled"]


@dataclass
class Params:
    max_dynamic_feature_age: int = 20
    min_distance: int = 2
    shrink_row: int = 0
    shrink_col: int = 0
    max_features: int = 200
    quality_level: float = 0.01
    age_buffer: int = 3
    min_tracks: int = 20
    min_iou: float = 0.1


@dataclass
class PerObjectStatus:
    object_id: int
    num_previous_track: int = 0
    num_track: int = 0
    num_sampled: int = 0
    num_outside_shrunken_image: int = 0
    num_tracked_with_different_label: int = 0
    num_tracked_with_background_label: int = 0
    object_new: bool = False
    object_resampled: bool = False
    reasons: list = field(default_factory=list)


def rect_and(a, b):
    """cv::Rect operator&= (OpenCV 4): an empty operand or no overlap gives Rect()"""
    ax, ay, aw, ah = a; bx, by, bw, bh = b
    if aw <= 0 or ah <= 0 or bw <= 0 or bh <= 0:
        return (0, 0, 0, 0)
    xmin, xmax = (a, b) if ax < bx else (b, a)
    ymin, ymax = (a, b) if ay < by else (b, a)
    if xmax[0] - xmin[0] >= xmin[2] or ymax[1] - ymin[1] >= ymin[3]:
        return (0, 0, 0, 0)
    return (xmax[0], ymax[1], min(xmin[2] - (xmax[0] - xmin[0]), xmax[2]), min(ymin[3] - (ymax[1] - ymin[1]), ymax[3]))


def calculate_iou(a, b):
    inter = rect_and(a, b)
    ia = float(inter[2]*inter[3])
    union = float(a[2]*a[3] + b[2]*b[3]) - ia
    return 0.0 if union == 0 else ia/union


def bounding_rect(pts):
    """cv::boundingRect of float points (as toOpenCV gives them)"""
    import cv2
    return tuple(int(v) for v in cv2.boundingRect(np.ascontiguousarray(np.asarray(pts, np.float32).reshape(-1, 1, 2))))


def _shrunken(kx, ky, rows, cols, prm):
    u, v = int(kx), int(ky)
    return prm.shrink_row < v < rows - prm.shrink_row and prm.shrink_col < u < cols - prm.shrink_col


def gftt(mono, motion_mask, det, object_id, prm):
    """goodFeaturesToTrack(mono, max_features, quality, min_distance, (motion_mask == id) & detection_mask_impl): (x, y) int"""
    import cv2
    obj = np.where(motion_mask == object_id, 255, 0).astype(np.uint8)
    combined = cv2.bitwise_and(obj, det)
    pts = cv2.goodFeaturesToTrack(mono, prm.max_features, prm.quality_level, prm.min_distance, mask=combined)
    return [] if pts is None else [(int(x), int(y)) for x, y in pts.reshape(-1, 2)]


def gftt_decomposed(eig, motion_mask, det, objects, prm):
    """The device's decomposition: one pass of raw 3x3 local maxima of the eigen image (1-px border excluded), then per object
    the masked maximum, the threshold (float)(maxVal * quality), the candidates above it in (value desc, address desc) order
    and the strict minDistance greedy with the maxCorners stop."""
    H, W = eig.shape
    pad = np.pad(eig, 1, constant_values=-np.inf)
    dil = np.max([pad[j:j + H, i:i + W] for j in range(3) for i in range(3)], axis=0)
    locmax = eig == dil
    locmax[0] = locmax[-1] = False; locmax[:, 0] = locmax[:, -1] = False
    out = {}
    for oid in objects:
        m = (motion_mask == oid) & (det != 0)
        mx = float(eig[m].max()) if m.any() else 0.0
        thr = np.float32(mx*prm.quality_level)
        ys, xs = np.nonzero(m & locmax & (eig > thr))
        v = eig[ys, xs]; addr = ys.astype(np.int64)*W + xs
        o = np.lexsort((-addr, -v)); ys, xs = ys[o], xs[o]
        kept = []
        md2 = prm.min_distance*prm.min_distance
        for x, y in zip(xs.tolist(), ys.tolist()):
            if all((x - a)**2 + (y - b)**2 >= md2 for a, b in kept):
                kept.append((x, y))
                if len(kept) == prm.max_features:
                    break
        out[int(oid)] = kept
    return out


def track_dynamic_klt(mono, motion_mask, boundary_mask, prev_kp, prev_label, prev_age, prev_tracklet, lk_pts, lk_status, objects, inner_bb,
                      prm: Params, next_tracklet_id):
    """Returns a dict with the per-feature state / measured_flow, the output features (keypoint, age, tracklet, label, source),
    the status rows over [0] + objects (STATUS_FIELDS), n_outside_image, next_tracklet_id, both masks and, per object, the
    sampling reasons ('new', 'old', 'few', 'iou') or 'skipped'."""
    import cv2
    rows, cols = motion_mask.shape
    det = boundary_mask.copy() if boundary_mask is not None else np.full((rows, cols), 255, np.uint8)
    trk = np.zeros((rows, cols), np.uint8)
    prev_kp = np.asarray(prev_kp, np.float32).reshape(-1, 2); lk_pts = np.asarray(lk_pts, np.float32).reshape(-1, 2)
    n = len(prev_kp)
    info = {}

    def status(oid):
        return info.setdefault(int(oid), PerObjectStatus(int(oid)))

    state = np.full(n, LOST, np.uint8); flow = np.zeros((n, 2))
    tracks = {}                                              # gtsam::FastMap<ObjectId, FeatureContainer>: iterated in key order
    n_outside = 0
    r = prm.min_distance
    for i in range(n):
        if not lk_status[i]:
            continue
        kx, ky = float(lk_pts[i, 0]), float(lk_pts[i, 1])
        x, y = int(kx), int(ky)                              # functional_keypoint::u / v
        if not (0 <= x < cols and 0 <= y < rows):
            state[i] = OUTSIDE; n_outside += 1
            continue
        predicted = int(motion_mask[y, x])
        if det[y, x] == 0:
            state[i] = MASKED
            continue
        previous = int(prev_label[i])
        st = status(predicted)
        st.num_previous_track += 1
        if predicted == 0:
            st.num_tracked_with_background_label += 1
        if predicted != previous:
            st.num_tracked_with_different_label += 1
        state[i] = REJECTED
        if 0.0 <= kx < cols and 0.0 <= ky < rows and predicted != 0 and predicted == previous:
            if not _shrunken(kx, ky, rows, cols, prm):
                st.num_outside_shrunken_image += 1
                continue
            age = int(prev_age[i]) + 1
            if age > prm.max_dynamic_feature_age:
                continue
            flow[i] = (kx - float(prev_kp[i, 0]), ky - float(prev_kp[i, 1]))
            tracks.setdefault(predicted, []).append(dict(kp=(kx, ky), age=age, tracklet=int(prev_tracklet[i]), label=predicted, source=i))
            st.num_track += 1
            cv2.circle(det, (x, y), r, 0, cv2.FILLED)
            cv2.circle(trk, (x, y), r, int(min(predicted, 255)), cv2.FILLED)
            state[i] = TRACKED
    features = [f for oid in sorted(tracks) for f in tracks[oid]]

    # requiresSampling
    expiry = prm.max_dynamic_feature_age - max(3, prm.age_buffer)
    assert expiry > 0
    to_sample, reasons = [], {}
    for j, oid in enumerate(int(o) for o in objects):
        if oid in info:
            st = info[oid]
            if oid not in tracks:
                reasons[oid] = ["skipped"]
                continue
            tr = tracks[oid]
            assert st.num_track == len(tr)
            geriatric = sum(1 for f in tr if f["age"] > expiry)
            why = []
            if geriatric/st.num_track > 0.8:
                why.append("old")
            if st.num_track < prm.min_tracks:
                why.append("few")
            if calculate_iou(tuple(int(v) for v in inner_bb[j]), bounding_rect([f["kp"] for f in tr])) < prm.min_iou:
                why.append("iou")
            reasons[oid] = why
            if why:
                to_sample.append(oid); st.object_resampled = True
        else:
            to_sample.append(oid); reasons[oid] = ["new"]
            st = status(oid); st.object_new = True; st.object_resampled = True

    # re-sampling: goodFeaturesToTrack, range-tree ANMS, the new features
    for oid in to_sample:
        pts = gftt(mono, motion_mask, det, oid, prm)
        k = max(prm.max_features - info[oid].num_track, 0)
        sel = SO.anms_range_tree(pts, k, np.float32(0.01), cols, rows) if pts else []
        info[oid].num_sampled = len(sel)
        for s in sel:
            kx, ky = float(pts[s][0]), float(pts[s][1])
            assert motion_mask[int(ky), int(kx)] == oid
            if not _shrunken(kx, ky, rows, cols, prm):
                continue
            features.append(dict(kp=(kx, ky), age=0, tracklet=next_tracklet_id, label=oid, source=-1)); next_tracklet_id += 1

    srows = []
    for oid in [0] + [int(o) for o in objects]:
        st = info.get(oid)
        srows.append([oid, int(st is not None)] + ([st.num_previous_track, st.num_track, st.num_outside_shrunken_image,
                                                    st.num_tracked_with_different_label, st.num_tracked_with_background_label,
                                                    int(st.object_new), int(st.object_resampled), int(oid in to_sample), st.num_sampled]
                                                   if st is not None else [0]*9))
    srows = np.array(srows, np.int32).reshape(-1, len(STATUS_FIELDS))
    return dict(state=state, measured_flow=flow,
                keypoint=np.array([f["kp"] for f in features], np.float64).reshape(-1, 2), age=np.array([f["age"] for f in features], np.int32),
                tracklet=np.array([f["tracklet"] for f in features], np.int64), label=np.array([f["label"] for f in features], np.int32),
                source=np.array([f["source"] for f in features], np.int32), status={f: srows[:, c] for c, f in enumerate(STATUS_FIELDS)},
                n_outside_image=n_outside, next_tracklet_id=next_tracklet_id, detection_mask=det, tracking_mask=trk, reasons=reasons)


def hand_built_frame(shift=4):
    """A 640 x 480 frame pair in which every sampling path of requiresSampling is taken, for the CPU tests (with the exact LK
    result: every point moves by -shift in x) and the device (whose LK follows the shift).  cur = prev moved left by `shift` px.
    Returns prev_gray, cur_gray, motion_mask (current frame), previous features (kp [n][2] float32, label, age, tracklet),
    objects, inner_bb and the LK points of an exact tracker.
      object 1: no feature lands on it: new;
      object 2: its only visitor lands there with previous label 3: a row but no track, skipped;
      object 3: 25 tracks, 21 of them older than the expiry age: geriatric;
      object 4: 5 young tracks: too few; plus a feature 1 px from an earlier accepted one (masked, uncounted);
      object 5: 30 young tracks in a 15 px patch of a 200 px box: small IoU;
      object 6: 210 young tracks in a small patch: small IoU with K = 0;
      object 7: 30 young tracks spread over it: not sampled;
      plus a point that the LK carries out of the image and one that leaves the shrunken image test untouched (shrink 0)."""
    import cv2
    Hh, Ww = 480, 640
    rng = np.random.default_rng(3)
    big = cv2.GaussianBlur(rng.integers(0, 256, (Hh, Ww + shift)).astype(np.uint8), (0, 0), 1.5)
    prev_gray = np.ascontiguousarray(big[:, :Ww]); cur_gray = np.ascontiguousarray(big[:, shift:shift + Ww])
    mask = np.zeros((Hh, Ww), np.int32)
    boxes = {1: (20, 20, 100, 80), 2: (140, 20, 80, 80), 3: (240, 20, 120, 100), 4: (380, 20, 120, 100), 5: (20, 200, 200, 150),
             6: (240, 200, 200, 180), 7: (460, 200, 160, 150)}
    for oid, (x, y, w, h) in boxes.items():
        mask[y:y + h, x:x + w] = oid
    kp, lab, age = [], [], []

    def add(pts, label, a):
        for x, y in pts:
            kp.append((x + 0.25, y + 0.25)); lab.append(label); age.append(a)

    add([(150, 50)], 3, 2)                                                            # object 2: wrong previous label
    g3 = [(250 + 20*(i % 5), 30 + 18*(i//5)) for i in range(25)]
    add(g3[:21], 3, 17); add(g3[21:], 3, 5)                                           # object 3: 21/25 reach age 18 > 17
    add([(390 + 25*i, 40 + 15*i) for i in range(5)], 4, 1)                          # object 4: 5 tracks
    add([(391, 40)], 4, 1)                                                            # 1 px right of the first: masked
    add([(100 + 3*(i % 6), 280 + 3*(i//6)) for i in range(30)], 5, 0)                 # object 5: 15 x 15 patch
    add([(300 + 3*(i % 15), 260 + 3*(i//15)) for i in range(210)], 6, 0)              # object 6: 210 tracks, 45 x 42 patch
    add([(470 + 30*(i % 5), 210 + 25*(i//5)) for i in range(30)], 7, 0)               # object 7: spread
    add([(-6, 300)], 5, 0)                                                            # carried out of the image
    add([(5, 5)], 1, 20)                                                              # background at the landing pixel
    kp = np.array(kp, np.float32); kp[:, 0] += shift                                   # previous positions: current + shift
    n = len(kp)
    lk = kp.copy(); lk[:, 0] -= shift
    objects = [1, 2, 3, 4, 5, 6, 7]
    inner = np.array([(x + 2, y + 2, w - 4, h - 4) for x, y, w, h in (boxes[o] for o in objects)], np.int32)
    return (prev_gray, cur_gray, mask, kp, np.array(lab, np.int32), np.array(age, np.int32), np.arange(100, 100 + n, dtype=np.int64),
            objects, inner, lk)
