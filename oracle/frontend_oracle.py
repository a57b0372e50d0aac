"""CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT) for the front-end rows a13 / a14 of SURVEY.md section 8.

Literal Python restatement (plain loops, the reference's iteration order) of
  * FeatureTracker::trackDynamic      dynosam/src/frontend/vision/FeatureTracker.cc:339-498
  * FeatureTracker::sampleDynamic     (candidate scan)  :864-953
  * FeatureTracker::propogateMask     :1212-1359
  * ExternalFlowFeatureTracker::trackStatic / constructStaticFeature   StaticFeatureTracker.cc:70-220
  * KltFeatureTracker::trackPoints forward-backward filter and post checks   StaticFeatureTracker.cc:486-592
  * FeatureTrackerBase::isWithinShrunkenImage  FeatureTrackerBase.cc:313-326,  Camera::isKeypointContained Camera.cc:71-74,
    functional_keypoint::u/v int truncation  dynosam_cv/include/dynosam_cv/Feature.hpp:46-55
cv::circle is the real OpenCV routine (cv2.circle), and the pyramidal KLT oracle is cv2.calcOpticalFlowPyrLK itself
(OpenCV 4.13 here; the reference's docker pins 4.x -- SURVEY.md Appendix B).  "Parity unpinned" by the reference:
it has no front-end tracking tests (SURVEY.md section 4); these functions are pinned only by being literal.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

BACKGROUND = 0


@dataclass
class TrackParams:
    max_dynamic_feature_age: int = 20          # params/FrontendParams.yaml:66
    min_distance: int = 2                      # min_distance_btw_tracked_and_detected_dynamic_features, :65
    shrink_row: int = 0
    shrink_col: int = 0


def saturate_u8(label) -> int:
    """cv::Scalar(label) drawn into a CV_8U image: saturate_cast<uchar>"""
    return min(max(int(label), 0), 255)


def libstdcxx_sort(seq, comp, heap_ranges=None):
    """std::sort(first, last, comp) of libstdc++ (<bits/stl_algo.h>), element moves and all: __introsort_loop (threshold 16,
    depth limit 2 floor(log2 n), __move_median_to_first of (first + 1, mid, last - 1), __unguarded_partition, __partial_sort
    = make_heap + sort_heap at the depth limit), then __final_insertion_sort.  Not stable: where comp ties, the result
    depends on all of these steps.  Returns a sorted copy; heap_ranges (a list), when given, receives the (first, last) of
    every range heap-sorted at the depth limit."""
    a = list(seq)
    n = len(a)

    def adjust_heap(f, hole, ln, v):
        top = hole; child = hole
        while child < (ln - 1)//2:
            child = 2*(child + 1)
            if comp(a[f + child], a[f + child - 1]):
                child -= 1
            a[f + hole] = a[f + child]; hole = child
        if ln % 2 == 0 and child == (ln - 2)//2:
            child = 2*(child + 1); a[f + hole] = a[f + child - 1]; hole = child - 1
        parent = (hole - 1)//2
        while hole > top and comp(a[f + parent], v):
            a[f + hole] = a[f + parent]; hole = parent; parent = (hole - 1)//2
        a[f + hole] = v

    def heap_sort(f, ln):
        if ln >= 2:
            for parent in range((ln - 2)//2, -1, -1):
                adjust_heap(f, parent, ln, a[f + parent])
        for last in range(ln - 1, 0, -1):
            v = a[f + last]; a[f + last] = a[f]; adjust_heap(f, 0, last, v)

    def partition_pivot(first, last):
        x, y, z = first + 1, first + (last - first)//2, last - 1
        if comp(a[x], a[y]):
            m = y if comp(a[y], a[z]) else (z if comp(a[x], a[z]) else x)
        else:
            m = x if comp(a[x], a[z]) else (z if comp(a[y], a[z]) else y)
        a[first], a[m] = a[m], a[first]
        i, j = first + 1, last
        while True:
            while comp(a[i], a[first]):
                i += 1
            j -= 1
            while comp(a[first], a[j]):
                j -= 1
            if not i < j:
                return i
            a[i], a[j] = a[j], a[i]
            i += 1

    def introsort_loop(first, last, depth):
        while last - first > 16:
            if depth == 0:
                if heap_ranges is not None:
                    heap_ranges.append((first, last))
                heap_sort(first, last - first)
                return
            depth -= 1
            cut = partition_pivot(first, last)
            introsort_loop(cut, last, depth)
            last = cut

    if n > 1:
        introsort_loop(0, n, 2*(n.bit_length() - 1))
        for i in range(1, n):                            # the guarded and unguarded insertion sorts move alike
            v = a[i]
            while i > 0 and comp(v, a[i - 1]):
                a[i] = a[i - 1]; i -= 1
            a[i] = v
    return a


def within_shrunken(kp, rows, cols, prm: TrackParams) -> bool:
    pc = int(kp[0]); pr = int(kp[1])          # C++ static_cast<int>: truncation toward zero
    return pr > prm.shrink_row and pr < rows - prm.shrink_row and pc > prm.shrink_col and pc < cols - prm.shrink_col


def keypoint_contained(kp, rows, cols) -> bool:
    return kp[0] >= 0.0 and kp[0] < cols and kp[1] >= 0.0 and kp[1] < rows


def track_dynamic(prev_pred_kp, prev_label, prev_age, prev_tracklet, flow, motion_mask, detection_mask, prm: TrackParams,
                  next_tracklet_id: int):
    """Returns (accepted[n], pred_kp[n,2], flow[n,2], age[n], tracklet[n], label[n], next_tracklet_id,
    detection_mask_out, tracking_mask_out).  Rows of rejected features are zero."""
    import cv2
    rows, cols = motion_mask.shape
    n = len(prev_label)
    det = detection_mask.copy() if detection_mask is not None else np.full((rows, cols), 255, np.uint8)
    trk = np.zeros((rows, cols), np.uint8)
    acc = np.zeros(n, np.uint8); pk = np.zeros((n, 2)); fl = np.zeros((n, 2))
    age = np.zeros(n, np.int32); tid = np.zeros(n, np.int64); lab = np.zeros(n, np.int32)
    for i in range(n):
        kp = prev_pred_kp[i]
        x = int(kp[0]); y = int(kp[1])
        predicted_label = int(motion_mask[y, x])
        if det[y, x] == 0:
            continue
        previous_label = int(prev_label[i])
        if keypoint_contained(kp, rows, cols) and predicted_label != BACKGROUND and predicted_label == previous_label:
            new_age = int(prev_age[i]) + 1
            fx = float(flow[y, x, 0]); fy = float(flow[y, x, 1])
            predicted = (kp[0] + fx, kp[1] + fy)
            if not within_shrunken(predicted, rows, cols, prm):
                continue
            if fx == 0 or fy == 0:
                continue
            t = int(prev_tracklet[i])
            if new_age > prm.max_dynamic_feature_age:
                t = next_tracklet_id; next_tracklet_id += 1
                new_age = 0
            acc[i] = 1; pk[i] = predicted; fl[i] = (fx, fy); age[i] = new_age; tid[i] = t; lab[i] = predicted_label
            cv2.circle(det, (x, y), prm.min_distance, 0, cv2.FILLED)
            cv2.circle(trk, (x, y), prm.min_distance, saturate_u8(predicted_label), cv2.FILLED)
    return acc, pk, fl, age, tid, lab, next_tracklet_id, det, trk


def sample_dynamic_candidates(flow, motion_mask, detection_mask, objects_to_sample, prm: TrackParams):
    """Per object: sorted linear pixel indices of the sampling candidates, and the zero-flow count.
    (The reference fills the per-object lists from a tbb::parallel_for over rows, so only the SET is defined.)"""
    rows, cols = motion_mask.shape
    cand = {int(o): [] for o in objects_to_sample}
    zero = {int(o): 0 for o in objects_to_sample}
    for i in range(rows):
        for j in range(cols):
            if detection_mask[i, j] == 0:
                continue
            o = int(motion_mask[i, j])
            if o not in cand or o == BACKGROUND:
                continue
            fx = float(flow[i, j, 0]); fy = float(flow[i, j, 1])
            if fx == 0 or fy == 0:
                zero[o] += 1
                continue
            if within_shrunken((float(j), float(i)), rows, cols, prm):
                cand[o].append(i*cols + j)
    return cand, zero


def propagate_mask(prev_pred_kp, prev_label, prev_mask, prev_flow, current_mask, prm: TrackParams, min_votes=150):
    """Returns the updated current mask (copy)."""
    cur = current_mask.copy()
    rows, cols = prev_mask.shape
    labels = sorted(set(int(l) for l in prev_label))
    for lab in labels:
        temp = []
        for i in range(len(prev_label)):
            if int(prev_label[i]) != lab:
                continue
            u = int(prev_pred_kp[i][0]); v = int(prev_pred_kp[i][1])
            if u < cols and u > 0 and v < rows and v > 0:
                temp.append(int(cur[v, u]))
        if not temp or len(temp) < min_votes:          # no vote: nothing to sort (the device's flag stays 0)
            continue
        counts = {}
        for k in temp:
            counts[k] = counts.get(k, -1) + 1      # first occurrence counts 0 (reference quirk)
        pairs = [(k, counts[k]) for k in sorted(counts)]                  # std::map order
        best = libstdcxx_sort(pairs, lambda a, b: a[1] > b[1])[0][0]
        if best != 0:
            continue
        for j in range(rows):
            for k in range(cols):
                if int(prev_mask[j, k]) != lab:
                    continue
                fx = float(prev_flow[j, k, 0]); fy = float(prev_flow[j, k, 1])
                if fx == 0 or fy == 0:
                    continue
                p = (k + fx, j + fy)
                if not within_shrunken(p, rows, cols, prm):
                    continue
                if p[0] < cols and p[0] > 0 and p[1] < rows and p[1] > 0:
                    cur[int(p[1]), int(p[0])] = lab
    return cur


def klt_track(prev_gray, cur_gray, prev_pts, win=21, max_level=3, max_count=30, eps=0.03, initial=None, min_eig=1e-4):
    """cv::calcOpticalFlowPyrLK as the reference calls it (StaticFeatureTracker.cc:486-489)."""
    import cv2
    p0 = np.ascontiguousarray(prev_pts, dtype=np.float32).reshape(-1, 1, 2)
    flags = 0
    p1 = None
    if initial is not None:
        p1 = np.ascontiguousarray(initial, dtype=np.float32).reshape(-1, 1, 2).copy(); flags = cv2.OPTFLOW_USE_INITIAL_FLOW
    nxt, st, err = cv2.calcOpticalFlowPyrLK(prev_gray, cur_gray, p0, p1, winSize=(win, win), maxLevel=max_level,
                                            criteria=(cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, max_count, eps),
                                            flags=flags, minEigThreshold=min_eig)
    return nxt.reshape(-1, 2), st.reshape(-1), err.reshape(-1)


def _construct_static_feature(kp, flow, motion_mask, rows, cols):
    """ExternalFlowFeatureTracker::constructStaticFeature (StaticFeatureTracker.cc:172-218): (flow, predicted kp) or None."""
    x = int(kp[0]); y = int(kp[1])
    if int(motion_mask[y, x]) != BACKGROUND:
        return None
    fx = float(flow[y, x, 0]); fy = float(flow[y, x, 1])
    if not (fx != 0 and fy != 0):
        return None
    pred = (kp[0] + fx, kp[1] + fy)
    if not keypoint_contained(pred, rows, cols):
        return None
    return (fx, fy), pred


def track_static_flow(prev_pred_kp, prev_age, prev_usable, det_xy, flow, motion_mask, cell_size, max_features, next_tracklet_id):
    """ExternalFlowFeatureTracker::trackStatic (StaticFeatureTracker.cc:70-170), literal loops.  The detections are the
    (integer) key-points the ORB extractor returned, in its order."""
    import math
    rows, cols = motion_mask.shape
    ncols = math.ceil(cols/cell_size); nrows = math.ceil(rows/cell_size)
    occ = [False]*(ncols*nrows)
    cell_of = lambda kp: int(math.floor(kp[1]/cell_size))*ncols + int(math.floor(kp[0]/cell_size))
    n = len(prev_age); m = len(det_xy)
    acc = np.zeros(n, np.uint8); fl = np.zeros((n, 2)); pk = np.zeros((n, 2)); age = np.zeros(n, np.int32)
    dacc = np.zeros(m, np.uint8); dfl = np.zeros((m, 2)); dpk = np.zeros((m, 2)); dtid = np.zeros(m, np.int64)
    count = 0
    for i in range(n):
        kp = (float(prev_pred_kp[i][0]), float(prev_pred_kp[i][1]))
        if not keypoint_contained(kp, rows, cols):
            continue
        x = int(kp[0]); y = int(kp[1])
        c = cell_of(kp)
        label = int(motion_mask[y, x])
        if occ[c]:
            continue
        if prev_usable[i] and label == BACKGROUND:
            f = _construct_static_feature(kp, flow, motion_mask, rows, cols)
            if f is not None:
                acc[i] = 1; fl[i] = f[0]; pk[i] = f[1]; age[i] = int(prev_age[i]) + 1
                occ[c] = True; count += 1
    n_tracked = count
    if count < max_features:
        for j in range(m):
            if count >= max_features:
                break
            x = int(det_xy[j][0]); y = int(det_xy[j][1])
            if int(motion_mask[y, x]) != BACKGROUND:
                continue
            kp = (float(x), float(y))
            c = cell_of(kp)
            if not occ[c]:
                f = _construct_static_feature(kp, flow, motion_mask, rows, cols)
                if f is not None:
                    dacc[j] = 1; dfl[j] = f[0]; dpk[j] = f[1]; dtid[j] = next_tracklet_id
                    next_tracklet_id += 1; occ[c] = True; count += 1
    return dict(acc=acc, flow=fl, pred=pk, age=age, det_acc=dacc, det_flow=dfl, det_pred=dpk, det_tracklet=dtid,
                next_tracklet_id=next_tracklet_id, n_tracked=n_tracked, n_detected=count - n_tracked)


def klt_track_fb(prev_gray, cur_gray, prev_pts, motion_mask=None, prev_age=None, max_feature_track_age=25, prm: TrackParams = None,
                 win=21, max_level=3, max_count=30, eps=0.03, initial=None):
    """KltFeatureTracker::trackPoints (StaticFeatureTracker.cc:486-534, 575-592 / 628-646): cv2 forward (retry without the
    initial flow below 10 successes), cv2 backward (21x21, maxLevel 5, default criteria), round trip <= 0.5 px in float,
    then the per-point label / border / age checks.  Returns (next, status, back, keep)."""
    import cv2
    prm = prm or TrackParams()
    p0 = np.ascontiguousarray(prev_pts, dtype=np.float32).reshape(-1, 2)
    nxt, st, _ = klt_track(prev_gray, cur_gray, p0, win, max_level, max_count, eps, initial)
    if initial is not None and int(st.sum()) < 10:
        nxt, st, _ = klt_track(prev_gray, cur_gray, p0, win, max_level, max_count, eps, None)
    back, stb, _ = cv2.calcOpticalFlowPyrLK(cur_gray, prev_gray, nxt.reshape(-1, 1, 2).astype(np.float32), None, winSize=(21, 21), maxLevel=5)
    back = back.reshape(-1, 2); stb = stb.reshape(-1)
    d = p0 - back
    dist = np.sqrt((d[:, 0]*d[:, 0] + d[:, 1]*d[:, 1]).astype(np.float32))
    status = ((st != 0) & (stb != 0) & (dist <= np.float32(0.5))).astype(np.uint8)
    keep = None
    if prev_age is not None:
        rows, cols = motion_mask.shape
        keep = np.zeros(len(status), np.uint8)
        for i in range(len(status)):
            if not status[i]:
                continue
            kp = (float(nxt[i, 0]), float(nxt[i, 1]))
            x = int(kp[0]); y = int(kp[1])
            if not (keypoint_contained(kp, rows, cols) and within_shrunken(kp, rows, cols, prm)):
                continue
            if int(motion_mask[y, x]) != BACKGROUND:
                continue
            if int(prev_age[i]) + 1 > max_feature_track_age:
                continue
            keep[i] = 1
    return nxt, status, back, keep


def stereo_track(left_gray, right_gray, left_pts, fx, baseline):
    """FeatureTracker::stereoTrack (FeatureTracker.cc:194-337) without the fundamental-matrix RANSAC: cv2 LK left -> right
    (21x21, maxLevel 5, default criteria), then disparity = uL - uR, rejected when <= 1 or uR < 0, depth = fx b / disparity."""
    import cv2
    p0 = np.ascontiguousarray(left_pts, dtype=np.float32).reshape(-1, 1, 2)
    rp, st, _ = cv2.calcOpticalFlowPyrLK(left_gray, right_gray, p0, None, winSize=(21, 21), maxLevel=5)
    rp = rp.reshape(-1, 2); st = st.reshape(-1)
    n = len(st); depth = np.zeros(n); valid = np.zeros(n, np.uint8)
    for i in range(n):
        if not st[i]:
            continue
        uL = float(p0[i, 0, 0]); uR = float(rp[i, 0])
        disparity = uL - uR
        if disparity <= 1.0 or rp[i, 0] < np.float32(0.0):
            continue
        valid[i] = 1; depth[i] = fx*baseline/disparity
    return rp, st, depth, valid
