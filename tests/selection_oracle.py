"""CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT) for feature selection on the device: the range-tree ANMS and
FeatureTracker::sampleDynamic after its candidate scan.

Literal Python restatement of
  * AdaptiveNonMaximumSuppression::suppressNonMax   dynosam/src/frontend/anms/NonMaximumSupression.cc:33-116
    (cv::sortIdx of the int responses, SORT_DESCENDING; both call sites pass responses that truncate to 0)
  * anms::RangeTree                                 dynosam/src/frontend/anms/anms.cc:278-362
    (an inclusive brute-force square search stands in for the range tree, whose search is inclusive on both axes)
  * FeatureTracker::sampleDynamic                    dynosam/src/frontend/vision/FeatureTracker.cc:864-1015
"""
from __future__ import annotations

import math

import numpy as np


def sort_idx_equal_keys(n):
    """cv::sortIdx(all-equal int keys, SORT_DESCENDING): libstdc++ introsort on equal keys swaps first with the middle
    element (__move_median_to_first, every comparison false), reverses the rest (__unguarded_partition), recurses right and
    loops left while more than 16 elements remain; the insertion sort then moves nothing and the result is reversed."""
    a = list(range(n))

    def introsort(lo, hi, depth):
        while hi - lo > 16:
            if depth == 0:
                raise RuntimeError("heapsort branch reached")
            depth -= 1
            mid = lo + (hi - lo)//2
            a[lo], a[mid] = a[mid], a[lo]
            i, j = lo + 1, hi
            while True:
                j -= 1
                if not i < j:
                    break
                a[i], a[j] = a[j], a[i]
                i += 1
            introsort(i, hi, depth)
            hi = i

    if n > 1:
        introsort(0, n, 2*int(math.floor(math.log2(n))))
    return a[::-1]


def _c_round(x):
    """C round(): half away from zero (exact for doubles)."""
    ax = abs(x); f = math.floor(ax)
    r = f + 1 if ax - f >= 0.5 else f
    return float(r if x >= 0 else -r)


def _c_div(a, b):
    """C integer division: truncation toward zero."""
    q = abs(a)//abs(b)
    return q if (a >= 0) == (b > 0) else -q


def anms_range_tree(xy, k_needed, tolerance, cols, rows):
    """suppressNonMax(RangeTree) on integer key-points xy[n][2] (col, row) of response 0.  Returns the indices of the
    selected key-points in selection order.  k_needed = 0 selects nothing and k_needed = 1 the first point in visiting
    order (the reference computes inf / NaN bounds there)."""
    n = len(xy)
    if n == 0:
        return []
    order = sort_idx_equal_keys(n)
    X = np.array([int(xy[i][0]) for i in order], np.int64); Y = np.array([int(xy[i][1]) for i in order], np.int64)
    K = int(k_needed)
    if K <= 0:
        return []
    if K == 1:
        return [order[0]]
    exp1 = rows + cols + 2*K
    exp2 = 4*cols + 4*K + 4*rows*K + rows*rows + cols*cols - 2*rows*cols + 4*rows*cols*K
    exp3 = math.sqrt(float(exp2)); exp4 = float(K - 1)
    sol1 = -_c_round((exp1 + exp3)/exp4); sol2 = -_c_round((exp1 - exp3)/exp4)
    high = int(sol1 if sol1 > sol2 else sol2)
    low = int(math.floor(math.sqrt(n/K)))
    Kf = np.float32(K); t = np.float32(tolerance)
    Kmin = int(_c_round(float(Kf - Kf*t))); Kmax = int(_c_round(float(Kf + Kf*t)))
    result = []; prevwidth = -1
    while True:
        width = low + _c_div(high - low, 2)
        if width == prevwidth or low > high:
            break                                   # the result of the previous iteration
        included = np.ones(n, bool)
        result = []
        for i in range(n):
            if included[i]:
                included[i] = False
                result.append(i)
                minx = max(int(X[i]) - width, 0); maxx = int(X[i]) + width
                miny = max(int(Y[i]) - width, 0); maxy = int(Y[i]) + width
                included &= ~((X >= minx) & (X <= maxx) & (Y >= miny) & (Y <= maxy))
        if Kmin <= len(result) <= Kmax:
            break
        elif len(result) < Kmin:
            high = width - 1
        else:
            low = width + 1
        prevwidth = width
    return [order[i] for i in result]


def sample_dynamic(flow, motion_mask, detection_mask, objects, num_track, prm, next_tracklet_id, max_features=200):
    """FeatureTracker::sampleDynamic: the literal candidate scan (oracle.frontend_oracle), each object's candidates in
    ascending pixel order through suppressNonMax(RangeTree, k = max(max_features - num_track, 0), tolerance 0.01), then the
    features with tracklet ids in object order and ANMS order (what a single-threaded run of the reference produces)."""
    from oracle import frontend_oracle as FO
    rows, cols = motion_mask.shape
    det = detection_mask if detection_mask is not None else np.full((rows, cols), 255, np.uint8)
    cand, zero = FO.sample_dynamic_candidates(flow, motion_mask, det, objects, prm)
    counts, num_sampled, zero_flow = [], [], []
    kp, fl, pk, tid, lab = [], [], [], [], []
    for o, nt in zip(objects, num_track):
        c = cand[int(o)]
        counts.append(len(c)); zero_flow.append(zero[int(o)])
        if not c:
            num_sampled.append(0)
            continue
        k = max(int(max_features) - int(nt), 0)
        sel = anms_range_tree([(p % cols, p//cols) for p in c], k, np.float32(0.01), cols, rows)
        num_sampled.append(len(sel))
        for s in sel:
            i, j = divmod(c[s], cols)
            fx = float(flow[i, j, 0]); fy = float(flow[i, j, 1])
            kp.append((float(j), float(i))); fl.append((fx, fy)); pk.append((j + fx, i + fy))
            tid.append(next_tracklet_id); next_tracklet_id += 1; lab.append(int(o))
    return dict(counts=np.array(counts, np.int32), num_sampled=np.array(num_sampled, np.int32), zero_flow=np.array(zero_flow, np.int32),
                keypoint=np.array(kp, np.float64).reshape(-1, 2), flow=np.array(fl, np.float64).reshape(-1, 2),
                predicted=np.array(pk, np.float64).reshape(-1, 2), tracklet=np.array(tid, np.int64), label=np.array(lab, np.int32),
                next_tracklet_id=next_tracklet_id)
