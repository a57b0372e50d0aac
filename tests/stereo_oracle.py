"""CPU restatement of FeatureTracker::stereoTrack (dynosam/src/frontend/vision/FeatureTracker.cc:194-337) (TEST INFRASTRUCTURE,
NOT PRODUCT), the reference of dynofront_stereo_match.

The input is what left_features.toOpenCV(&tracklets_ids, true) gives (Feature.cc:389-401): the usable static features in
container order as float points; the tracklet ids are their positions here.  The steps, literally:
  * fewer than 8 points: return false (:205), nothing is marked;
  * LK left -> right (oracle.frontend_oracle.stereo_track's cv2 call: 21x21, maxLevel 5, default criteria), or a given LK
    result; the right -> left pass is not run, its filter being commented out (:240-253);
  * the status-good points in order (:259-267); fewer than 8: return false (:273);
  * cv::findFundamentalMat(FM_RANSAC, 1.0, 0.99) over them: fundamental_oracle.find_fundamental or cv2.findFundamentalMat.
    The reference's mask is a std::vector<uchar> that findFundamentalMat resizes to m zeros and writes only when a model is
    found, so a failed RANSAC leaves every tracked point an epipolar outlier; LMedS's mask is used even when F comes back empty;
  * per inlier: disparity = uL - uR in double, markOutlier when disparity <= 1 or uR < 0, else depth = fx * baseline / disparity
    and the right key-point (uR, v) (:301-328);
  * determineOutlierIds(inliers, all ids) marks every point that is not an epipolar inlier (:330-334).
Only tests/ may import this module.
"""
from __future__ import annotations

import numpy as np

UNTOUCHED, MATCHED, LOST, EPIPOLAR, DISPARITY = 0, 1, 2, 3, 4      # dynofront_stereo_match states


def per_feature(left_pts, right_pts, status, mask, fx, baseline):
    """the loop after the RANSAC: mask[m] over the status-good points in order.  Returns (state, depth, right_u) per input point"""
    left = np.asarray(left_pts, np.float32).reshape(-1, 2); right = np.asarray(right_pts, np.float32).reshape(-1, 2)
    n = len(left)
    features = [dict(inlier=True, depth=np.nan, right_u=np.nan) for _ in range(n)]     # feature i has tracklet id i
    tracklet_ids = list(range(n))
    good = [i for i in range(n) if status[i]]
    pts_left_tracked = [left[i] for i in good]; pts_right_tracked = [right[i] for i in good]
    assert len(mask) == len(good)
    inlier_ids, pts_left_inlier, pts_right_inlier = [], [], []
    for k in range(len(mask)):
        if mask[k]:
            pts_left_inlier.append(pts_left_tracked[k]); pts_right_inlier.append(pts_right_tracked[k]); inlier_ids.append(good[k])
    stereo = []
    for k, tid in enumerate(inlier_ids):
        f = features[tid]
        uL = float(pts_left_inlier[k][0]); uR = float(pts_right_inlier[k][0])
        disparity = uL - uR
        if disparity <= 1.0 or uR < np.float32(0.0):
            f["inlier"] = False                                        # markOutlier
            continue
        f["depth"] = fx*baseline/disparity; f["right_u"] = uR
        stereo.append(tid)
    inlier_set = set(inlier_ids)
    outliers = [t for t in tracklet_ids if t not in inlier_set]        # determineOutlierIds
    state = np.zeros(n, np.uint8); depth = np.full(n, np.nan); right_u = np.full(n, np.nan)
    for t in outliers:
        features[t]["inlier"] = False
        state[t] = LOST if not status[t] else EPIPOLAR
    for t in inlier_ids:
        state[t] = DISPARITY if not features[t]["inlier"] else MATCHED
    for t in stereo:
        depth[t] = features[t]["depth"]; right_u[t] = features[t]["right_u"]
    return state, depth, right_u


def fundamental(a, b, which="oracle", thr=1.0, confidence=0.99, max_iters=1000):
    """(F or None, mask[m], status) of findFundamentalMat over the tracked points: which = "oracle" (fundamental_oracle) or "cv2".
    With cv2 the mask array is allocated as the reference's vector is (m zeros) and handed in, so what cv2 does not write stays 0."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 2); b = np.ascontiguousarray(b, np.float32).reshape(-1, 2)
    if which == "oracle":
        import fundamental_oracle as FO
        o = FO.find_fundamental(a, b, thr, confidence, max_iters)
        return (o.F[0] if o.F else None), o.mask.astype(np.uint8), o.status
    import cv2
    mask = np.zeros((len(a), 1), np.uint8)
    F, mk = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, thr, confidence, max_iters, mask=mask)
    mk = mask if mk is None else mk
    return (None if F is None or F.size == 0 else F.reshape(3, 3)), mk.ravel().copy(), None


def stereo_match(left_gray, right_gray, left_pts, fx, baseline, lk=None, which="oracle", thr=1.0, confidence=0.99, max_iters=1000):
    """the whole of stereoTrack.  lk = (right_pts, status) replaces the cv2 LK.  Returns a dict with matched, state, depth,
    right_u, right_pts, lk_status, F, mask (over the tracked points), fund_status (fundamental_oracle's, None with cv2, -1 when
    the RANSAC did not run), n_tracked, n_inliers, n_stereo"""
    p0 = np.ascontiguousarray(left_pts, np.float32).reshape(-1, 2); n = len(p0)
    out = dict(matched=False, state=np.zeros(n, np.uint8), depth=np.full(n, np.nan), right_u=np.full(n, np.nan), right_pts=None,
               lk_status=None, F=None, mask=None, fund_status=-1, n_tracked=0, n_inliers=0, n_stereo=0)
    if n < 8:
        return out
    if lk is None:
        from oracle import frontend_oracle
        rp, st, _, _ = frontend_oracle.stereo_track(left_gray, right_gray, p0, fx, baseline)
    else:
        rp, st = lk
    rp = np.asarray(rp, np.float32).reshape(-1, 2); st = np.asarray(st, np.uint8).reshape(-1)
    good = np.flatnonzero(st)
    out.update(right_pts=rp, lk_status=st, n_tracked=len(good))
    if len(good) < 8:
        return out
    F, mask, fstat = fundamental(p0[good], rp[good], which, thr, confidence, max_iters)
    state, depth, right_u = per_feature(p0, rp, st, mask, fx, baseline)
    out.update(matched=True, state=state, depth=depth, right_u=right_u, F=F, mask=mask, fund_status=fstat,
               n_inliers=int(mask.sum()), n_stereo=int((state == MATCHED).sum()))
    return out


def per_feature_vectorised(left_pts, right_pts, status, mask, fx, baseline):
    """an independent numpy statement of per_feature's rules"""
    left = np.asarray(left_pts, np.float32).reshape(-1, 2); right = np.asarray(right_pts, np.float32).reshape(-1, 2)
    st = np.asarray(status).astype(bool)
    inl = np.zeros(len(left), bool); inl[np.flatnonzero(st)] = np.asarray(mask).astype(bool)
    disparity = left[:, 0].astype(np.float64) - right[:, 0].astype(np.float64)
    bad = (disparity <= 1.0) | (right[:, 0] < 0)
    state = np.select([~st, ~inl, bad], [LOST, EPIPOLAR, DISPARITY], MATCHED).astype(np.uint8)
    ok = state == MATCHED
    with np.errstate(divide="ignore", invalid="ignore"):
        depth = np.where(ok, fx*baseline/disparity, np.nan)
    return state, depth, np.where(ok, right[:, 0].astype(np.float64), np.nan)


FX, BASELINE = 721.5377, 0.5372          # SyntheticStream.right's defaults (KITTI-like)


def c4_stereo_frame(stream, k, n_points=800):
    """frame k of a C4 stream as a stereo pair: (left gray, right gray, motion mask, left points [n][2] float32), the points
    being up to n_points good features to track on the background, the static features a stereo frame would carry"""
    import cv2
    left, mask, _ = stream.frame(k)
    right = stream.right(k, FX, BASELINE)
    pts = cv2.goodFeaturesToTrack(left, n_points, 0.001, 15, mask=(mask == 0).astype(np.uint8))
    return left, right, mask, np.ascontiguousarray(pts.reshape(-1, 2), np.float32)
