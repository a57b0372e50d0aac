"""The front end's image kernels at every frame size of tests/frame_cases.py (the reference's dataset sizes and the edge sizes of
the geometry rules), against the existing oracles and bars:
  * every pyramid level and its Scharr derivatives against the cv2.pyrDown chain and cv2.Scharr (BORDER_REFLECT_101), bit for bit;
  * klt_track against cv2.calcOpticalFlowPyrLK with a third of the points near the edges, max_level 3 and 5 (the cap binds on
    the small cases), with and without initial flow: test_klt_matches_opencv's bar;
  * detect_stages (CLAHE, eigen image, GFTT corners) bit-exact against cv2, detect_static against detection_oracle.detect;
at the dataset sizes:
  * klt_track_fb / klt_track_points against cv2 and the host chain;
  * track_dynamic, sample_dynamic, propagate_mask, track_static_flow (partial last grid cell), track_dynamic_klt, update_depths,
    back_project and dense_cloud bit-exact against their literal oracles (fewer features, never a cropped frame);
  * stereo_match on the resident frame (752x480, 1241x376) against the call-by-call composition and cv2's LK;
  * streaming against call by call (640x360, 1241x376);
and the refusal of frames smaller than the LK window by every LK entry point."""
import math

import numpy as np
import pytest

import depth_oracle as DPO
import detection_oracle as DO
import dynamic_klt_oracle as KO
import frame_cases as FC
import selection_oracle as SLO
import stereo_oracle as STO
from dynosam_b200.synth_frames import SyntheticStream

pytestmark = pytest.mark.gpu
needs_opencv_orders = pytest.mark.skipif(not DO.opencv_float_orders_apply(),
                                         reason="cv2 does not run OpenCV's AVX2 + FMA3 code path, whose float orders the device reproduces")
NAMES = list(FC.CASES)
CAL = (718.856, 718.856, 0.0, 607.1928, 185.2157)


def _tracker(c):
    from dynosam_b200.frontend import FeatureTrackerGPU
    return FeatureTrackerGPU(c.w, c.h)


def _edge_points(rng, w, h, n, margin=25.0):
    """n points: a third within `margin` px of the four edges and corners (some just outside), the rest anywhere"""
    pts = np.stack([rng.uniform(-5, w + 5, n), rng.uniform(-5, h + 5, n)], 1)
    k = n//3
    side = rng.integers(0, 4, k)
    d = rng.uniform(-3, margin, k)
    along = rng.uniform(0, 1, k)
    pts[:k, 0] = np.select([side == 0, side == 1], [d, w - 1 - d], along*w)
    pts[:k, 1] = np.select([side == 2, side == 3], [d, h - 1 - d], along*h)
    corner = slice(0, k//4)                                            # a quarter of them near a corner
    pts[corner, 1] = np.where(rng.random(k//4) < 0.5, d[corner], h - 1 - d[corner])
    return pts.astype(np.float32)


def _assert_klt_bar(t, nxt, stt, rn, rs, w, h, win=21):
    """test_klt_matches_opencv's bar; returns (status agreement, 99th percentile position error)"""
    agree = stt == rs
    assert agree.mean() >= 0.998, agree.mean()
    eig = t.klt_last_min_eig(len(stt))
    for i in np.flatnonzero(~agree):
        near_threshold = abs(float(eig[i, 0]) - 1e-4) <= 441*2.0**-24*max(float(eig[i, 1]), 1e-4)
        x, y = (rn[i] if rs[i] else nxt[i])
        at_border = min(x, y, w - 1 - x, h - 1 - y) < win + 1 + 1e-2
        assert near_threshold or at_border, (i, eig[i], stt[i], rs[i], nxt[i], rn[i])
    both = (stt == 1) & (rs == 1)
    d = np.abs(nxt[both] - rn[both]).max(axis=1)
    assert both.sum() > 0.3*len(stt), both.sum()
    assert np.percentile(d, 99) < 1e-2 and np.median(d) < 1e-3, (np.percentile(d, 99), np.median(d))
    return float(agree.mean()), float(np.percentile(d, 99))


# ------------------------------------------------------------------------------------------------ pyramid, Scharr, LK
@pytest.mark.parametrize("name", NAMES)
def test_pyramid_and_scharr_bit_exact(name):
    """next_frame builds levels 0-5 with derivatives (down to 2 px); two calls leave the first frame in pyramid 0"""
    import cv2
    from dynosam_b200.frontend import FrontendError
    c = FC.CASES[name]
    (g0, m0, f0), (g1, m1, f1) = FC.frame(c, 0), FC.frame(c, 1)
    t = _tracker(c)
    t.next_frame(g0, f0, m0); t.next_frame(g1, f1, m1)
    ref, lvl = g0, 0
    while lvl <= 5 and min(ref.shape) >= 2:
        try:
            img, der = t.pyramid_level(0, lvl)
        except FrontendError:
            break                                                      # no level this small on the device
        assert img.shape == ref.shape and np.array_equal(img, ref), (lvl, img.shape, ref.shape)
        dx = cv2.Scharr(ref, cv2.CV_16S, 1, 0, borderType=cv2.BORDER_REFLECT_101)
        dy = cv2.Scharr(ref, cv2.CV_16S, 0, 1, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(der[..., 0], dx) and np.array_equal(der[..., 1], dy), lvl
        ref = cv2.pyrDown(ref); lvl += 1
    assert lvl >= min(FC.klt_top_level(c.w, c.h, 5, 21) + 1, 6)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("max_level,initial", [(3, False), (5, False), (3, True), (5, True)])
def test_klt_matches_opencv(name, max_level, initial):
    from oracle import frontend_oracle as FO
    c = FC.CASES[name]
    rng = np.random.default_rng(9)
    g0, g1 = FC.frame(c, 10)[0], FC.frame(c, 11)[0]
    pts = _edge_points(rng, c.w, c.h, 1000)
    init = (pts + rng.normal(0, 1.0, pts.shape)).astype(np.float32) if initial else None
    t = _tracker(c)
    nxt, stt, err = t.klt_track(g0, g1, pts, win=21, max_level=max_level, max_count=30, eps=0.03, initial=init)
    rn, rs, re = FO.klt_track(g0, g1, pts, 21, max_level, 30, 0.03, init)
    agree, p99 = _assert_klt_bar(t, nxt, stt, rn, rs, c.w, c.h)
    both = (stt == 1) & (rs == 1)
    assert np.abs(err[both] - re[both]).max() < 0.5
    print(f"KLT {name} max_level {max_level} initial {initial}: status agreement {agree:.4f}, p99 {p99:.2e} px")


def test_smallest_admitted_frame_tracks():
    """a frame of exactly win + 1 rows is admitted, and tracks as cv2 does"""
    from oracle import frontend_oracle as FO
    c = FC.Case("h22", 64, 22, ())
    g0, g1 = FC.frame(c, 0)[0], FC.frame(c, 1)[0]
    pts = _edge_points(np.random.default_rng(3), c.w, c.h, 300)
    t = _tracker(c)
    nxt, stt, _ = t.klt_track(g0, g1, pts, win=21, max_level=3)
    rn, rs, _ = FO.klt_track(g0, g1, pts, 21, 3, 30, 0.03)
    _assert_klt_bar(t, nxt, stt, rn, rs, c.w, c.h)


@pytest.mark.parametrize("name", FC.DATASET)
def test_klt_fb_and_track_points_at_dataset_sizes(name):
    """klt_track_fb against cv2 + the literal checks (test_klt_forward_backward_on_device), klt_track_points against klt_track_fb +
    cv2.findHomography on the host (test_klt_track_points_equals_host_chain)"""
    import cv2
    from dynosam_b200.frontend import TrackParams
    from oracle import frontend_oracle as FO
    c = FC.CASES[name]
    rng = np.random.default_rng(4)
    (g0, _, _), (g1, m1, f1) = FC.frame(c, 20), FC.frame(c, 21)
    n = 800
    pts = np.stack([rng.uniform(5, c.w - 5, n), rng.uniform(5, c.h - 5, n)], 1).astype(np.float32)
    age = rng.integers(0, 30, n).astype(np.int32)
    prm = TrackParams(shrink_row=20, shrink_col=20)
    t = _tracker(c); t.set_frame(f1, m1, None)
    nxt, stt, back, keep = t.klt_track_fb(g0, g1, pts, prm, age, 25)
    rn, rs, rb, rk = FO.klt_track_fb(g0, g1, pts, m1, age, 25, FO.TrackParams(shrink_row=20, shrink_col=20))
    assert (stt == rs).mean() >= 0.99, (stt == rs).mean()
    both = (stt == 1) & (rs == 1)
    assert np.percentile(np.abs(nxt[both] - rn[both]).max(axis=1), 99) < 1e-2
    same_px = both & (nxt.astype(np.float64).astype(np.int64) == rn.astype(np.float64).astype(np.int64)).all(axis=1)
    assert same_px.sum() > 0.8*both.sum() and np.array_equal(keep[same_px], rk[same_px])
    assert 0 < keep.sum() < stt.sum() and t.last_counts == (int(stt.sum()), int(keep.sum()))
    # klt_track_points: the same stages, then the homography RANSAC over the round-trip survivors
    b = _tracker(c); b.set_frame(f1, m1, None)
    tn, ts, ver, tk, Hd = t.klt_track_points(g0, g1, pts, prm, age, 25)
    hn, hs, _, hk = b.klt_track_fb(g0, g1, pts, prm, age, 25)
    good = np.flatnonzero(hs)
    Hc, mk = cv2.findHomography(pts[good], hn[good], cv2.RANSAC, 5.0)
    rv = np.zeros(n, np.uint8); rv[good] = mk.ravel()
    assert np.array_equal(tn, hn) and np.array_equal(ts, hs) and np.array_equal(ver, rv) and np.array_equal(tk, hk & rv)
    assert Hd is not None and np.abs(Hd - Hc).max() <= 1e-6*np.abs(Hc).max()
    assert 0 < ver.sum() <= ts.sum()


# ------------------------------------------------------------------------------------------------ detection
@needs_opencv_orders
@pytest.mark.parametrize("name", NAMES)
def test_detect_stages_bit_exact(name):
    import cv2
    c = FC.CASES[name]
    g, m, f = FC.frame(c, 3)
    rng = np.random.default_rng(1)
    kp = FC.cur_features(rng, m, min(150, c.w*c.h//4000))
    t = _tracker(c); t.set_frame(f, m, None)
    for p in (DO.Params(), DO.Params(min_distance=8, max_corners=3000)):
        t.detect_static(g, kp, FC.dev_params(p), 0)
        cl, eig, corners = t.detect_stages()
        ref_cl, ref_eig, ref_pts, _ = DO.stages(g, DO.detection_mask(m, None, kp, p.min_distance), p)
        assert np.array_equal(cl, cv2.createCLAHE(2.0, (8, 8)).apply(g))
        assert np.array_equal(eig, ref_eig) and np.array_equal(eig, DO.min_eigen_image(ref_cl))
        assert len(ref_pts) > 0 and corners.shape == ref_pts.shape and np.array_equal(corners, ref_pts.astype(np.int32))


@needs_opencv_orders
@pytest.mark.parametrize("name", NAMES)
def test_detect_static_bit_exact(name):
    c = FC.CASES[name]
    g, m, f = FC.frame(c, 4)
    rng = np.random.default_rng(7)
    kp = FC.cur_features(rng, m, min(300, c.w*c.h//3000))
    p = DO.Params()
    t = _tracker(c); t.set_frame(f, m, None)
    got, gid, gnext, gnc = t.detect_static(g, kp, FC.dev_params(p), 5000)
    ref, rid, rnext, rnc, starts = DO.detect(g, m, None, kp, p, 5000)
    assert gnc == rnc and len(ref) > 0
    DO.assert_keypoints(got, ref, DO.processed(g), starts)
    assert np.array_equal(gid, rid) and gnext == rnext


# ------------------------------------------------------------------------------------------------ dense flow and depth, per dataset size
def _features_on_objects(rng, m, f, per_object):
    """previous-frame dynamic features on the objects of m, predicted by the flow, inside the image"""
    h, w = m.shape
    kps, labs = [], []
    for lab in sorted(set(np.unique(m).tolist()) - {0}):
        ys, xs = np.nonzero(m == lab)
        sel = rng.choice(len(ys), size=min(per_object, len(ys)), replace=False)
        x = xs[sel] + rng.uniform(0, 0.9, len(sel)); y = ys[sel] + rng.uniform(0, 0.9, len(sel))
        kps.append(np.stack([x + f[ys[sel], xs[sel], 0], y + f[ys[sel], xs[sel], 1]], 1)); labs += [lab]*len(sel)
    kps = np.concatenate(kps); labs = np.array(labs, np.int32)
    keep = (kps[:, 0] > 1) & (kps[:, 0] < w - 1) & (kps[:, 1] > 1) & (kps[:, 1] < h - 1)
    return kps[keep], labs[keep]


def _cell_size(w, h):
    """the smallest trackStatic cell of 13-25 px that leaves a partial last column and row"""
    return next(s for s in range(13, 26) if w % s and h % s)


@pytest.mark.parametrize("name", FC.DATASET)
def test_dense_flow_paths_bit_exact(name):
    from dynosam_b200.frontend import TrackParams
    from oracle import frontend_oracle as FO
    c = FC.CASES[name]
    rng = np.random.default_rng(1)
    (_, m0, f0), (_, m1, f1) = FC.frame(c, 4, n_objects=8), FC.frame(c, 5, n_objects=8)
    zy, zx = np.nonzero(m1 == m1.max())
    f1 = f1.copy(); f1[zy[::3], zx[::3]] = 0.0                                 # exact-zero flow on an object: skipped / counted
    # track_dynamic with a detection mask, then sample_dynamic on the mask it leaves
    kp, lab = _features_on_objects(rng, m0, f0, 120)
    age = rng.integers(0, 22, len(lab)).astype(np.int32); tid = np.arange(1000, 1000 + len(lab), dtype=np.int64)
    det = np.full((c.h, c.w), 255, np.uint8); det[:, c.w - 21:c.w - 3] = 0; det[c.h - 9:, :] = 0
    prm = TrackParams(max_dynamic_feature_age=20, min_distance=3, shrink_row=2, shrink_col=3)
    fprm = FO.TrackParams(20, 3, 2, 3)
    t = _tracker(c); t.set_frame(f1, m1, det)
    got = t.track_dynamic(kp, lab, age, tid, prm, 5000)
    ref = FO.track_dynamic(kp, lab, age, tid, f1, m1, det, fprm, 5000)
    assert 0 < ref[0].sum() < len(lab)
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)
    objs = [int(o) for o in np.unique(m1) if o != 0] + [77]
    ntr = rng.integers(0, 6, len(objs)).astype(np.int32)
    g = t.sample_dynamic(objs, ntr, prm, 7000)
    o = SLO.sample_dynamic(f1, m1, ref[7], objs, ntr, fprm, 7000)
    for key in ("counts", "num_sampled", "zero_flow", "tracklet", "label", "keypoint", "flow", "predicted"):
        assert np.array_equal(g[key], o[key]), key
    assert g["next_tracklet_id"] == o["next_tracklet_id"] and g["zero_flow"].sum() > 0 and g["num_sampled"][:-1].sum() > 0
    # propagate_mask: the first two objects lost by the detector in the current frame
    cur = m1.copy()
    for l in sorted(set(np.unique(m0).tolist()) - {0})[:2]:
        cur[cur == l] = 0
    out = t.propagate_mask(kp, lab, m0, f0, cur, TrackParams(), min_votes=20)
    assert np.array_equal(out, FO.propagate_mask(kp, lab, m0, f0, cur, FO.TrackParams(), min_votes=20)) and (out != cur).any()
    # track_static_flow with a partial last grid column and row
    cell = _cell_size(c.w, c.h)
    n_prev, n_det = 900, 1500
    skp = np.stack([rng.uniform(-3, c.w + 3, n_prev), rng.uniform(-3, c.h + 3, n_prev)], 1)
    skp[:60] = np.stack([rng.uniform(c.w - c.w % cell, c.w, 60), rng.uniform(0, c.h, 60)], 1)      # the last column of cells
    skp[60:120] = np.stack([rng.uniform(0, c.w, 60), rng.uniform(c.h - c.h % cell, c.h, 60)], 1)   # the last row of cells
    sage = rng.integers(0, 30, n_prev).astype(np.int32); usable = (rng.uniform(0, 1, n_prev) > 0.1).astype(np.uint8)
    sdet = np.stack([rng.integers(0, c.w, n_det), rng.integers(0, c.h, n_det)], 1).astype(np.int32)
    sdet[:40] = np.stack([rng.integers(c.w - c.w % cell, c.w, 40), rng.integers(0, c.h, 40)], 1)
    t.set_frame(f1, m1, None)
    gs = t.track_static_flow(skp, sage, usable, sdet, cell, 3000, 5000)
    os_ = FO.track_static_flow(skp, sage, usable, sdet, f1, m1, cell, 3000, 5000)
    for k in ("acc", "age", "det_acc", "det_tracklet", "flow", "pred", "det_flow", "det_pred"):
        assert np.array_equal(gs[k], os_[k]), k
    assert (gs["next_tracklet_id"], gs["n_tracked"], gs["n_detected"]) == (os_["next_tracklet_id"], os_["n_tracked"], os_["n_detected"])
    ncols = math.ceil(c.w/cell)
    last_col = {int(y//cell)*ncols + ncols - 1 for (x, y), a in zip(skp, gs["acc"]) if a and x >= c.w - c.w % cell}
    assert gs["n_tracked"] > 100 and gs["n_detected"] > 100 and last_col


def _objects(m):
    """objects_detected and inner boxes: each label's bounding box shrunk by 2 px (at least 1 px wide)"""
    objs, bb = [], []
    for oid in sorted(set(np.unique(m).tolist()) - {0}):
        ys, xs = np.nonzero(m == oid)
        objs.append(oid); bb.append((xs.min() + 2, ys.min() + 2, max(xs.max() - xs.min() - 3, 1), max(ys.max() - ys.min() - 3, 1)))
    return objs, np.array(bb, np.int32).reshape(-1, 4)


@needs_opencv_orders
@pytest.mark.parametrize("name", FC.DATASET)
def test_track_dynamic_klt_bit_exact(name):
    """the oracle is fed the device's own LK result; every other output equal bit for bit (test_dynamic_klt_gpu's bar)"""
    c = FC.CASES[name]
    rng = np.random.default_rng(5)
    (g0, m0, _), (g1, m1, f1) = FC.frame(c, 6, n_objects=8), FC.frame(c, 7, n_objects=8)
    kp, lab = [], []
    for oid in sorted(set(np.unique(m0).tolist()) - {0})[1:]:          # the first object has no previous features: new
        ys, xs = np.nonzero(m0 == oid)
        s = rng.choice(len(ys), min(60, len(ys)), replace=False)
        kp.append(np.stack([xs[s] + 0.5, ys[s] + 0.5], 1)); lab += [oid]*len(s)
    kp = np.concatenate(kp).astype(np.float32); lab = np.array(lab, np.int32)
    prev = (kp, lab, rng.integers(0, 18, len(lab)).astype(np.int32), np.arange(len(lab), dtype=np.int64))
    boundary = np.full((c.h, c.w), 255, np.uint8); boundary[:, :12] = 0
    objs, bb = _objects(m1)
    t = _tracker(c); t.set_frame(f1, m1, boundary)
    dev = t.track_dynamic_klt(g0, g1, *prev, objs, bb, 1000)
    ref = KO.track_dynamic_klt(g1, m1, boundary, *prev, dev["lk_pts"], dev["lk_status"], objs, bb, KO.Params(), 1000)
    assert np.array_equal(dev["state"], ref["state"]) and np.array_equal(dev["measured_flow"], ref["measured_flow"])
    for k in ("keypoint", "age", "tracklet", "label", "source"):
        assert dev[k].shape == ref[k].shape and np.array_equal(dev[k], ref[k]), k
    assert dev["next_tracklet_id"] == ref["next_tracklet_id"] and dev["n_outside_image"] == ref["n_outside_image"]
    for fld in KO.STATUS_FIELDS:
        assert np.array_equal(dev["status"][fld], ref["status"][fld]), fld
    assert np.array_equal(dev["detection_mask"], ref["detection_mask"]) and np.array_equal(dev["tracking_mask"], ref["tracking_mask"])
    assert (dev["state"] == KO.TRACKED).sum() > 50 and (dev["source"] < 0).sum() > 0


@pytest.mark.parametrize("name", FC.DATASET)
def test_depth_paths_bit_exact(name):
    c = FC.CASES[name]
    st = SyntheticStream(n_objects=8, seed=42, width=c.w, height=c.h)
    rng = np.random.default_rng(11)
    _, m, f = st.frame(2); depth = st.depth(2)
    n = 600
    kp = np.concatenate([np.stack([rng.uniform(-3, c.w + 3, n), rng.uniform(-3, c.h + 3, n)], 1),
                         [[c.w - 0.001, c.h - 0.001], [c.w - 1, 0.0], [0.0, c.h - 1], [c.w, 3.0], [3.0, c.h]]])
    lab = m[np.clip(kp[:, 1], 0, c.h - 1).astype(int), np.clip(kp[:, 0], 0, c.w - 1).astype(int)].astype(np.int32)
    t = _tracker(c); t.set_frame(f, m, None); t.set_depth(depth)
    d, v, ninv, nout = t.update_depths(kp, lab, 200.0, 30.0)
    rd, rv, rninv, rnout = DPO.update_depths(kp, lab, depth, 200.0, 30.0)
    assert np.array_equal(d, rd, equal_nan=True) and np.array_equal(v, rv) and (ninv, nout) == (rninv, rnout) and nout > 0
    usable = v.copy(); usable[rng.random(len(v)) < 0.1] = 0
    right = np.full(len(kp), np.nan); sub = (rng.random(len(kp)) < 0.3) & ~np.isnan(d)
    right[sub] = kp[sub, 0] - rng.uniform(1, 40, sub.sum())
    for rgbd, r in ((True, None), (True, right), (False, right)):
        bp = t.back_project(kp, d, usable, CAL, 0.537, rgbd, r)
        idx, pt, sp, out = DPO.back_project(kp, d, usable, CAL, c.w, 0.537, rgbd, r)
        assert bp["m"] == len(idx) and np.array_equal(bp["index"], idx)
        for a, b in ((bp["point"], pt), (bp["stereo"], sp), (bp["outlier"], out)):
            assert a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")
    det = np.full((c.h, c.w), 255, np.uint8); det[:, :17] = 0; det[c.h - 5:, :] = 0
    t.set_frame(f, m, det); t.set_depth(depth)
    xyz, rgb, labo, valid, nv = t.dense_cloud(CAL, 200.0, 30.0)
    rx, rr, rl, rvd = DPO.dense_cloud(depth, m, det, CAL, 200.0, 30.0)
    assert np.array_equal(xyz, rx, equal_nan=True) and np.array_equal(rgb, rr) and np.array_equal(labo, rl) and np.array_equal(valid, rvd)
    assert nv == int(rvd.sum()) and 0 < nv < c.w*c.h and (rl[rvd == 1] != 0).any()


# ------------------------------------------------------------------------------------------------ stereo and streaming
@pytest.mark.parametrize("name", ["viode_752x480", "kitti20_1241x376"])
def test_stereo_match_resident(name):
    """next_frame + set_right + stereo_match against the call-by-call composition (stereo_track, host compaction,
    find_fundamental_batch, stereo_oracle.per_feature) bit for bit, and the LK against cv2"""
    from oracle import frontend_oracle as FO
    c = FC.CASES[name]
    s = SyntheticStream(n_objects=8, seed=42, width=c.w, height=c.h)
    a, b = _tracker(c), _tracker(c)
    agree = []
    for k in (3, 4):
        left, right, mask, pts = STO.c4_stereo_frame(s, k)
        a.next_frame(np.ascontiguousarray(left), np.ascontiguousarray(s.frame(k)[2]), np.ascontiguousarray(mask))
        a.set_right(right)
        d = a.stereo_match(pts, STO.FX, STO.BASELINE)
        rp, st, _, _ = b.stereo_track(left, right, pts, STO.FX, STO.BASELINE)
        good = np.flatnonzero(st)
        r = b.find_fundamental_batch([(pts[good], rp[good])])
        state, depth, ru = STO.per_feature(pts, rp, st, r["masks"][0], STO.FX, STO.BASELINE)
        assert np.array_equal(d["right_pts"], rp) and np.array_equal(d["lk_status"], st) and d["n_tracked"] == len(good)
        assert d["matched"] and d["fund_status"] == int(r["status"][0]) and np.array_equal(d["F"], r["F"][0][0])
        assert np.array_equal(d["state"], state)
        assert np.array_equal(d["depth"], depth, equal_nan=True) and np.array_equal(d["right_u"], ru, equal_nan=True)
        assert d["n_stereo"] == int((state == STO.MATCHED).sum()) > 100
        orp, ost, _, _ = FO.stereo_track(left, right, pts, STO.FX, STO.BASELINE)
        agree.append(st == ost)
        both = (st == 1) & (ost == 1)
        assert np.percentile(np.abs(rp[both] - orp[both]).max(axis=1), 99) < 1e-2
    assert np.concatenate(agree).mean() >= 0.99


@pytest.mark.parametrize("name", ["tartan_aria_640x360", "kitti20_1241x376"])
def test_streaming_equals_call_by_call(name):
    """next_frame's resident pair against re-uploaded images: mask propagation, dynamic tracking, the forward-backward KLT,
    klt_track_points and detection"""
    from dynosam_b200.frontend import DetectParams, TrackParams
    c = FC.CASES[name]
    rng = np.random.default_rng(3)
    frames = [FC.frame(c, k, seed=5) for k in range(4)]
    prm = TrackParams()
    pts = np.stack([rng.uniform(25, c.w - 25, 300), rng.uniform(25, c.h - 25, 300)], 1).astype(np.float32)
    age = rng.integers(0, 30, 300).astype(np.int32)
    a, b = _tracker(c), _tracker(c)
    a.next_frame(frames[0][0], frames[0][2], frames[0][1])
    for k in range(1, 4):
        g0, m0, f0 = frames[k - 1]; g1, m1, f1 = frames[k]
        kp, lab = _features_on_objects(rng, m0, f0, 100)
        fage = rng.integers(0, 22, len(lab)).astype(np.int32); tid = np.arange(len(lab), dtype=np.int64)
        a.next_frame(g1, f1, m1)
        a.propagate_mask_resident(kp, lab, prm, min_votes=20)
        ra = a.track_dynamic(kp, lab, fage, tid, prm, 9000)
        ka = a.klt_track_fb(None, None, pts, prm, age, 25)
        pa = a.klt_track_points(None, None, pts, prm, age, 25)
        da = a.detect_static(None, pts[:100], DetectParams(), 100)
        cur = b.propagate_mask(kp, lab, m0, f0, m1, prm, min_votes=20)
        b.set_frame(f1, cur, None)
        rb = b.track_dynamic(kp, lab, fage, tid, prm, 9000)
        kb = b.klt_track_fb(g0, g1, pts, prm, age, 25)
        pb = b.klt_track_points(g0, g1, pts, prm, age, 25)
        db = b.detect_static(g1, pts[:100], DetectParams(), 100)
        assert np.array_equal(a.motion_mask(), cur), k
        for x, y in list(zip(ra, rb)) + list(zip(ka, kb)) + list(zip(pa, pb)) + list(zip(da, db)):
            assert (x is None and y is None) or np.array_equal(x, y), k


# ------------------------------------------------------------------------------------------------ frames smaller than the window
def test_frames_smaller_than_the_lk_window_are_refused():
    """a 20-row handle at win 21: every LK entry point refuses on the host before anything runs"""
    from dynosam_b200.frontend import FeatureTrackerGPU, FrontendError
    w, h = 64, 20
    g0 = FC.value_noise(h, w, 1); g1 = FC.value_noise(h, w, 1, (0.5, 0.0))
    m = np.zeros((h, w), np.int32); f = np.zeros((h, w, 2), np.float32)
    pts = np.stack([np.linspace(3, w - 3, 12), np.linspace(3, h - 3, 12)], 1).astype(np.float32)
    t = FeatureTrackerGPU(w, h); t.set_frame(f, m, None)
    calls = {
        "klt_track": lambda: t.klt_track(g0, g1, pts, win=21),
        "klt_track_fb": lambda: t.klt_track_fb(g0, g1, pts),
        "klt_track_points": lambda: t.klt_track_points(g0, g1, pts),
        "track_dynamic_klt": lambda: t.track_dynamic_klt(g0, g1, pts, np.ones(12, np.int32), np.zeros(12, np.int32),
                                                         np.arange(12, dtype=np.int64), [], np.zeros((0, 4), np.int32), 0),
        "stereo_track": lambda: t.stereo_track(g0, g1, pts, 700.0, 0.5),
        "stereo_match": lambda: t.stereo_match(pts, 700.0, 0.5, left=g0, right=g1),
    }
    for name, call in calls.items():
        with pytest.raises(FrontendError, match="smaller than the LK window"):
            call()
    nxt, st, _ = t.klt_track(g0, g1, pts, win=19)                      # a window that fits is still served
    assert st.shape == (12,)
