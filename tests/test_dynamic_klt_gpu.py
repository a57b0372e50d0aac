"""FeatureTracker::trackDynamicKLT on the device (dynofront_track_dynamic_klt) against the CPU oracle (tests/dynamic_klt_oracle.py).

The oracle is fed the device's own LK result (status and points), so that LK rounding stays apart; every other output must be
equal bit for bit: per-feature states and measured flows, the output features in order with their ids, next_tracklet_id, the
status rows and both masks.  A 20-frame C4 run carries its features forward and takes every sampling reason; streaming and
explicit images agree; the hand-built frame, zero objects and zero previous features; the LK stage against CPU cv2.
"""
import numpy as np
import pytest

import detection_oracle as DO
import dynamic_klt_oracle as KO
from dynosam_b200.synth_frames import SyntheticStream

W, H = 1242, 375
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not DO.opencv_float_orders_apply(),
                                 reason="cv2 does not run OpenCV's AVX2 + FMA3 code path, whose eigen-image float orders the device reproduces")]


def _frames(n, seed=42):
    st = SyntheticStream(n_objects=10, seed=seed)
    out = []
    for k in range(n):
        g, m, f = st.frame(k)
        out.append((np.ascontiguousarray(g.astype(np.uint8)), np.ascontiguousarray(m.astype(np.int32)), np.ascontiguousarray(f.astype(np.float32))))
    return out


def _objects(m):
    """objects_detected and inner boxes: each label's bounding box shrunk by 2 px (at least 1 px wide)"""
    objs, bb = [], []
    for oid in sorted(set(np.unique(m).tolist()) - {0}):
        ys, xs = np.nonzero(m == oid)
        x0, y0, x1, y1 = xs.min(), ys.min(), xs.max(), ys.max()
        objs.append(oid); bb.append((x0 + 2, y0 + 2, max(x1 - x0 - 3, 1), max(y1 - y0 - 3, 1)))
    return objs, np.array(bb, np.int32).reshape(-1, 4)


def _oracle(dev, cur_g, m, boundary, prev, objs, bb, prm, nid):
    kp, lab, age, tid = prev
    return KO.track_dynamic_klt(cur_g, m, boundary, kp, lab, age, tid, dev["lk_pts"], dev["lk_status"], objs, bb, prm, nid)


def _assert_equal(dev, ref):
    assert np.array_equal(dev["state"], ref["state"])
    assert np.array_equal(dev["tracked"], (ref["state"] == KO.TRACKED).astype(np.uint8))
    assert np.array_equal(dev["measured_flow"], ref["measured_flow"])
    for k in ("keypoint", "age", "tracklet", "label", "source"):
        assert dev[k].shape == ref[k].shape and np.array_equal(dev[k], ref[k]), k
    assert dev["next_tracklet_id"] == ref["next_tracklet_id"] and dev["n_outside_image"] == ref["n_outside_image"]
    for f in KO.STATUS_FIELDS:
        assert np.array_equal(dev["status"][f], ref["status"][f]), (f, dev["status"][f], ref["status"][f])
    assert np.array_equal(dev["detection_mask"], ref["detection_mask"])
    assert np.array_equal(dev["tracking_mask"], ref["tracking_mask"])


def _kprm(p: KO.Params):
    from dynosam_b200.frontend import KltDynamicParams
    return KltDynamicParams(max_dynamic_feature_age=p.max_dynamic_feature_age, min_distance=p.min_distance, shrink_row=p.shrink_row,
                            shrink_col=p.shrink_col, max_features=p.max_features, quality_level=p.quality_level, age_buffer=p.age_buffer,
                            min_tracks=p.min_tracks, min_iou=p.min_iou)


def _seed_features(m, rng):
    """previous features of frame 0 that set up each sampling reason at frame 1: label 1 old (age 17), label 2 only 5
    features, label 3 all in a 12 px patch (small IoU), labels 4 and 5 none (new), the others 80 young ones spread out,
    some of them 1 px apart (masked by the earlier one's disc)"""
    kp, lab, age = [], [], []
    for oid in sorted(set(np.unique(m).tolist()) - {0, 4, 5}):
        ys, xs = np.nonzero(m == oid)
        if oid == 3:
            sel = (xs < xs.min() + 12) & (ys < ys.min() + 12); ys, xs = ys[sel], xs[sel]
        k = min({2: 5}.get(oid, 80), len(ys))
        s = rng.choice(len(ys), k, replace=False)
        p = np.stack([xs[s] + 0.5, ys[s] + 0.5], 1)
        if oid not in (2, 3):
            p[1::10] = p[0::10][:len(p[1::10])] + [1.0, 0.0]
        kp.append(p); lab += [oid]*k; age += [17 if oid == 1 else int(a) for a in rng.integers(0, 6, k)]
    kp = np.concatenate(kp).astype(np.float32)
    return kp, np.array(lab, np.int32), np.array(age, np.int32), np.arange(len(kp), dtype=np.int64)


def test_c4_run_carries_features_forward_bit_exact():
    from dynosam_b200.frontend import FeatureTrackerGPU
    frames = _frames(21)
    rng = np.random.default_rng(5)
    prm = KO.Params()
    t = FeatureTrackerGPU(W, H)
    t.next_frame(frames[0][0], frames[0][2], frames[0][1])
    prev = _seed_features(frames[0][1], rng); nid = 10**6
    reasons = set(); states = np.zeros(6, np.int64); masked_by_disc = 0; age_dropped = 0
    for k in range(1, 21):
        g, m, f = frames[k]
        t.next_frame(g, f, m)
        objs, bb = _objects(m)
        dev = t.track_dynamic_klt(None, None, *prev, objs, bb, nid, _kprm(prm))
        ref = _oracle(dev, g, m, None, prev, objs, bb, prm, nid)
        _assert_equal(dev, ref)
        for why in ref["reasons"].values():
            reasons.update(why)
        states += np.bincount(dev["state"], minlength=6)
        masked_by_disc += int((dev["state"] == KO.MASKED).sum())                    # no boundary mask: every masked one is a disc
        age_dropped += int(((dev["state"] == KO.REJECTED) & (prev[2] + 1 > prm.max_dynamic_feature_age)).sum())
        nid = dev["next_tracklet_id"]
        prev = (dev["keypoint"].astype(np.float32), dev["label"], dev["age"], dev["tracklet"])
    print("reasons", sorted(reasons), "states", states.tolist(), "masked", masked_by_disc, "age-dropped", age_dropped, "last ms", t.last_ms)
    assert {"new", "old", "few", "iou"} <= reasons, reasons
    assert masked_by_disc > 0 and age_dropped > 0 and states[KO.TRACKED] > 1000


def test_streaming_equals_explicit_images():
    from dynosam_b200.frontend import FeatureTrackerGPU
    frames = _frames(4, seed=7)
    rng = np.random.default_rng(2)
    boundary = np.full((H, W), 255, np.uint8); boundary[:30, :] = 0; boundary[:, 1100:] = 0
    a = FeatureTrackerGPU(W, H); b = FeatureTrackerGPU(W, H)
    a.next_frame(frames[0][0], frames[0][2], frames[0][1], boundary)
    prev = _seed_features(frames[0][1], rng); nid = 50
    for k in (1, 2, 3):
        g, m, f = frames[k]
        objs, bb = _objects(m)
        a.next_frame(g, f, m, boundary)
        ra = a.track_dynamic_klt(None, None, *prev, objs, bb, nid)
        b.set_frame(f, m, boundary)
        rb = b.track_dynamic_klt(frames[k - 1][0], g, *prev, objs, bb, nid)
        for key in ("lk_pts", "lk_status", "state", "measured_flow", "keypoint", "age", "tracklet", "label", "source", "detection_mask", "tracking_mask"):
            assert np.array_equal(ra[key], rb[key]), key
        for fld in KO.STATUS_FIELDS:
            assert np.array_equal(ra["status"][fld], rb["status"][fld]), fld
        assert ra["next_tracklet_id"] == rb["next_tracklet_id"]
        _assert_equal(ra, _oracle(ra, g, m, boundary, prev, objs, bb, KO.Params(), nid))
        assert (ra["state"] == KO.MASKED).sum() > 0
        nid = ra["next_tracklet_id"]
        prev = (ra["keypoint"].astype(np.float32), ra["label"], ra["age"], ra["tracklet"])


def test_hand_built_frame_on_the_device():
    from dynosam_b200.frontend import FeatureTrackerGPU
    prev_g, cur_g, mask, kp, lab, age, tid, objects, inner, _ = KO.hand_built_frame()
    h, w = mask.shape
    t = FeatureTrackerGPU(w, h)
    t.set_frame(np.zeros((h, w, 2), np.float32), mask, None)
    for prm in (KO.Params(), KO.Params(shrink_row=8, shrink_col=6, min_distance=3)):
        dev = t.track_dynamic_klt(prev_g, cur_g, kp, lab, age, tid, objects, inner, 1000, _kprm(prm))
        ref = _oracle(dev, cur_g, mask, None, (kp, lab, age, tid), objects, inner, prm, 1000)
        _assert_equal(dev, ref)
        if prm.shrink_row == 0:
            assert ref["reasons"] == {1: ["new"], 2: ["skipped"], 3: ["old"], 4: ["few"], 5: ["iou"], 6: ["iou"], 7: []}
            assert dev["n_outside_image"] == 1 and dev["state"][31] == KO.MASKED
            assert dev["status"]["num_sampled"][6] == 0 and dev["status"]["sampled"][6] == 1      # K = 0


def test_zero_objects_and_zero_features():
    from dynosam_b200.frontend import FeatureTrackerGPU
    frames = _frames(2, seed=3)
    (g0, m0, f0), (g1, m1, f1) = frames
    t = FeatureTrackerGPU(W, H); t.set_frame(f1, m1, None)
    prev = _seed_features(m0, np.random.default_rng(1))
    objs, bb = _objects(m1)
    none = (np.zeros((0, 2), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int64))
    for p, o, b in ((prev, [], np.zeros((0, 4), np.int32)), (none, objs, bb), (none, [], np.zeros((0, 4), np.int32))):
        dev = t.track_dynamic_klt(g0, g1, *p, o, b, 7)
        ref = _oracle(dev, g1, m1, None, p, o, b, KO.Params(), 7)
        _assert_equal(dev, ref)
        if len(o) == 0:
            assert dev["next_tracklet_id"] == 7 and (dev["source"] >= 0).all()
        else:
            assert (dev["status"]["object_new"][1:] == 1).all() and len(dev["keypoint"]) > 100


def test_capacity_and_refusals():
    import ctypes as C

    from dynosam_b200.frontend import FeatureTrackerGPU, FrontendError, KltDynamicParams
    (g0, m0, f0), (g1, m1, f1) = _frames(2, seed=3)
    t = FeatureTrackerGPU(W, H); t.set_frame(f1, m1, None)
    prev = _seed_features(m0, np.random.default_rng(1)); objs, bb = _objects(m1)
    full = t.track_dynamic_klt(g0, g1, *prev, objs, bb, 7)
    with pytest.raises(FrontendError):
        t.track_dynamic_klt(g0, g1, *prev, objs, bb, 7, capacity=5)
    with pytest.raises(FrontendError):
        t.track_dynamic_klt(g0, g1, *prev, [3, 3], np.zeros((2, 4), np.int32), 7)               # duplicate objects
    with pytest.raises(FrontendError):
        t.track_dynamic_klt(g0, g1, *prev, objs, bb, 7, KltDynamicParams(max_dynamic_feature_age=3))   # expiry age <= 0
    with pytest.raises(FrontendError):
        FeatureTrackerGPU(W, H).track_dynamic_klt(None, None, *prev, objs, bb, 7)             # no resident frames
    assert len(full["keypoint"]) > 100 and C.sizeof(C.c_int32) == 4


def test_lk_stage_matches_opencv():
    """the forward LK at (21x21, 3 levels, 30, 0.03) against CPU cv2, with the per-point proof of test_klt_matches_opencv"""
    from dynosam_b200.frontend import FeatureTrackerGPU
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(12)
    (g0, m0, f0), (g1, m1, f1) = _frames(2, seed=42)
    n = 1000
    pts = np.stack([rng.uniform(-5, W + 5, n), rng.uniform(-5, H + 5, n)], 1).astype(np.float32)
    pts[:50] = np.stack([rng.uniform(0, 12, 50), rng.uniform(0, H, 50)], 1)
    t = FeatureTrackerGPU(W, H); t.set_frame(f1, m1, None)
    dev = t.track_dynamic_klt(g0, g1, pts, np.ones(n, np.int32), np.zeros(n, np.int32), np.arange(n, dtype=np.int64), [], np.zeros((0, 4), np.int32), 0)
    nxt, stt = dev["lk_pts"], dev["lk_status"]
    rn, rs, _ = FO.klt_track(g0, g1, pts, 21, 3, 30, 0.03)
    agree = stt == rs
    assert agree.mean() >= 0.998, agree.mean()
    eig = t.klt_last_min_eig(n)
    for i in np.flatnonzero(~agree):
        near_threshold = abs(float(eig[i, 0]) - 1e-4) <= 441*2.0**-24*max(float(eig[i, 1]), 1e-4)
        x, y = (rn[i] if rs[i] else nxt[i])
        at_border = min(x, y, W - 1 - x, H - 1 - y) < 22 + 1e-2
        assert near_threshold or at_border, (i, eig[i], stt[i], rs[i], nxt[i], rn[i])
    both = (stt == 1) & (rs == 1)
    d = np.abs(nxt[both] - rn[both]).max(axis=1)
    assert np.percentile(d, 99) < 1e-2 and np.median(d) < 1e-3, (np.percentile(d, 99), np.median(d))
    ref, _, _ = t.klt_track(g0, g1, pts, 21, 3, 30, 0.03)
    assert np.array_equal(ref, nxt)                                              # the same kernel as dynofront_klt_track
