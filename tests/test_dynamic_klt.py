"""FeatureTracker::trackDynamicKLT on the device (dynofront_track_dynamic_klt), CPU side.

The oracle (tests/dynamic_klt_oracle.py) is pinned here against independent code: the shared local-maximum decomposition the
device uses for the per-object goodFeaturesToTrack against cv2.goodFeaturesToTrack on every object, its IoU against an
integer-rectangle formula and its float bounding rectangle against cv2.boundingRect, and a hand-built frame (with an exact
LK result) that takes every path of requiresSampling and of the per-feature tests.
GPU (tests/test_dynamic_klt_gpu.py): the device against the oracle, bit for bit.
"""
import os

import numpy as np
import pytest

import detection_oracle as DO
import dynamic_klt_oracle as KO
from dynosam_b200.synth_frames import SyntheticStream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _texture(h, w, seed):
    import cv2
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(cv2.GaussianBlur(rng.integers(0, 256, (h, w)).astype(np.uint8), (0, 0), 1.2))


@pytest.mark.skipif(not DO.opencv_float_orders_apply(),
                    reason="cv2 does not run OpenCV's AVX2 + FMA3 code path, whose eigen-image float orders the device reproduces")
@pytest.mark.parametrize("which", ["c4_3", "c4_8", "texture"])
def test_shared_local_max_decomposition_matches_cv2(which):
    """One pass of raw 3x3 local maxima plus a per-object threshold and mask gives cv2.goodFeaturesToTrack's corners, in
    content and order, for every object (also with discs cut out of the detection mask and a tiny object)."""
    import cv2
    rng = np.random.default_rng(4)
    if which == "texture":
        g = _texture(251, 333, 2); m = np.zeros(g.shape, np.int32)
        m[20:120, 30:150] = 1; m[100:240, 160:320] = 2; m[5:8, 5:9] = 3; m[130:200, 10:90] = 4
    else:
        g, m, _ = SyntheticStream(n_objects=10, seed=42).frame(int(which[3:]))
        g = np.ascontiguousarray(g.astype(np.uint8)); m = m.astype(np.int32)
    det = np.full(g.shape, 255, np.uint8); det[:, :25] = 0
    ys, xs = np.nonzero(m > 0)
    for s in rng.choice(len(ys), min(400, len(ys)), replace=False):
        cv2.circle(det, (int(xs[s]), int(ys[s])), 2, 0, cv2.FILLED)
    objects = sorted(set(np.unique(m).tolist()) - {0}) + [77]                     # 77: not in the image, empty mask
    eig = cv2.cornerMinEigenVal(g, 3, 3)
    for prm in (KO.Params(), KO.Params(max_features=40, min_distance=5, quality_level=0.05)):
        dec = KO.gftt_decomposed(eig, m, det, objects, prm)
        total = 0
        for oid in objects:
            ref = KO.gftt(g, m, det, oid, prm)
            assert dec[oid] == ref, (which, oid, len(dec[oid]), len(ref))
            total += len(ref)
        assert total > 50


def _rect_pixels(r):
    x, y, w, h = r
    return {(i, j) for i in range(x, x + max(w, 0)) for j in range(y, y + max(h, 0))}


def test_iou_and_bounding_rect():
    """calculateIoU with cv::Rect's intersection equals |A & B| / |A | B| over the pixel sets; the float bounding rectangle is
    floor(min) .. floor(max) inclusive, as cv2.boundingRect computes it"""
    import cv2
    rng = np.random.default_rng(8)
    for _ in range(400):
        a = tuple(int(v) for v in (rng.integers(-5, 30), rng.integers(-5, 30), rng.integers(0, 20), rng.integers(0, 20)))
        b = tuple(int(v) for v in (rng.integers(-5, 30), rng.integers(-5, 30), rng.integers(0, 20), rng.integers(0, 20)))
        pa, pb = _rect_pixels(a), _rect_pixels(b)
        union = len(pa | pb)
        want = 0.0 if union == 0 else len(pa & pb)/union
        assert KO.calculate_iou(a, b) == pytest.approx(want, abs=0, rel=1e-15), (a, b)
    for _ in range(300):
        k = int(rng.integers(1, 12))
        pts = rng.uniform(-3, 50, (k, 2)).astype(np.float32)
        sel = rng.random(k) < 0.3; pts[sel] = np.round(pts[sel])                  # whole-pixel points too
        lo = np.floor(pts.min(0)).astype(int); hi = np.floor(pts.max(0)).astype(int)
        want = (int(lo[0]), int(lo[1]), int(hi[0] - lo[0] + 1), int(hi[1] - lo[1] + 1))
        assert KO.bounding_rect(pts) == want == tuple(cv2.boundingRect(pts.reshape(-1, 1, 2)))


def test_hand_built_frame_takes_every_path():
    """The oracle on the hand-built frame with the exact LK result: each sampling reason, the skipped object, K = 0, an LK
    point outside the image and a feature masked by an earlier accepted disc (and not counted)"""
    prev_g, cur_g, mask, kp, lab, age, tid, objects, inner, lk = KO.hand_built_frame()
    r = KO.track_dynamic_klt(cur_g, mask, None, kp, lab, age, tid, lk, np.ones(len(kp), np.uint8), objects, inner, KO.Params(), 1000)
    assert r["reasons"] == {1: ["new"], 2: ["skipped"], 3: ["old"], 4: ["few"], 5: ["iou"], 6: ["iou"], 7: []}
    st = {f: dict(zip(r["status"]["object_id"].tolist(), r["status"][f].tolist())) for f in KO.STATUS_FIELDS}
    assert st["object_new"] == {0: 0, 1: 1, 2: 0, 3: 0, 4: 0, 5: 0, 6: 0, 7: 0}
    assert st["sampled"] == {0: 0, 1: 1, 2: 0, 3: 1, 4: 1, 5: 1, 6: 1, 7: 0}
    assert st["num_track"] == {0: 0, 1: 0, 2: 0, 3: 25, 4: 5, 5: 30, 6: 210, 7: 30}
    assert st["num_previous_track"][4] == 5                                     # the masked feature is not counted
    assert st["num_tracked_with_different_label"][2] == 1 and st["exists"][2] == 1
    assert st["num_tracked_with_background_label"][0] == 1
    assert st["num_sampled"][6] == 0 and st["num_sampled"][1] > 0 and st["num_sampled"][3] > 0      # K = 0 for object 6
    assert r["n_outside_image"] == 1
    s = r["state"]
    assert (s == KO.MASKED).sum() == 1 and s[31] == KO.MASKED and (s == KO.OUTSIDE).sum() == 1
    # tracked features first, by ascending label, each group in input order; then the new ones with ids from 1000
    ntr = int((r["source"] >= 0).sum())
    assert ntr == 300 and (r["source"][ntr:] == -1).all()
    assert (np.diff(r["label"][:ntr]) >= 0).all() and all((np.diff(r["source"][:ntr][r["label"][:ntr] == L]) > 0).all() for L in (3, 4, 5, 6, 7))
    assert list(r["tracklet"][ntr:]) == list(range(1000, r["next_tracklet_id"]))
    new_labels = r["label"][ntr:]
    assert [int(L) for L in dict.fromkeys(new_labels.tolist())] == [1, 3, 4, 5]
    assert (r["age"][ntr:] == 0).all() and (r["age"][:ntr] >= 1).all()
    flow = r["measured_flow"][s == KO.TRACKED]
    assert np.allclose(flow, [-4.0, 0.0])
    assert (r["tracking_mask"][mask == 6] == 6).sum() > 0 and r["detection_mask"][40, 390] == 0


def test_dynamic_klt_exports_and_defaults():
    import ctypes as C

    import __graft_entry__ as g
    if not os.path.exists(os.path.join(ROOT, "dynosam_b200", "libdynofront.so")):
        g.build()
    from dynosam_b200 import frontend
    lib = frontend.load()
    for s in ("dynofront_track_dynamic_klt", "dynofront_klt_dynamic_default_params"):
        assert s in frontend.EXPORTS and hasattr(lib, s), s
    c = frontend.KltDynamicParamsC()
    lib.dynofront_klt_dynamic_default_params(C.byref(c))
    p = frontend.KltDynamicParams().c()
    for name, _ in frontend.KltDynamicParamsC._fields_:
        if name == "track":
            for f, _ in frontend.TrackParamsC._fields_:
                assert getattr(c.track, f) == getattr(p.track, f), f
        else:
            assert getattr(c, name) == getattr(p, name), name
    kp = KO.Params()
    assert (p.track.max_dynamic_feature_age, p.track.min_distance, p.max_features, p.quality_level, p.age_buffer, p.min_tracks, p.min_iou) == \
        (kp.max_dynamic_feature_age, kp.min_distance, kp.max_features, kp.quality_level, kp.age_buffer, kp.min_tracks, kp.min_iou)
