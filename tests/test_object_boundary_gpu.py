"""dynofront_object_boundary on the device against the literal cv2 composition of tests/boundary_oracle.py, bit for bit: the
boundary mask, the objects, bb and inner_bb on every case of tests/boundary_cases.py and at 1920 x 1080.  The hand-off: on a
streaming C4 run, detect_static, track_dynamic_klt, track_dynamic and dense_cloud give the same outputs after object_boundary as
after an upload of the oracle's mask through next_frame.  The refusals leave the resident mask as it was."""
import numpy as np
import pytest

import boundary_cases as BC
import boundary_oracle as BO
import frame_cases as FC

pytestmark = pytest.mark.gpu
CASES = BC.cases()
CALIB5 = np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854])


def _tracker(w, h):
    from dynosam_b200.frontend import FeatureTrackerGPU
    return FeatureTrackerGPU(w, h)


def _run(M, t):
    H, W = M.shape
    tr = _tracker(W, H)
    tr.set_frame(np.zeros((H, W, 2), np.float32), M, None)
    out = tr.object_boundary(t, want_mask=True)
    tr.close()
    return out


def _assert_same(got, ref, what):
    for k, x, y in zip(("objects", "bb", "inner_bb", "mask"), got, ref):
        assert x.shape == y.shape and np.array_equal(x, y), (what, k)


def _resident_boundary(tr):
    """the boundary mask on the device, as track_dynamic's detection mask with no features"""
    from dynosam_b200.frontend import TrackParams
    e = np.zeros(0)
    out = tr.track_dynamic(e.reshape(0, 2), e.astype(np.int32), e.astype(np.int32), e.astype(np.int64), TrackParams(), 0)
    return out[7]


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_oracle(name):
    M, t = CASES[name]
    _assert_same(_run(M, t), BO.object_boundary(M, t), name)


def test_full_hd_thickness_68():
    case = FC.Case("hd_1920x1080", 1920, 1080, ())
    for n_obj in (5, 20):
        M = FC.frame(case, 3, n_objects=n_obj)[1]
        t = BO.thickness(1920, 1080)
        assert t == 68
        _assert_same(_run(M, -1), BO.object_boundary(M, t), n_obj)


def test_default_thickness_is_the_scaled_one():
    for name in FC.DATASET:
        c = FC.CASES[name]
        M = FC.frame(c, 5)[1]
        _assert_same(_run(M, -1), BO.object_boundary(M, BO.thickness(c.w, c.h)), name)


def test_hand_off_equals_uploaded_mask_on_c4_stream():
    from dynosam_b200.frontend import DetectParams, KltDynamicParams, TrackParams
    from dynosam_b200.synth_frames import SyntheticStream
    W, H = 1242, 375
    st = SyntheticStream(n_objects=10, seed=42)
    a = _tracker(W, H); b = _tracker(W, H)
    prev = (np.zeros((0, 2), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int64))
    cur_static = np.zeros((0, 2)); nid = 1000; tracked = 0
    for k in range(8):
        g, m, f = FC.c4(k)
        depth = np.ascontiguousarray(st.depth(k), np.float64)
        a.next_frame(g, f, m)
        objs, bb, ib, mask = a.object_boundary(want_mask=True)
        ref = BO.object_boundary(m, BO.thickness(W, H))
        _assert_same((objs, bb, ib, mask), ref, k)
        b.next_frame(g, f, m, ref[3])
        outs = []
        for tr in (a, b):
            tr.set_depth(depth)
            ds = tr.detect_static(None, cur_static, DetectParams(), nid)
            kl = tr.track_dynamic_klt(None, None, *prev, objs, ib, nid, KltDynamicParams()) if k > 0 else None
            td = tr.track_dynamic(prev[0].astype(np.float64), prev[1], prev[2], prev[3], TrackParams(), nid)
            dc = tr.dense_cloud(CALIB5)
            outs.append((ds, kl, td, dc))
        (da, ka, ta, ca), (db, kb, tb, cb) = outs
        for x, y in zip(da, db):
            assert np.array_equal(x, y)
        for x, y in zip(ta, tb):
            assert np.array_equal(x, y)
        for x, y in zip(ca, cb):
            assert np.array_equal(x, y)
        if ka is not None:
            for key in ("lk_pts", "lk_status", "state", "measured_flow", "keypoint", "age", "tracklet", "label", "source", "detection_mask",
                        "tracking_mask"):
                assert np.array_equal(ka[key], kb[key]), key
            for fld, v in ka["status"].items():
                assert np.array_equal(v, kb["status"][fld]), fld
            tracked += int(ka["tracked"].sum())
            nid = ka["next_tracklet_id"]
            prev = (ka["keypoint"].astype(np.float32), ka["label"], ka["age"], ka["tracklet"])
        else:
            prev = (np.zeros((0, 2), np.float32),) + prev[1:]
            nid += 1
        cur_static = da[0][:200]
        assert (mask == 0).any() and (ca[3][mask == 0] == 0).all()
    assert tracked > 0
    a.close(); b.close()


def test_refused_after_propagate_and_accepted_next_frame():
    from dynosam_b200.frontend import FrontendError, TrackParams
    a = _tracker(1242, 375)
    g0, m0, f0 = FC.c4(0); g1, m1, f1 = FC.c4(1); g2, m2, f2 = FC.c4(2)
    a.next_frame(g0, f0, m0); a.next_frame(g1, f1, m1)
    before = a.object_boundary(want_mask=True)[3]
    ys, xs = np.nonzero(m0 > 0)
    kp = np.stack([xs[::50], ys[::50]], 1).astype(np.float64); lab = m0[ys[::50], xs[::50]]
    a.propagate_mask_resident(kp, lab, TrackParams())
    with pytest.raises(FrontendError, match="propagate"):
        a.object_boundary()
    assert np.array_equal(_resident_boundary(a), before)
    a.next_frame(g2, f2, m2)
    _assert_same(a.object_boundary(want_mask=True), BO.object_boundary(m2, 15), "next frame")
    a.close()


def test_refusals_leave_the_resident_mask():
    from dynosam_b200.frontend import FrontendError
    W, H = 160, 120
    fresh = _tracker(W, H)
    with pytest.raises(FrontendError, match="no motion mask"):
        fresh.object_boundary()
    fresh.close()
    rng = np.random.default_rng(3)
    M = BC.ellipses(rng, H, W, 5, r=(5, 25))
    uploaded = np.full((H, W), 255, np.uint8); uploaded[40:60] = 0
    tr = _tracker(W, H)
    flow = np.zeros((H, W, 2), np.float32)
    for bad_value in (256, -1, 1000):
        bad = M.copy(); bad[7, 9] = bad_value
        tr.set_frame(flow, bad, uploaded)
        with pytest.raises(FrontendError, match=r"\[0, 255\]"):
            tr.object_boundary()
        assert np.array_equal(_resident_boundary(tr), uploaded)
    tr.set_frame(flow, M, uploaded)
    with pytest.raises(FrontendError, match="thickness"):
        tr.object_boundary(BC.CAP + 1)
    assert np.array_equal(_resident_boundary(tr), uploaded)
    got = tr.object_boundary(BC.CAP, want_mask=True)
    _assert_same(got, BO.object_boundary(M, BC.CAP), "cap")
    assert np.array_equal(_resident_boundary(tr), got[3])
    tr.close()


def test_capacity_empty_and_repeats():
    M, t = CASES["all_255_labels"]
    H, W = M.shape
    tr = _tracker(W, H)
    tr.set_frame(np.zeros((H, W, 2), np.float32), M, None)
    full = tr.object_boundary(t, want_mask=True)
    again = tr.object_boundary(t, want_mask=True)
    _assert_same(again, full, "repeat")
    part = tr.object_boundary(t, want_mask=True, capacity=10)
    assert tr.last_n_objects == 255 and len(part[0]) == 10
    for x, y in zip(part[:3], full[:3]):
        assert np.array_equal(x, y[:10])
    assert np.array_equal(part[3], full[3])
    none = tr.object_boundary(t, capacity=0)
    assert tr.last_n_objects == 255 and len(none[0]) == 0
    tr.set_frame(np.zeros((H, W, 2), np.float32), np.zeros((H, W), np.int32), None)
    objs, bb, ib, mask = tr.object_boundary(t, want_mask=True)
    assert len(objs) == 0 and bb.shape == (0, 4) and (mask == 255).all()
    tr.close()
