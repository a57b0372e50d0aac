"""dynofront_stereo_match on the device: bit-identical with dynofront_stereo_track + host compaction +
dynofront_find_fundamental_batch + the restatement's per-feature loop; against tests/stereo_oracle.py fed the call's own LK result
(F and mask through the RANSAC trace, with test_fundamental_gpu's proofs); the LK against cv2; a 20-frame streaming run whose
temporal outputs the stereo calls leave untouched; the early returns, LMedS, a failed RANSAC, every state and the refusals."""
import numpy as np
import pytest

import fundamental_oracle as FO
import stereo_oracle as SO
from dynosam_b200.synth_frames import SyntheticStream, W, H
from test_fundamental_gpu import _check

pytestmark = pytest.mark.gpu
FX, B = SO.FX, SO.BASELINE


def _tracker():
    from dynosam_b200.frontend import FeatureTrackerGPU
    return FeatureTrackerGPU(W, H)


def _composition(t, left, right, pts, prm=None):
    """the existing calls: dynofront_stereo_track's LK, compaction on the host, dynofront_find_fundamental_batch, the loop"""
    rp, st, _, _ = t.stereo_track(left, right, pts, FX, B)
    good = np.flatnonzero(st)
    if len(pts) < 8 or len(good) < 8:
        return rp, st, None
    r = t.find_fundamental_batch([(pts[good], rp[good])], prm)
    state, depth, ru = SO.per_feature(pts, rp, st, r["masks"][0], FX, B)
    return rp, st, dict(F=r["F"][0][0], status=int(r["status"][0]), mask=r["masks"][0], state=state, depth=depth, right_u=ru)


def _assert_same_as_composition(d, comp, pts):
    rp, st, c = comp
    if len(pts) >= 8:
        assert np.array_equal(d["right_pts"], rp) and np.array_equal(d["lk_status"], st)
    assert d["n_tracked"] == (int(st.sum()) if len(pts) >= 8 else 0)
    if c is None:
        assert not d["matched"] and (d["state"] == SO.UNTOUCHED).all() and d["fund_status"] == -1
        assert np.isnan(d["depth"]).all() and np.isnan(d["right_u"]).all() and not d["F"].any()
        return
    assert d["matched"] and d["fund_status"] == c["status"] and np.array_equal(d["F"], c["F"])
    assert np.array_equal(d["state"], c["state"])
    assert np.array_equal(d["depth"], c["depth"], equal_nan=True) and np.array_equal(d["right_u"], c["right_u"], equal_nan=True)
    assert d["n_inliers"] == int(c["mask"].sum()) and d["n_stereo"] == int((c["state"] == SO.MATCHED).sum())


def test_bit_identical_with_the_existing_calls():
    s = SyntheticStream(n_objects=10, seed=42)
    t = _tracker()
    for k in (0, 5, 12):
        left, right, _, pts = SO.c4_stereo_frame(s, k)
        d = t.stereo_match(pts, FX, B, left=left, right=right)
        _assert_same_as_composition(d, _composition(t, left, right, pts), pts)
        assert d["n_stereo"] > 500, d["n_stereo"]


def _device_trace(t, d, cap):
    tr = t.fundamental_trace(cap)
    rec = tr["record"][0]
    good = np.flatnonzero(d["lk_status"])
    F3 = np.zeros((3, 3, 3)); F3[0] = d["F"]
    return dict(record=rec, status=d["fund_status"], iterations=int((~np.isnan(rec[:, 0])).sum()), groups=int(tr["groups"][0]),
                rejected=int(tr["rejected"][0]), best=(int(tr["best"][0]), int(tr["best_root"][0])), success=int(tr["success"][0]),
                n_models=1 if d["fund_status"] in (FO.OK, FO.LMEDS) else 0, F=F3, n_inl=d["n_inliers"],
                mask=(d["state"][good] != SO.EPIPOLAR).astype(np.uint8))


def test_matches_the_oracle_on_its_own_lk():
    s = SyntheticStream(n_objects=10, seed=7)
    t = _tracker()
    cap = 1000
    t.fundamental_record(cap)
    proven = []
    for k in (1, 4, 9, 16):
        left, right, _, pts = SO.c4_stereo_frame(s, k)
        d = t.stereo_match(pts, FX, B, left=left, right=right)
        o = SO.stereo_match(None, None, pts, FX, B, lk=(d["right_pts"], d["lk_status"]))
        good = np.flatnonzero(d["lk_status"])
        a, b = pts[good], d["right_pts"][good]
        ro = FO.find_fundamental(a, b)
        why = _check(f"c4_{k}", a, b, _device_trace(t, d, cap), ro)
        assert d["matched"] == o["matched"] and (d["n_tracked"], d["fund_status"]) == (o["n_tracked"], o["fund_status"])
        diff = d["state"] != o["state"]
        if diff.any():                                     # only on mask points _check proved to sit on their threshold margin
            assert why is not None and (d["lk_status"][diff] == 1).all(), (k, why)
            proven.append(why)
        same = ~diff
        assert np.array_equal(d["depth"][same], o["depth"][same], equal_nan=True)
        assert np.array_equal(d["right_u"][same], o["right_u"][same], equal_nan=True)
        if not diff.any():
            assert (d["n_inliers"], d["n_stereo"]) == (o["n_inliers"], o["n_stereo"])
    t.fundamental_record(0)
    print("proven differences:", proven)


def test_lk_matches_opencv():
    from oracle import frontend_oracle as FOR
    s = SyntheticStream(n_objects=10, seed=42)
    t = _tracker()
    agree = []
    for k in (2, 8):
        left, right, _, pts = SO.c4_stereo_frame(s, k)
        d = t.stereo_match(pts, FX, B, left=left, right=right)
        rp, st, _, _ = FOR.stereo_track(left, right, pts, FX, B)
        agree.append(d["lk_status"] == st)
        both = (d["lk_status"] == 1) & (st == 1)
        assert np.percentile(np.abs(d["right_pts"][both] - rp[both]).max(axis=1), 99) < 1e-2
    assert np.concatenate(agree).mean() >= 0.99


def _dynamic_features(mask, rng, per_object=40):
    kp, lab = [], []
    for oid in sorted(set(np.unique(mask).tolist()) - {0}):
        ys, xs = np.nonzero(mask == oid)
        sel = rng.choice(len(ys), min(per_object, len(ys)), replace=False)
        kp.append(np.stack([xs[sel] + 0.5, ys[sel] + 0.5], 1)); lab += [oid]*len(sel)
    kp = np.concatenate(kp).astype(np.float32) if kp else np.zeros((0, 2), np.float32)
    n = len(kp)
    return kp, np.array(lab, np.int32), np.zeros(n, np.int32), np.arange(n, dtype=np.int64)


def _objects(m):
    objs, bb = [], []
    for oid in sorted(set(np.unique(m).tolist()) - {0}):
        ys, xs = np.nonzero(m == oid)
        objs.append(oid); bb.append((xs.min() + 2, ys.min() + 2, max(xs.max() - xs.min() - 3, 1), max(ys.max() - ys.min() - 3, 1)))
    return objs, np.array(bb, np.int32).reshape(-1, 4)


def test_streaming_leaves_the_temporal_pair_alone():
    from dynosam_b200.frontend import FrontendError
    s = SyntheticStream(n_objects=10, seed=42)
    a, b = _tracker(), _tracker()                          # a: with the stereo calls, b: without
    rng = np.random.default_rng(4)
    c = _tracker()
    prev_pts = None; prev_mask = None; stats = np.zeros(5, np.int64)
    for k in range(20):
        left, right, mask, pts = SO.c4_stereo_frame(s, k)
        left, mask, flow = (np.ascontiguousarray(x) for x in (left, mask, s.frame(k)[2]))
        for t in (a, b):
            t.next_frame(left, flow, mask)
        with pytest.raises(FrontendError):                 # next_frame made the previous right image stale
            a.stereo_match(pts, FX, B)
        a.set_right(right)
        outs = {}
        for name, t in (("a", a), ("b", b)):
            r = {}
            if prev_pts is not None:
                r["ktp"] = t.klt_track_points(None, None, prev_pts)
            if name == "a":
                r1 = t.stereo_match(pts, FX, B)
                shifted = pts + np.float32([0.37, -0.21])
                r2 = t.stereo_match(shifted, FX, B)
                e1 = t.stereo_match(pts, FX, B, left=left, right=right)         # explicit images: same result, temporal pair untouched
                e2 = t.stereo_match(shifted, FX, B, left=left, right=right)
                for x, y in ((r1, e1), (r2, e2)):
                    for key in ("state", "depth", "right_u", "right_pts", "lk_status", "F"):
                        assert np.array_equal(x[key], y[key], equal_nan=True), (k, key)
                    assert (x["matched"], x["fund_status"], x["n_tracked"], x["n_inliers"], x["n_stereo"]) == \
                           (y["matched"], y["fund_status"], y["n_tracked"], y["n_inliers"], y["n_stereo"])
                _assert_same_as_composition(r1, _composition(c, left, right, pts), pts)
                stats += np.bincount(r1["state"], minlength=5)
            if prev_mask is not None:
                objs, bb = _objects(mask)
                r["dklt"] = t.track_dynamic_klt(None, None, *dyn, objs, bb, 1000)
            outs[name] = r
        for key in outs["a"]:
            for x, y in zip(outs["a"][key], outs["b"][key]) if key == "ktp" else ((outs["a"][key][q], outs["b"][key][q]) for q in
                                                                                    ("lk_pts", "lk_status", "state", "keypoint", "tracklet",
                                                                                     "detection_mask", "tracking_mask")):
                assert (x is None and y is None) or np.array_equal(x, y), (k, key)
        prev_pts = pts; prev_mask = mask; dyn = _dynamic_features(mask, rng)
    assert stats[SO.MATCHED] > 10000 and stats[SO.EPIPOLAR] > 0, stats


def _hand_pair():
    """a textured left image with a flat patch (LK fails there), and a right image shifted by 9-13 px per 300-column band, except
    the bottom 70 rows (zero disparity) and rows 20-90, shifted 6 rows as well (off their epipolar lines)"""
    left, _, _ = SyntheticStream(n_objects=6, seed=3).frame(5)
    left = left.copy(); left[150:210, 600:660] = 128
    cols = np.arange(W); src = np.minimum(cols + 9 + cols//300, W - 1)
    right = left[:, src].copy()
    right[H - 70:] = left[H - 70:]
    right[20:90] = np.roll(left, -6, axis=0)[20:90][:, src]
    return left, right


def test_edge_cases_states_and_refusals():
    from dynosam_b200.frontend import FrontendError, FundamentalParams
    left, right = _hand_pair()
    rng = np.random.default_rng(9)
    t = _tracker()
    seen = set()

    def run(pts, expect_status=None, prm=None):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
        d = t.stereo_match(pts, FX, B, prm, left=left, right=right)
        _assert_same_as_composition(d, _composition(t, left, right, pts, prm), pts)
        if expect_status is not None:
            assert d["fund_status"] == expect_status, (d["fund_status"], expect_status)
        seen.update(np.unique(d["state"]).tolist())
        return d

    def tex(n, x0=30):                                                     # textured, between the off-line rows and the bottom band
        return np.stack([rng.uniform(x0, W - 60, n), rng.uniform(100, H - 80, n)], 1)

    def tex_ok(n):                                                         # ... and clear of the flat patch
        return tex(n, 700)

    d = run(np.zeros((0, 2)))
    assert not d["matched"] and d["state"].size == 0
    d = run(tex_ok(7))                                                     # n = 7: nothing runs
    assert not d["matched"] and t.fundamental_trace()["groups"].size == 0
    p = np.concatenate([tex_ok(7), [[630.0, 180.0]]])                      # 8 inputs, the one in the flat patch lost
    d = run(p)
    assert d["n_tracked"] == 7 and d["lk_status"][7] == 0 and not d["matched"]
    tr = t.fundamental_trace()
    assert tr["groups"].tolist() == [0]                                    # one problem of 0 points
    run(tex_ok(12), FO.LMEDS)                                              # 8-14 tracked: LMedS
    row = np.stack([np.linspace(700, 1150, 20), np.full(20, 150.0)], 1)   # one row: every subset collinear
    d = run(row, FO.FAILED)
    assert d["matched"] and (d["state"][d["lk_status"] == 1] == SO.EPIPOLAR).all() and not d["F"].any()
    mix = np.concatenate([tex(250), np.stack([rng.uniform(40, W - 60, 25), rng.uniform(30, 80, 25)], 1),        # off the line
                          np.stack([rng.uniform(40, W - 60, 25), rng.uniform(H - 55, H - 15, 25)], 1),        # zero disparity
                          np.stack([rng.uniform(621, 639, 10), rng.uniform(171, 189, 10)], 1)])               # flat: lost
    d = run(mix, FO.OK)
    assert {SO.MATCHED, SO.LOST, SO.EPIPOLAR, SO.DISPARITY} <= set(np.unique(d["state"]).tolist()), np.bincount(d["state"])
    run(mix, prm=FundamentalParams(threshold_px=3.0, confidence=0.999, max_iters=50))
    assert seen == {SO.UNTOUCHED, SO.MATCHED, SO.LOST, SO.EPIPOLAR, SO.DISPARITY}, seen
    for bad in (FundamentalParams(threshold_px=0.0), FundamentalParams(confidence=1.0)):
        with pytest.raises(FrontendError):
            t.stereo_match(mix, FX, B, bad, left=left, right=right)
    nan = mix.copy(); nan[3, 1] = np.nan
    with pytest.raises(FrontendError):
        t.stereo_match(nan, FX, B, left=left, right=right)
    with pytest.raises(FrontendError):
        t.stereo_match(mix, FX, B, left=left)                              # one image only
    with pytest.raises(FrontendError):
        _tracker().stereo_match(mix, FX, B)                                # no resident frame
