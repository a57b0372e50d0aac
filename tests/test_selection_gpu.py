"""Feature selection on the device, against the CPU oracle (tests/selection_oracle.py): bit-exact.

  * the batched range-tree ANMS: selected indices and their order, many lists (n, K, tolerance) in one launch;
  * sample_dynamic on C4 frames (1242x375): counts, num_sampled, zero_flow, key-points, flows, predicted key-points,
    tracklet ids, labels and next_tracklet_id, with and without the detection mask left by track_dynamic, with
    num_track near 0 and near max_dynamic_features_per_frame (200); streaming and call-by-call runs agree.
"""
import numpy as np
import pytest

import selection_oracle as SO
from dynosam_b200.synth_frames import SyntheticStream

W, H = 1242, 375


@pytest.mark.gpu
def test_anms_batched_bit_exact():
    from dynosam_b200.frontend import FeatureTrackerGPU
    rng = np.random.default_rng(3)
    lists, ks, tols = [], [], []
    for n in (0, 1, 16, 17, 1000, 50000):
        for k in (0, 1, 2, 5, 199, 200, 800):
            for tol in (0.01, 0.1):
                if n == 1000 and k == 200:                           # a dense object region: every pixel of a 40 x 25 patch
                    yy, xx = np.mgrid[200:225, 600:640]
                    xy = np.stack([xx.ravel(), yy.ravel()], 1)
                else:
                    flat = rng.choice(W*H, n, replace=False)
                    xy = np.stack([flat % W, flat//W], 1)
                lists.append(xy.astype(np.int32)); ks.append(k); tols.append(tol)
    t = FeatureTrackerGPU(W, H)
    got = t.anms_range_tree(lists, ks, np.array(tols, np.float32))
    for xy, k, tol, g in zip(lists, ks, tols, got):
        ref = SO.anms_range_tree(xy, k, np.float32(tol), W, H)
        assert g.tolist() == ref, (len(xy), k, tol, len(g), len(ref))
    assert any(len(g) > 0 for g in got)


def _dynamic_inputs(rng, m0, f0, per_object=150):
    kps, labs = [], []
    for lab in np.unique(m0):
        if lab == 0:
            continue
        ys, xs = np.nonzero(m0 == lab)
        sel = rng.choice(len(ys), size=min(per_object, len(ys)), replace=False)
        kps += [(x + 0.5 + f0[y, x, 0], y + 0.5 + f0[y, x, 1]) for y, x in zip(ys[sel], xs[sel])]; labs += [lab]*len(sel)
    kps = np.array(kps); labs = np.array(labs, np.int32)
    ok = (kps[:, 0] > 1) & (kps[:, 0] < W - 1) & (kps[:, 1] > 1) & (kps[:, 1] < H - 1)
    kps, labs = kps[ok], labs[ok]
    return kps, labs, rng.integers(0, 22, len(labs)).astype(np.int32), np.arange(len(labs), dtype=np.int64)


def _assert_same(g, o):
    for key in ("counts", "num_sampled", "zero_flow", "tracklet", "label"):
        assert np.array_equal(g[key], o[key]), key
    for key in ("keypoint", "flow", "predicted"):
        assert g[key].shape == o[key].shape and np.array_equal(g[key], o[key]), key     # doubles from the same floats
    assert g["next_tracklet_id"] == o["next_tracklet_id"]


@pytest.mark.gpu
@pytest.mark.parametrize("with_det,near", [(False, 0), (True, 0), (True, 200)])
def test_sample_dynamic_bit_exact(with_det, near):
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(8)
    st = SyntheticStream(n_objects=10, seed=42)
    _, m0, f0 = st.frame(3); _, m1, f1 = st.frame(4)
    f1 = f1.copy(); f1[60:90, 300:380] = 0.0                          # zero-flow pixels are counted, not sampled
    objs = [int(o) for o in np.unique(m1) if o != 0] + [77]          # 77: an object with no pixels
    ntr = (rng.integers(0, 6, len(objs)) if near == 0 else rng.integers(196, 204, len(objs))).astype(np.int32)   # K in {0 .. 4} near 200
    prm = TrackParams(shrink_row=2, shrink_col=3)
    fprm = FO.TrackParams(20, 2, 2, 3)
    t = FeatureTrackerGPU(W, H)
    det = None
    if with_det:
        kp, lab, age, tid = _dynamic_inputs(rng, m0, f0)
        t.set_frame(f1, m1, None)
        t.track_dynamic(kp, lab, age, tid, prm, 1000, want_masks=False)     # leaves its detection mask on the device
        det = FO.track_dynamic(kp, lab, age, tid, f1, m1, None, fprm, 1000)[7]
    else:
        t.set_frame(f1, m1, None)
    g = t.sample_dynamic(objs, ntr, prm, 5000)
    o = SO.sample_dynamic(f1, m1, det, objs, ntr, fprm, 5000)
    _assert_same(g, o)
    assert g["counts"][-1] == 0 and g["num_sampled"][-1] == 0 and g["zero_flow"].sum() > 0
    if near == 0:                                                    # the search often ends on its fall-back, below K (1 - 0.01)
        assert (g["num_sampled"][:-1] > 100).all()
    assert t.last_ms > 0


@pytest.mark.gpu
def test_sample_dynamic_streaming_equals_call_by_call():
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    rng = np.random.default_rng(4)
    stream = SyntheticStream(n_objects=8, seed=9)
    frames = [tuple(np.ascontiguousarray(a) for a in stream.frame(k)) for k in range(3)]
    frames = [(g.astype(np.uint8), m.astype(np.int32), f.astype(np.float32)) for g, m, f in frames]
    prm = TrackParams()
    a = FeatureTrackerGPU(W, H); b = FeatureTrackerGPU(W, H)
    a.next_frame(frames[0][0], frames[0][2], frames[0][1])
    for k in (1, 2):
        g0, m0, f0 = frames[k-1]; g1, m1, f1 = frames[k]
        kp, lab, age, tid = _dynamic_inputs(rng, m0, f0, per_object=120)
        objs = list(range(1, 9)); ntr = rng.integers(0, 200, 8).astype(np.int32)
        a.next_frame(g1, f1, m1)
        a.propagate_mask_resident(kp, lab, prm, min_votes=20)
        a.track_dynamic(kp, lab, age, tid, prm, 9000, want_masks=False)
        ra = a.sample_dynamic(objs, ntr, prm, 20000)
        cur = b.propagate_mask(kp, lab, m0, f0, m1, prm, min_votes=20)
        b.set_frame(f1, cur, None)
        b.track_dynamic(kp, lab, age, tid, prm, 9000, want_masks=False)
        rb = b.sample_dynamic(objs, ntr, prm, 20000)
        _assert_same(ra, rb)
        assert ra["num_sampled"].sum() > 0


@pytest.mark.gpu
def test_anms_rejects_u16_wrap():
    """The reference's range tree stores u16 coordinates, so x + width above 65535 would wrap; such lists are refused."""
    from dynosam_b200.frontend import FeatureTrackerGPU, FrontendError
    t = FeatureTrackerGPU(W, H)
    with pytest.raises(FrontendError):
        t.anms_range_tree([np.array([[65530, 10], [65000, 20]])], 2, 0.01)          # widths up to 497 for K = 2 at 1242x375
    assert t.anms_range_tree([np.array([[64000, 10], [64020, 20]])], 2, 0.01)[0].tolist() == \
        SO.anms_range_tree([(64000, 10), (64020, 20)], 2, np.float32(0.01), W, H)


@pytest.mark.gpu
def test_sample_dynamic_capacity():
    """A capacity below the number of new features: the C call writes the first `capacity` of them and reports the total
    (tracklet ids are still handed out for all); the Python wrapper then calls again with room for all."""
    import ctypes as C
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams, _p
    st = SyntheticStream(n_objects=6, seed=13)
    _, m1, f1 = st.frame(2)
    objs = [int(o) for o in np.unique(m1) if o != 0]
    prm = TrackParams()
    t = FeatureTrackerGPU(W, H); t.set_frame(f1, m1, None)
    full = t.sample_dynamic(objs, 0, prm, 100)
    total = len(full["tracklet"])
    assert total > 20
    _assert_same(t.sample_dynamic(objs, 0, prm, 100, capacity=10), full)       # the wrapper's second call
    cap = 10
    o = np.array(objs, np.int32); ntr = np.zeros(len(objs), np.int32)
    counts = np.zeros(len(objs), np.int32); ns = np.zeros(len(objs), np.int32); zero = np.zeros(len(objs), np.int32)
    kp = np.full((cap + 1, 2), -7.0); fl = np.full((cap + 1, 2), -7.0); pk = np.full((cap + 1, 2), -7.0)
    tid = np.full(cap + 1, -7, np.int64); lab = np.full(cap + 1, -7, np.int32)
    nid = C.c_int64(100); nf = C.c_int32(); pc = prm.c()
    t._ck(t.lib.dynofront_sample_dynamic(t.h, len(objs), _p(o), _p(ntr), 200, C.byref(pc), C.byref(nid), _p(counts), _p(ns), _p(zero), cap,
                                         _p(kp), _p(fl), _p(pk), _p(tid), _p(lab), C.byref(nf), None))
    assert nf.value == total and nid.value == 100 + total
    assert np.array_equal(ns, full["num_sampled"]) and np.array_equal(counts, full["counts"])
    assert np.array_equal(kp[:cap], full["keypoint"][:cap]) and np.array_equal(fl[:cap], full["flow"][:cap])
    assert np.array_equal(pk[:cap], full["predicted"][:cap]) and np.array_equal(tid[:cap], full["tracklet"][:cap])
    assert np.array_equal(lab[:cap], full["label"][:cap])
    assert (kp[cap] == -7.0).all() and tid[cap] == -7 and lab[cap] == -7                 # nothing written past capacity
