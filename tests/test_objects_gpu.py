"""The front end's per-object kernels along the object axis (tests/object_cases.py), bit for bit against the oracles: up to 64
objects in a call, labels up to 2^31 - 1 (and negative ones where no object list is involved), object lists in every order,
listed objects without pixels and present labels that are not listed; propagate_mask's vote on hand-built votes; the refusals
of the three object-list entry points.

  * track_dynamic (both masks) against frontend_oracle.track_dynamic;
  * sample_candidates against frontend_oracle.sample_dynamic_candidates, sample_dynamic against selection_oracle.sample_dynamic;
  * track_dynamic_klt against dynamic_klt_oracle, fed the device's own LK result (as test_dynamic_klt_gpu.py);
  * update_depths, back_project and dense_cloud against depth_oracle, and Color::uniqueId at large and negative ids;
  * propagate_mask against frontend_oracle.propagate_mask (votes of any int32 label, libstdc++'s std::sort tie rule).
"""
import numpy as np
import pytest

import depth_oracle as DPO
import detection_oracle as DO
import dynamic_klt_oracle as KO
import object_cases as OC
import selection_oracle as SO
from oracle import frontend_oracle as FO

pytestmark = pytest.mark.gpu
W, H = OC.W, OC.H
NAMES = list(OC.CASES)
CAL = (718.856, 718.856, 0.0, 607.1928, 185.2157)
needs_opencv_orders = pytest.mark.skipif(not DO.opencv_float_orders_apply(),
                                         reason="cv2 does not run OpenCV's AVX2 + FMA3 code path, whose eigen-image float orders the device reproduces")


def _features(rng, m, f, per_object=30):
    """previous dynamic features on every label of mask m (frame k-1): predicted key-point = pixel + jitter + flow"""
    kps, labs = [], []
    for lab in np.unique(m):
        if lab == 0:
            continue
        ys, xs = np.nonzero(m == lab)
        s = rng.choice(len(ys), size=min(per_object, len(ys)), replace=False)
        kps.append(np.stack([xs[s] + rng.uniform(0, 0.9, len(s)) + f[ys[s], xs[s], 0], ys[s] + rng.uniform(0, 0.9, len(s)) + f[ys[s], xs[s], 1]], 1))
        labs.append(np.full(len(s), lab, np.int32))
    kp = np.concatenate(kps); lab = np.concatenate(labs)
    keep = (kp[:, 0] > 1) & (kp[:, 0] < W - 1) & (kp[:, 1] > 1) & (kp[:, 1] < H - 1)
    return kp[keep], lab[keep]


def _tracker(f, m, det=None):
    from dynosam_b200.frontend import FeatureTrackerGPU
    t = FeatureTrackerGPU(W, H); t.set_frame(f, m, det)
    return t


@pytest.mark.parametrize("name", NAMES)
def test_track_dynamic_bit_exact(name):
    from dynosam_b200.frontend import TrackParams
    (_, m0, f0), (_, m1, f1) = OC.frames(OC.CASES[name])
    rng = np.random.default_rng(1)
    kp, lab = _features(rng, m0, f0)
    age = rng.integers(0, 22, len(lab)).astype(np.int32); tid = np.arange(1000, 1000 + len(lab), dtype=np.int64)
    t = _tracker(f1, m1)
    got = t.track_dynamic(kp, lab, age, tid, TrackParams(min_distance=3), 5000)
    ref = FO.track_dynamic(kp, lab, age, tid, f1, m1, None, FO.TrackParams(20, 3, 0, 0), 5000)
    assert 0 < ref[0].sum() < len(lab)
    for k, (a, b) in enumerate(zip(got, ref)):
        assert np.array_equal(a, b), k
    assert set(np.unique(ref[8]).tolist()) <= {0} | {FO.saturate_u8(l) for l in ref[5][ref[0] == 1]}


@pytest.mark.parametrize("name", NAMES)
def test_sample_candidates_and_dynamic_bit_exact(name):
    from dynosam_b200.frontend import TrackParams
    c = OC.CASES[name]
    (_, m0, f0), (_, m1, f1) = OC.frames(c)
    rng = np.random.default_rng(2)
    f1 = f1.copy(); f1[100:104, :] = 0.0                              # zero-flow pixels: counted, not sampled
    objs = list(c.listed)
    prm = TrackParams(shrink_row=2, shrink_col=3); fprm = FO.TrackParams(20, 2, 2, 3)
    t = _tracker(f1, m1)
    cand, zero = t.sample_candidates(objs, prm)
    rc, rz = FO.sample_dynamic_candidates(f1, m1, np.full((H, W), 255, np.uint8), objs, fprm)
    for o in objs:
        assert np.array_equal(cand[o], np.array(rc[o], np.int32)) and zero[o] == rz[o], o
    kp, lab = _features(rng, m0, f0)
    age = rng.integers(0, 22, len(lab)).astype(np.int32); tid = np.arange(len(lab), dtype=np.int64)
    t.track_dynamic(kp, lab, age, tid, prm, 1000, want_masks=False)       # leaves its detection mask on the device
    det = FO.track_dynamic(kp, lab, age, tid, f1, m1, None, fprm, 1000)[7]
    ntr = rng.integers(0, 6, len(objs)).astype(np.int32)
    g = t.sample_dynamic(objs, ntr, prm, 5000)
    o = SO.sample_dynamic(f1, m1, det, objs, ntr, fprm, 5000)
    for key in ("counts", "num_sampled", "zero_flow", "tracklet", "label", "keypoint", "flow", "predicted", "next_tracklet_id"):
        assert np.array_equal(g[key], o[key]), key
    shown = set(np.unique(m1).tolist())
    assert all((g["num_sampled"][i] > 0) == (ob in shown) for i, ob in enumerate(objs))


def _objects_bb(m, objs):
    """inner boxes of the listed objects (each label's bounding box shrunk by 2 px; an absent object gets an empty box)"""
    bb = []
    for oid in objs:
        ys, xs = np.nonzero(m == oid)
        if len(ys) == 0:
            bb.append((0, 0, 0, 0)); continue
        x0, y0, x1, y1 = xs.min(), ys.min(), xs.max(), ys.max()
        bb.append((x0 + 2, y0 + 2, max(x1 - x0 - 3, 1), max(y1 - y0 - 3, 1)))
    return np.array(bb, np.int32).reshape(-1, 4)


@needs_opencv_orders
@pytest.mark.parametrize("name", NAMES)
def test_track_dynamic_klt_bit_exact(name):
    """status rows, output order, ids and both masks; every third listed object has no previous feature (new), the others 25
    young ones (tracked, some resampled)"""
    c = OC.CASES[name]
    (g0, m0, _), (g1, m1, f1) = OC.frames(c)
    rng = np.random.default_rng(3)
    kp, lab = [], []
    for j, oid in enumerate(sorted(set(np.unique(m0).tolist()) - {0})):
        if j % 3 == 2:
            continue
        ys, xs = np.nonzero(m0 == oid)
        s = rng.choice(len(ys), min(25, len(ys)), replace=False)
        kp.append(np.stack([xs[s] + 0.5, ys[s] + 0.5], 1)); lab += [oid]*len(s)
    kp = np.concatenate(kp).astype(np.float32); lab = np.array(lab, np.int32)
    age = rng.integers(0, 6, len(lab)).astype(np.int32); tid = np.arange(len(lab), dtype=np.int64)
    objs = list(c.listed); bb = _objects_bb(m1, objs)
    t = _tracker(f1, m1)
    dev = t.track_dynamic_klt(g0, g1, kp, lab, age, tid, objs, bb, 10**6)
    ref = KO.track_dynamic_klt(g1, m1, None, kp, lab, age, tid, dev["lk_pts"], dev["lk_status"], objs, bb, KO.Params(), 10**6)
    assert np.array_equal(dev["state"], ref["state"]) and np.array_equal(dev["measured_flow"], ref["measured_flow"])
    for k in ("keypoint", "age", "tracklet", "label", "source"):
        assert dev[k].shape == ref[k].shape and np.array_equal(dev[k], ref[k]), k
    assert dev["next_tracklet_id"] == ref["next_tracklet_id"] and dev["n_outside_image"] == ref["n_outside_image"]
    for f in KO.STATUS_FIELDS:
        assert np.array_equal(dev["status"][f], ref["status"][f]), (f, dev["status"][f], ref["status"][f])
    assert np.array_equal(dev["detection_mask"], ref["detection_mask"]) and np.array_equal(dev["tracking_mask"], ref["tracking_mask"])
    assert (dev["state"] == KO.TRACKED).sum() > 0
    if len(objs) == 64:
        assert dev["status"]["sampled"][1:].sum() >= 21 and (dev["source"] < 0).sum() > 0      # every third object is new


@pytest.mark.parametrize("name", NAMES)
def test_depths_and_dense_cloud_bit_exact(name):
    (_, _, _), (_, m, _) = OC.frames(OC.CASES[name])
    rng = np.random.default_rng(4)
    depth = rng.uniform(1.0, 250.0, (H, W))
    for lab in np.unique(m):
        if lab != 0:
            depth[m == lab] = rng.uniform(8.0, 60.0)
    kp, lab = _features(rng, m, np.zeros((H, W, 2), np.float32), per_object=20)
    kp = np.concatenate([kp, rng.uniform(0, [W, H], (300, 2))]); lab = np.concatenate([lab, np.zeros(300, np.int32)])
    t = _tracker(np.zeros((H, W, 2), np.float32), m); t.set_depth(depth)
    d, v, ni, no = t.update_depths(kp, lab)
    rd, rv, rni, rno = DPO.update_depths(kp, lab, depth)
    assert np.array_equal(d, rd, equal_nan=True) and np.array_equal(v, rv) and (ni, no) == (rni, rno)
    r = t.back_project(kp, d, v, CAL, 0.537, True)
    idx, pt, sp, out = DPO.back_project(kp, d, v, CAL, W, 0.537, True)
    assert np.array_equal(r["index"], idx) and np.array_equal(r["point"], pt, equal_nan=True)
    assert np.array_equal(r["stereo"], sp, equal_nan=True) and np.array_equal(r["outlier"], out)
    xyz, rgb, labo, valid, nv = t.dense_cloud(CAL)
    rx, rr, rl, rvv = DPO.dense_cloud(depth, m, None, CAL)
    assert np.array_equal(xyz, rx) and np.array_equal(rgb, rr) and np.array_equal(labo, rl) and np.array_equal(valid, rvv)
    assert nv == int(rvv.sum()) and set(np.unique(rl[rvv == 1]).tolist()) - {0}


UNIQUE_IDS = [1, 255, 256, 257, 1000, 65535, 65536, 2**24 - 1, 2**24, 2**24 + 1, 2**24 + 3, 2**31 - 1, -1, -2, -255, -2**24 - 1, -2**31]


def test_unique_id_rgb_at_large_and_negative_ids():
    """Color::uniqueId((size_t)id) through dense_cloud: one 4 x 4 block per id, depth 10 m everywhere"""
    from dynosam_b200.frontend import FeatureTrackerGPU
    w, h = 4*len(UNIQUE_IDS), 8
    m = np.zeros((h, w), np.int32)
    for j, oid in enumerate(UNIQUE_IDS):
        m[2:6, 4*j:4*j + 4] = oid
    t = FeatureTrackerGPU(w, h); t.set_frame(np.zeros((h, w, 2), np.float32), m, None); t.set_depth(np.full((h, w), 10.0))
    xyz, rgb, labo, valid, nv = t.dense_cloud(CAL)
    rx, rr, rl, rv = DPO.dense_cloud(np.full((h, w), 10.0), m, None, CAL)
    assert np.array_equal(rgb, rr) and np.array_equal(labo, rl) and nv == w*h
    assert np.array_equal(rgb[3, 2::4], DPO.unique_id_rgb(UNIQUE_IDS))


@pytest.mark.parametrize("name", list(OC.VOTES))
def test_propagate_mask_votes_bit_exact(name):
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    v = OC.VOTES[name]
    kp, lab, prev, flow, cur = OC.vote_frame(v)
    h, w = cur.shape
    t = FeatureTrackerGPU(w, h)
    out = t.propagate_mask(kp, lab, prev, flow, cur, TrackParams(), v.min_votes)
    ref = FO.propagate_mask(kp, lab, prev, flow, cur, FO.TrackParams(), v.min_votes)
    assert np.array_equal(out, ref)


def _spread(mode, mode_votes, extra=()):
    """votes of one object: 60 on each of 40 labels outside [0, 256) (-1 .. -20, 256 .. 275), 30 on each of 1 .. 10, mode_votes
    on mode and the extra (label, count) pairs"""
    vs = {l: 60 for l in list(range(-20, 0)) + list(range(256, 276))}
    vs.update({l: 30 for l in range(1, 11)})
    vs[mode] = mode_votes
    vs.update(dict(extra))
    return tuple(sorted(vs.items()))


# (votes, propagated): labels outside [0, 256) are sorted in the vote kernel, in shared memory up to 2048 of them, above that in
# place in the global vote buffer
MANY_VOTES = {
    "global_mode0": (_spread(0, 700), True),                                   # 2400 votes outside [0, 256)
    "global_mode70000": (_spread(70000, 700, ((0, 30),)), False),              # 3100
    "global_tie_0_256_m7": (_spread(0, 700, ((256, 700), (-7, 700))), None),    # 2400 + 700: std::sort decides the tie
    "shared_mode0": (tuple((l, c) for l, c in _spread(0, 700) if not -20 <= l <= -1), True),    # 1200
}


@pytest.mark.parametrize("name", list(MANY_VOTES))
def test_propagate_mask_many_votes_and_labels(name):
    """one object with thousands of votes on 51-53 labels, negative ones and ones >= 256 among them, bit for bit against the
    oracle; the count of votes outside [0, 256) puts the kernel's sort in global memory (> 2048) or in shared memory"""
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    vs, painted = MANY_VOTES[name]
    outside = sum(c for l, c in vs if not 0 <= l < 256)
    assert (outside > 2048) == name.startswith("global")
    v = OC.VoteCase(name, ((500, vs, None),), 150, ())
    kp, lab, prev, flow, cur = OC.vote_frame(v)
    h, w = cur.shape
    out = FeatureTrackerGPU(w, h).propagate_mask(kp, lab, prev, flow, cur, TrackParams(), 150)
    ref = FO.propagate_mask(kp, lab, prev, flow, cur, FO.TrackParams(), 150)
    assert np.array_equal(out, ref) and len(kp) == sum(c for _, c in vs)
    if painted is not None:
        assert ((out == 500).sum() > 0) == painted


def test_propagate_mask_object_without_votes():
    """min_votes = 0 and an object whose key-points all fall outside the image: no vote, nothing propagated"""
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    prev = np.zeros((40, 60), np.int32); prev[5:15, 5:20] = 3
    flow = np.zeros((40, 60, 2), np.float32); flow[..., 0] = 2.5; flow[..., 1] = 1.5
    cur = np.zeros((40, 60), np.int32)
    kp = np.array([[0.5, 10.5], [70.0, 10.0]])
    out = FeatureTrackerGPU(60, 40).propagate_mask(kp, [3, 3], prev, flow, cur, TrackParams(), 0)
    assert np.array_equal(out, FO.propagate_mask(kp, [3, 3], prev, flow, cur, FO.TrackParams(), 0)) and np.array_equal(out, cur)


def test_object_list_refusals():
    """65 objects, a duplicate id and an id <= 0 are refused by every object-list entry point, with a message, before anything
    is launched: the tracker then gives what a fresh one gives"""
    from dynosam_b200.frontend import FrontendError, TrackParams
    c = OC.CASES["n64_contiguous_shuffled"]
    (g0, m0, _), (g1, m1, f1) = OC.frames(c)
    prm = TrackParams()
    kp = np.array([[10.5, 10.5]], np.float32); one = (kp, np.ones(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int64))
    bad = [("at most 64 objects", list(range(1, 66))), ("distinct", [3, 5, 3]), ("must be > 0", [4, 0]), ("must be > 0", [2, -7])]
    t = _tracker(f1, m1)
    for msg, objs in bad:
        with pytest.raises(FrontendError, match=msg):
            t.sample_candidates(objs, prm)
        with pytest.raises(FrontendError, match=msg):
            t.sample_dynamic(objs, 0, prm, 100)
        with pytest.raises(FrontendError, match=msg):
            t.track_dynamic_klt(g0, g1, *one, objs, np.zeros((len(objs), 4), np.int32), 100)
    objs = list(c.listed)
    fresh = _tracker(f1, m1)
    a, b = t.sample_dynamic(objs, 0, prm, 100), fresh.sample_dynamic(objs, 0, prm, 100)
    for key in ("counts", "num_sampled", "keypoint", "tracklet", "label", "next_tracklet_id"):
        assert np.array_equal(a[key], b[key]), key
    assert a["num_sampled"].min() > 0
