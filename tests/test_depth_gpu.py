"""Depth and back-projection on the device: dynofront_set_depth / update_depths / back_project / dense_cloud, bit-exact against
tests/depth_oracle.py (NaN compared by position, signed zero by value) on 1242x375 frames of the C4 synthetic stream."""
import numpy as np
import pytest

import depth_oracle as DO
from dynosam_b200.synth_frames import SyntheticStream, W, H

pytestmark = pytest.mark.gpu

CAL = (718.856, 718.856, 0.0, 607.1928, 185.2157)          # KITTI-like intrinsics at 1242x375
BASELINE = 0.537


def _eq(a, b):
    a = np.asarray(a); b = np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def _pose(seed=9):
    rng = np.random.default_rng(seed)
    a = rng.normal(size=3); th = np.linalg.norm(a); k = a/th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th)*Kx + (1 - np.cos(th))*Kx @ Kx
    return np.concatenate([R.ravel(), rng.normal(size=3)*5])


def _features(st, k, rng, n_static=800, per_object=200):
    """~800 static and ~2000 dynamic key-points of frame k: static ones spread a little beyond the image (out-of-image points),
    the depth edge pixels hit exactly (also through -0.5 / 0.999 offsets, which truncate onto them), dynamic ones on the objects"""
    _, m, _ = st.frame(k)
    kp = [np.stack([rng.uniform(-3, W + 3, n_static), rng.uniform(-3, H + 3, n_static)], 1)]
    lab = [np.zeros(n_static, np.int32)]
    for ys, xs in st.depth_edge_pixels().values():
        for off in (0.0, 0.999):
            kp.append(np.stack([xs + off, ys + off], 1)); lab.append(m[ys, xs])
    kp.append(np.array([[-0.5, -0.5], [W - 0.001, H - 0.001], [-1.0, 3.0], [W, 3.0], [3.0, H], [np.nan, 2.0]]))
    lab.append(np.array([0, 0, 0, 0, 0, 0], np.int32))
    for o in range(1, 11):
        ys, xs = np.nonzero(m == o)
        if len(ys):
            sel = rng.choice(len(ys), size=min(per_object, len(ys)), replace=False)
            kp.append(np.stack([xs[sel] + rng.uniform(0, 1, len(sel)), ys[sel] + rng.uniform(0, 1, len(sel))], 1)); lab.append(np.full(len(sel), o, np.int32))
    return np.concatenate(kp), np.concatenate(lab)


def _frame(st, k):
    """frame k as the C-contiguous (gray, mask, flow) arrays next_frame takes"""
    return tuple(np.ascontiguousarray(a) for a in st.frame(k))


def _tracker(st, k, det=None):
    from dynosam_b200.frontend import FeatureTrackerGPU
    _, m, f = st.frame(k)
    t = FeatureTrackerGPU(W, H); t.set_frame(f, m, det); t.set_depth(st.depth(k))
    return t


@pytest.mark.parametrize("k", [0, 3])
def test_update_depths_bit_exact(k):
    st = SyntheticStream(n_objects=10, seed=42); rng = np.random.default_rng(k)
    kp, lab = _features(st, k, rng)
    assert (lab == 0).sum() >= 800 and (lab != 0).sum() >= 1500
    t = _tracker(st, k)
    d, v, ninv, nout = t.update_depths(kp, lab, 200.0, 30.0)
    rd, rv, rninv, rnout = DO.update_depths(kp, lab, st.depth(k), 200.0, 30.0)
    assert _eq(d, rd) and _eq(v, rv) and (ninv, nout) == (rninv, rnout)
    assert 0 < rnout < ninv < len(kp) and np.isnan(d[v == 1]).any() and (d == 30.0).any() and (d == 200.0).any()


@pytest.mark.parametrize("rgbd,stereo,world", [(False, False, False), (True, False, False), (True, True, False), (True, True, True),
                                               (False, True, True)])
def test_back_project_bit_exact(rgbd, stereo, world):
    st = SyntheticStream(n_objects=10, seed=42); rng = np.random.default_rng(11)
    kp, lab = _features(st, 2, rng)
    t = _tracker(st, 2)
    d, v, _, _ = t.update_depths(kp, lab)
    usable = v.copy(); usable[rng.random(len(v)) < 0.1] = 0             # unusable features, including valid ones
    usable[np.isnan(d) & (v == 1)] = 1                                  # every NaN-depth (valid, no depth) feature is walked
    # uR exactly at 0 and at W (fx b / d = 250 / 2.5 = 100 exactly): kept, strict tests; just beyond W: an outlier
    extra = np.array([[100.0, 10.0], [W + 100.0, 20.0], [W + 100.5, 30.0], [200.0, 40.0]])
    kp = np.concatenate([kp, extra]); d = np.concatenate([d, [2.5, 2.5, 2.5, np.nan]])
    usable = np.concatenate([usable, [1, 1, 1, 1]]).astype(np.uint8)
    cal = (CAL[0], CAL[1], CAL[2], CAL[3], CAL[4]) if not (rgbd and not stereo) else (500.0, 500.0, 0.0, CAL[3], CAL[4])
    b = 0.5 if cal[0] == 500.0 else BASELINE
    right = None
    if stereo:
        right = np.full(len(kp), np.nan); sub = (rng.random(len(kp)) < 0.3) & ~np.isnan(d)
        right[sub] = kp[sub, 0] - rng.uniform(1, 40, sub.sum())
    X = _pose() if world else None
    r = t.back_project(kp, d, usable, cal, b, rgbd, right, X)
    idx, pt, sp, out = DO.back_project(kp, d, usable, cal, W, b, rgbd, right, X)
    assert r["m"] == len(idx) and _eq(r["index"], idx) and _eq(r["point"], pt) and _eq(r["stereo"], sp) and _eq(r["outlier"], out)
    assert np.isnan(pt[:, 2]).any()                                     # key-point-only measurements are emitted
    if rgbd and not stereo:
        n = len(kp)
        assert out[n - 4] == 0 and out[n - 3] == 0 and out[n - 2] == 1 and out.sum() > 1
        row = {i: j for j, i in enumerate(idx)}
        assert sp[row[n - 4], 1] == 0.0 and sp[row[n - 3], 1] == float(W)


def test_back_project_capacity_and_refusal():
    from dynosam_b200.frontend import FrontendError
    st = SyntheticStream(n_objects=10, seed=42); rng = np.random.default_rng(12)
    kp, lab = _features(st, 1, rng)
    t = _tracker(st, 1)
    d, v, _, _ = t.update_depths(kp, lab)
    full = t.back_project(kp, d, v, CAL, BASELINE, True)
    part = t.back_project(kp, d, v, CAL, BASELINE, True, capacity=37)
    assert part["m"] == full["m"] > 37 and len(part["index"]) == 37
    assert _eq(part["index"], full["index"][:37]) and _eq(part["point"], full["point"][:37]) and _eq(part["stereo"], full["stereo"][:37])
    right = np.full(len(kp), np.nan); j = np.flatnonzero(np.isnan(d) & (v == 1))[0]; right[j] = 5.0
    with pytest.raises(FrontendError, match="right key-point but no depth"):
        t.back_project(kp, d, v, CAL, BASELINE, True, right)


@pytest.mark.parametrize("with_det", [False, True])
def test_dense_cloud_after_propagate_mask(with_det):
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    st = SyntheticStream(n_objects=10, seed=42); rng = np.random.default_rng(13)
    g0, m0, f0 = _frame(st, 4); g1, m1, f1 = _frame(st, 5)
    det = None
    if with_det:
        det = np.full((H, W), 255, np.uint8); det[:, :40] = 0; det[200:230, :] = 0
    t = FeatureTrackerGPU(W, H)
    t.next_frame(g0, f0, m0); t.next_frame(g1, f1, m1, det)
    kp, lab = _features(st, 4, rng); obj = lab != 0
    kp = kp[obj] + f0[kp[obj, 1].astype(int), kp[obj, 0].astype(int)]; lab = lab[obj]
    t.propagate_mask_resident(kp, lab, TrackParams(), min_votes=30)
    mask = t.motion_mask()
    depth = st.depth(5); t.set_depth(depth)
    xyz, rgb, labo, valid, nv = t.dense_cloud(CAL, 200.0, 30.0)
    rx, rr, rl, rv = DO.dense_cloud(depth, mask, det, CAL, 200.0, 30.0)
    assert _eq(xyz, rx) and _eq(rgb, rr) and _eq(labo, rl) and _eq(valid, rv) and nv == int(rv.sum())
    assert 0 < nv < W*H and (rl[rv == 1] != 0).any() and (rr.reshape(-1, 3)[rl.ravel() != 0] != 0).all()


def test_streaming_equals_call_by_call_and_refusals():
    from dynosam_b200.frontend import FeatureTrackerGPU, FrontendError
    st = SyntheticStream(n_objects=10, seed=42); rng = np.random.default_rng(14)
    t = FeatureTrackerGPU(W, H)
    with pytest.raises(FrontendError, match="no frame"):
        t.set_depth(st.depth(0))
    frames = [_frame(st, k) for k in range(3)]; depths = [np.ascontiguousarray(st.depth(k)) for k in range(3)]
    for d in depths:
        t.pin(d)
    for k in range(3):
        g, m, f = frames[k]
        t.next_frame(g, f, m)
        with pytest.raises(FrontendError, match="no depth for the current frame"):
            t.update_depths(np.zeros((1, 2)), [0])
        with pytest.raises(FrontendError, match="no depth for the current frame"):
            t.dense_cloud(CAL)
        t.set_depth(depths[k])
        kp, lab = _features(st, k, rng)
        s = (t.update_depths(kp, lab), t.dense_cloud(CAL))
        c = _tracker(st, k)
        r = (c.update_depths(kp, lab), c.dense_cloud(CAL))
        for a, b in zip(s[0] + s[1], r[0] + r[1]):
            assert _eq(a, b)
        c.close()
    for bad in [(0.0, 30.0), (200.0, -1.0), (np.nan, 30.0)]:
        with pytest.raises(FrontendError, match="thresholds must be > 0"):
            t.update_depths(np.zeros((1, 2)), [0], *bad)
        with pytest.raises(FrontendError, match="thresholds must be > 0"):
            t.dense_cloud(CAL, *bad)
    for d in depths:
        t.unpin(d)


def test_existing_outputs_unchanged_by_depth_calls():
    """the streaming frame loop gives byte-equal results with and without set_depth / update_depths / dense_cloud in it"""
    from dynosam_b200.frontend import DetectParams, FeatureTrackerGPU, TrackParams
    st = SyntheticStream(n_objects=10, seed=42); prm = TrackParams(); dprm = DetectParams()
    frames = [_frame(st, k) for k in range(5)]
    static_pts = np.stack([np.linspace(30, W - 30, 300), np.linspace(20, H - 20, 300)], 1).astype(np.float32)

    def run(with_depth):
        rng = np.random.default_rng(15)
        t = FeatureTrackerGPU(W, H); outs = []
        t.next_frame(*[frames[0][i] for i in (0, 2, 1)])
        for k in range(1, 5):
            g, m, f = frames[k]
            t.next_frame(g, f, m)
            kp, lab = _features(st, k - 1, rng, n_static=0)
            kp, lab = kp[lab != 0], lab[lab != 0]
            if with_depth:
                t.set_depth(st.depth(k)); t.update_depths(kp, lab); t.dense_cloud(CAL)
            t.propagate_mask_resident(kp, lab, prm)
            outs.append(t.motion_mask())
            outs.extend(t.track_dynamic(kp, lab, np.zeros(len(lab), np.int32), np.arange(len(lab)), prm, 10**6)[:7])
            r = t.sample_dynamic(list(range(1, 11)), 0, prm, 10**6)
            outs.extend(r[key] for key in ("keypoint", "tracklet", "num_sampled"))
            outs.extend(t.klt_track_fb(None, None, static_pts, prm, np.zeros(300, np.int32), 25))
            outs.extend(t.detect_static(None, static_pts, dprm, 0)[:2])
        t.close()
        return outs
    a, b = run(False), run(True)
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()


def _tracked_features(st, k, n_static=400, per_object=60):
    """features that keep their tracklet ids over the frames: a fixed static grid (ids 0..), and per object the same slots of
    its pixels in raster order (ids 100000 + 1000 object + slot)"""
    _, m, _ = st.frame(k)
    gx, gy = np.meshgrid(np.linspace(3.3, W - 4.1, 25), np.linspace(2.7, H - 3.2, n_static//25))
    kp = [np.stack([gx.ravel(), gy.ravel()], 1)]; lab = [np.zeros(gx.size, np.int32)]; tid = [np.arange(gx.size, dtype=np.int64)]
    for o in range(1, 11):
        ys, xs = np.nonzero(m == o)
        if len(ys) < per_object:
            continue
        sel = np.linspace(0, len(ys) - 1, per_object).astype(int)
        kp.append(np.stack([xs[sel] + 0.25, ys[sel] + 0.75], 1)); lab.append(np.full(per_object, o, np.int32))
        tid.append(100000 + 1000*o + np.arange(per_object, dtype=np.int64))
    return np.concatenate(kp), np.concatenate(lab), np.concatenate(tid)


def test_hand_off_to_the_graph_builder():
    """5 frames: update_depths -> back_project -> builder, against the builder fed with the oracle's measurements"""
    from dynosam_b200.builder import GraphBuilder
    from dynosam_b200.frontend import FeatureTrackerGPU, builder_measurements
    st = SyntheticStream(n_objects=10, seed=42)
    t = FeatureTrackerGPU(W, H); gb, ob = GraphBuilder(), GraphBuilder()
    I = np.concatenate([np.eye(3).ravel(), np.zeros(3)])
    for k in range(5):
        g, m, f = _frame(st, k); depth = st.depth(k)
        t.next_frame(g, f, m); t.set_depth(depth)
        kp, lab, tid = _tracked_features(st, k)
        d, v, _, _ = t.update_depths(kp, lab)
        bp = t.back_project(kp, d, v, CAL, BASELINE, True)
        rd, rv, _, _ = DO.update_depths(kp, lab, depth)
        ri, rp, _, _ = DO.back_project(kp, rd, rv, CAL, W, BASELINE, True)
        for b, res in ((gb, bp), (ob, dict(index=ri, point=rp))):
            (ts, zs), (td, od, zd) = builder_measurements(res, tid, lab)
            b.add_frame(k, I, None if k == 0 else I)
            b.add_static(k, ts, zs); b.add_dynamic(k, td, od, zd)
    p, q = gb.problem(), ob.problem()
    assert len(p.blocks) == len(q.blocks) > 0 and p.point.shape == q.point.shape and p.point.shape[0] > 0
    assert _eq(p.pose, q.pose) and _eq(p.point, q.point) and _eq(p.aux_pose, q.aux_pose)
    for x, y in zip(p.blocks, q.blocks):
        assert x.type == y.type and _eq(x.idx, y.idx) and _eq(x.sigma, y.sigma)
        assert (x.meas is None) == (y.meas is None) and (x.meas is None or _eq(x.meas, y.meas))
        assert (x.aux_idx is None) == (y.aux_idx is None) and (x.aux_idx is None or _eq(x.aux_idx, y.aux_idx))
