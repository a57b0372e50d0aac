"""STEREO_PROJECTION static landmarks in the graph builder (dynoba_builder_set_static_stereo / add_static_stereo), on the
host build of the triangulation: the landmarks, their factor frames, initial points, sigma and Huber k against the
independent statement of the rules in tests/triangulation_reference.py (with its 50-digit triangulation), the disparity
test at 0.5 px and measurements without a right key-point, composition with dynamic landmarks and the IMU chain, the
refusals, and a builder that never selects stereo emitting bit for bit what it did before."""
import hashlib

import numpy as np
import pytest

import triangulation_reference as TR
from dynosam_b200 import lie, synth, synth_stereo
from dynosam_b200.binding import DynobaError, ERR_BAD_ARG
from dynosam_b200.builder import GraphBuilder
from dynosam_b200.problem import BETWEEN6, HYBRID3, PRIOR6, SMOOTH_HYBRID6, STEREO3, static_landmark_key
from test_builder import _feed, _feed_world_centric

K6 = synth.KITTI_K


def mp_tri(poses, kp, K5):
    r = TR.triangulate(poses, kp, K5)
    return r["status"], r["point"]


def feed(b, p, st, device=-1, sigma_px=1.0):
    """frames (and odometry) of problem p, then the stereo static observations st"""
    N = p.meta["n_frames"]
    odo = [x for x in p.blocks if x.type == BETWEEN6]
    rel = {int(i[1]): m for i, m in zip(odo[-1].idx, odo[-1].meas)} if odo else {}
    b.set_static_stereo(K6, sigma_px, device)
    for k in range(N):
        b.add_frame(k, p.pose[k], rel.get(k))
        sel = np.flatnonzero(st["frame"] == k)
        b.add_static_stereo(k, st["tracklet"][sel], st["stereo"][sel])


def stereo_block(q):
    blk = [x for x in q.blocks if x.type == STEREO3]
    assert len(blk) == 1 and q.blocks[0] is blk[0]
    return blk[0]


def check_against_rules(q, b, p, st, sigma_px=1.0):
    N = p.meta["n_frames"]
    obs = [(int(f), int(t), z) for f, t, z in zip(st["frame"], st["tracklet"], st["stereo"])]
    ref = TR.stereo_graph({k: p.pose[k] for k in range(N)}, obs, K6, mp_tri)
    land = ref["landmarks"]
    assert np.array_equal(q.point_keys[:len(land)], static_landmark_key(np.array(land)))
    blk = stereo_block(q)
    assert blk.sigma.tolist() == [sigma_px]*3 and blk.robust_k == 1e-4 and np.array_equal(q.calib, K6)
    got = {}
    for (cam, pi), z in zip(blk.idx, blk.meas):
        got.setdefault(land[pi], []).append((int(q.pose_order[cam]), z))
    for i, t in enumerate(land):
        assert [f for f, _ in got[t]] == ref["factors"][t], t
        zs = {int(f): z for f, tt, z in obs if tt == t}
        assert all(np.array_equal(z, zs[f], equal_nan=True) for f, z in got[t])
        r = TR.triangulate(*ref["cameras"][t], K6[:5])
        assert np.linalg.norm(q.point[i] - ref["points"][t]) <= TR.point_bound(r), t
    s = b.static_stereo_stats()
    assert s["added"] == len(land) and s["never_added"] == len(ref["never"])
    assert s["failed"] == [ref["failed"][k] for k in range(4)]
    return ref


@pytest.mark.parametrize("cfg", [dict(n_frames=20, n_static=120, seed=3, far_fraction=0.2, nan_right=0.1, outlier_fraction=0.03),
                                 dict(n_frames=12, n_static=80, seed=8, pixel_sigma=1.5, nan_right=0.3)])
def test_builder_stereo_matches_the_rules(cfg):
    p, st = synth_stereo.make_scene(**cfg)
    b = GraphBuilder(); feed(b, p, st)
    q = b.problem()
    assert [x.type for x in q.blocks] == [STEREO3, PRIOR6, BETWEEN6]
    ref = check_against_rules(q, b, p, st)
    assert len(ref["landmarks"]) > 0.25*cfg["n_static"] and len(ref["never"]) > 0
    b.close()


def test_disparity_and_missing_right_keypoint():
    """attempts fail until two observations with uL - uR > 0.5 exist; after that every observation with a right key-point
    adds a factor, whatever its disparity, and one without adds none"""
    N = 6
    X = [lie.pack(np.eye(3)[None], np.array([[0.0, 0.0, 0.1*k]]))[0] for k in range(N)]
    pw = np.array([2.0, 1.0, 775.0])
    disp = [0.5, 0.5 + 1e-6, np.nan, 0.6, np.nan, 0.1]
    b = GraphBuilder(); b.set_static_stereo(K6, 1.0, -1)
    for k in range(N):
        b.add_frame(k, X[k], None if k == 0 else lie.identity()[0])
        q = lie.transform_to(X[k][None], pw[None])[0]
        uL, v = K6[3] + K6[0]*q[0]/q[2], K6[4] + K6[1]*q[1]/q[2]
        b.add_static_stereo(k, [7], [[uL, uL - disp[k], v]])
    q = b.problem()
    blk = stereo_block(q)
    assert q.n_point == 1 and blk.idx[:, 0].tolist() == [1, 3, 5]
    s = b.static_stereo_stats()
    assert s == dict(added=1, failed=[3, 0, 0, 0], never_added=0)               # frames 0, 1, 2: a valid point, < 2 factors
    b.close()


def test_composes_with_dynamic_landmarks_and_imu():
    p, st = synth_stereo.make_scene(n_frames=15, n_static=60, seed=4, n_objects=1, n_dynamic=40)
    b = GraphBuilder(); feed(b, p, st)
    ref_b = GraphBuilder()
    h = [x for x in p.blocks if x.type == HYBRID3][0]
    for bb in (b, ref_b):
        for k in range(p.meta["n_frames"]):
            if bb is ref_b:
                bb.add_frame(k, p.pose[k], None if k == 0 else lie.between(p.pose[k - 1][None], p.pose[k][None])[0])
            sel = np.flatnonzero(h.idx[:, 0] == k)
            bb.add_dynamic(k, h.idx[sel, 2], h.aux_idx[sel] + 1, h.meas[sel])
    q, r = b.problem(), ref_b.problem()
    assert [x.type for x in q.blocks] == [STEREO3, HYBRID3, PRIOR6, SMOOTH_HYBRID6, PRIOR6, BETWEEN6]
    ns = stereo_block(q).idx[:, 1].max() + 1
    assert np.array_equal(q.point[ns:], r.point) and np.array_equal(q.pose, r.pose)
    for x, y in zip(q.blocks[1:4], r.blocks[0:3]):
        assert np.array_equal(x.idx - (ns if x.type == HYBRID3 else 0)*np.array([0, 0, 1])[:x.idx.shape[1]], y.idx)
    b.close(); ref_b.close()
    # the IMU chain: initial camera poses predicted, the attempts still use the add_frame poses
    from dynosam_b200 import synth_imu  # noqa: F401
    pi, sti = synth_stereo.make_scene(n_frames=10, n_static=40, seed=6, imu=True)
    b = GraphBuilder()
    b.set_static_stereo(K6, 1.0, -1)
    for k in range(10):
        b.add_frame(k, pi.pose[k], None)
        sel = np.flatnonzero(sti["frame"] == k)
        b.add_static_stereo(k, sti["tracklet"][sel], sti["stereo"][sel])
    imu = [x for x in pi.blocks if x.type == 13][0]
    for k in range(10):
        if k == 0:
            b.set_imu(0, imu.meas[0], imu.sigma[0])
        else:
            b.set_imu(k, imu.meas[k - 1], imu.sigma[k - 1])
    q = b.problem()
    assert [x.type for x in q.blocks][:1] == [STEREO3] and q.vel.shape[0] == 10
    check_against_rules(q, b, pi, sti)
    b.close()


def test_refusals():
    I = lie.identity()[0]
    b = GraphBuilder(); b.add_static(0, [1], [[0, 0, 4.0]])
    with pytest.raises(DynobaError):
        b.set_static_stereo(K6, 1.0, -1)                                   # after point-to-point observations
    b = GraphBuilder()
    with pytest.raises(DynobaError):
        b.add_static_stereo(0, [1], [[600.0, 590.0, 170.0]])              # before set_static_stereo
    for K, s in ((np.r_[0.0, K6[1:]], 1.0), (np.r_[K6[:5], 0.0], 1.0), (np.r_[np.nan, K6[1:]], 1.0), (K6, 0.0), (K6, np.inf)):
        with pytest.raises(DynobaError) as e:
            b.set_static_stereo(K, s, -1)
        assert e.value.status == ERR_BAD_ARG
    b.set_static_stereo(K6, 1.0, -1)
    with pytest.raises(DynobaError):
        b.add_static(0, [1], [[0, 0, 4.0]])                                # mixing the formulations
    for z in ([np.nan, 590.0, 170.0], [600.0, np.inf, 170.0], [600.0, 590.0, np.nan]):
        with pytest.raises(DynobaError):
            b.add_static_stereo(0, [1], [z])
    b.add_frame(0, I); b.add_frame(1, I, I)
    b.add_static_stereo(0, [1], [[600.0, 590.0, 170.0]]); b.add_static_stereo(0, [1], [[601.0, 591.0, 170.0]])
    with pytest.raises(DynobaError):
        b.problem()                                                        # a tracklet observed twice in one frame
    b = GraphBuilder(); b.set_static_stereo(K6, 1.0, -1); b.add_frame(0, I)
    b.add_static_stereo(3, [1], [[600.0, 590.0, 170.0]])
    with pytest.raises(DynobaError):
        b.problem()                                                        # an unknown frame


def _digest(q):
    h = hashlib.sha256()
    for a in (q.pose, q.point, q.aux_pose, q.pose_order, q.pose_keys, q.point_keys, q.vel, q.bias):
        h.update(np.ascontiguousarray(a).tobytes())
    for x in q.blocks:
        h.update(np.int64([x.type, x.n]).tobytes()); h.update(x.idx.tobytes()); h.update(np.float64([x.robust_k]).tobytes())
        for a in (x.meas, x.sigma, x.aux_idx):
            if a is not None:
                h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def test_without_stereo_the_builder_is_unchanged():
    """digests of the builder's output before the stereo formulation existed"""
    p = synth.make_problem(n_frames=30, n_objects=2, n_static=400, n_dynamic=200, seed=11, object_span=(10, 20), formulation="hybrid")
    b = GraphBuilder(); _feed(p, b)
    assert _digest(b.problem()) == "1a49d4ce2f195de42974cf0f48aaf5d239524cf644cf3e14680620beb468bef4"
    p = synth.make_problem(n_frames=30, n_objects=2, n_static=300, n_dynamic=300, seed=12, object_span=(10, 20), formulation="wcpe")
    b = GraphBuilder(formulation="wcpe", backtrack=0); _feed_world_centric(p, b)
    assert _digest(b.problem()) == "db077f806780cfffc4e6171e6117fc8ccd2978b497c0c126fe489d119f945b27"
