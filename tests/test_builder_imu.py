"""The graph builder's visual-inertial rules (dynoba_builder_set_imu; RegularBackendModule.cc:528-570,
VisionImuBackendModule.hpp:114-290), block by block against the independent numpy statement synth_imu.imu_graph, under the
three formulations and both backtrack settings, on a seeded stream:
  * camera poses, velocities and biases: the predict chain from the first frame (frame 0 keeps the front end's pose);
  * the IMU / prior blocks, and no odometry BetweenFactor;
  * every other block and every point and pose-like variable equal those of a builder without IMU fed the predicted
    poses as its frame poses -- points are initialised from the predicted pose;
  * nav order hints (frame ids) and V / b keys;
  * every refusal.
Initial values are held to 1e-12 of their scale: the builder and the numpy statement evaluate the same fp64 predict in a
different operation order, over at most 8 frames."""
import numpy as np
import pytest

from dynosam_b200 import lie, synth_imu
from dynosam_b200.binding import DynobaError
from dynosam_b200.problem import BETWEEN6, COMBINED_IMU15, PRIOR_BIAS6, PRIOR_VEL3, symbol_key

N = 8
XI = np.array([0.02, -0.03, 0.05, 0.3, 0.05, 0.8])


def _stream(seed=3):
    """front-end poses (the truth perturbed), IMU records and R per frame, observations"""
    rng = np.random.default_rng(seed)
    X_gt = np.concatenate([lie.se3_exp((k*XI)[None]) for k in range(N)])
    X_fe = np.concatenate([lie.compose(X_gt[k:k + 1], lie.se3_exp(rng.normal(0, 0.02, (1, 6)))) for k in range(N)])
    X_fe[0] = X_gt[0]
    st, ag = synth_imu.imu_stream(X_gt, XI, samples_per_frame=10, bias_true=np.array([0.02, -0.01, 0.03, 1e-3, -2e-3, 5e-4]), seed=seed)
    recs = [synth_imu.preintegrate(a[:-1, :3], a[:-1, 3:], float(s[1] - s[0])) for s, a in zip(st, ag)]
    Rs = [synth_imu.sqrt_info(rng)[1] for _ in recs]
    return X_fe, recs, Rs


def _feed(b, X, recs=None, Rs=None):
    I = lie.identity()[0]
    for k in range(N):
        b.add_frame(k, X[k], None if k == 0 else I)
        if recs is not None and k > 0:
            b.set_imu(k, recs[k - 1], Rs[k - 1])
    for k in range(2, 6):
        b.add_static(k, [7], [[0.1*k, 0.0, 4.0]])
    for k in range(4, 8):
        b.add_static(k, [8], [[1.0, 0.2*k, 6.0]])
    b.add_static(1, [9, 10], [[0.0, 0.0, 3.0], [0.5, -0.2, 5.0]]); b.add_static(2, [9, 10], [[0.1, 0.0, 3.0], [0.5, -0.1, 5.0]])
    for k in range(6):
        b.add_dynamic(k, [1, 2], [1, 1], [[1.0 + 0.1*k, 0.0, 5.0], [3.0 + 0.1*k, 0.0, 5.0]])
    for k in range(3, 8):
        b.add_dynamic(k, [3], [2], [[2.0, 1.0 + 0.05*k, 6.0]])


def _close(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.abs(a - b).max(initial=0.0) <= 1e-12*max(1.0, np.abs(b).max(initial=0.0))


@pytest.mark.parametrize("backtrack", [1, 0])
@pytest.mark.parametrize("formulation", ["hybrid", "wcme", "wcpe"])
def test_imu_rules_against_the_numpy_statement(formulation, backtrack):
    from dynosam_b200.builder import GraphBuilder
    X_fe, recs, Rs = _stream()
    X_pred, V, B, blocks = synth_imu.imu_graph(X_fe, recs, Rs)
    assert not _close(X_pred[1:], X_fe[1:])                          # the prediction differs from the front end's poses
    b = GraphBuilder(formulation=formulation, backtrack=backtrack); _feed(b, X_fe, recs, Rs); q = b.problem()
    vk, bk = b.nav_keys
    c = GraphBuilder(formulation=formulation, backtrack=backtrack); _feed(c, X_pred); r = c.problem()
    # camera poses, velocities, biases: the predict chain
    assert _close(q.pose[:N], X_pred) and np.array_equal(q.pose[0], X_fe[0])
    assert _close(q.vel, V) and np.array_equal(q.bias, B)
    assert q.vel_order.tolist() == list(range(N)) and q.bias_order.tolist() == list(range(N))
    assert vk.tolist() == [int(symbol_key('V', k)) for k in range(N)] and bk.tolist() == [int(symbol_key('b', k)) for k in range(N)]
    # IMU and prior blocks exactly as stated, no odometry
    nav = [x for x in q.blocks if x.type in (PRIOR_VEL3, PRIOR_BIAS6, COMBINED_IMU15)]
    assert [x.type for x in nav] == [x.type for x in blocks]
    for x, y in zip(nav, blocks):
        assert np.array_equal(x.idx, y.idx) and np.array_equal(x.meas, y.meas), x.type
        assert np.array_equal(np.ravel(x.sigma), np.ravel(y.sigma)), x.type
    odo = [x for x in q.blocks if x.type == BETWEEN6 and x.idx.max() < N]
    assert not odo                                                     # WCME's BETWEEN6 smoothing links motions only
    # everything else: the builder without IMU fed the predicted poses (points from the predicted X_k)
    rest = [x for x in q.blocks if x.type not in (PRIOR_VEL3, PRIOR_BIAS6, COMBINED_IMU15)]
    rest_r = [x for x in r.blocks if not (x.type == BETWEEN6 and x.idx.max() < N)]
    assert [x.type for x in rest] == [x.type for x in rest_r]
    for x, y in zip(rest, rest_r):
        assert np.array_equal(x.idx, y.idx), x.type
        assert (x.meas is None and y.meas is None) or _close(x.meas, y.meas), x.type
    assert _close(q.point, r.point) and _close(q.pose, r.pose) and _close(q.aux_pose, r.aux_pose)
    assert np.array_equal(q.pose_order, r.pose_order) and np.array_equal(q.pose_keys, r.pose_keys)
    assert r.n_vel == 0 and r.n_bias == 0
    b.close(); c.close()


def test_imu_on_the_first_frame_only_marks_presence():
    from dynosam_b200.builder import GraphBuilder
    X_fe, recs, Rs = _stream()
    b = GraphBuilder(); _feed(b, X_fe, recs, Rs); q = b.problem()
    c = GraphBuilder(); _feed(c, X_fe, recs, Rs); c.set_imu(0, recs[0], Rs[0]); r = c.problem()
    assert np.array_equal(q.pose, r.pose) and np.array_equal(q.vel, r.vel)
    assert [x.n for x in q.blocks] == [x.n for x in r.blocks]


def test_refusals():
    from dynosam_b200.builder import GraphBuilder
    X_fe, recs, Rs = _stream()

    def refused(fn):
        with pytest.raises(DynobaError) as e:
            fn()
        assert e.value.status == -1
    b = GraphBuilder()
    z = recs[0].copy(); z[15] = 0.0
    refused(lambda: b.set_imu(1, z, Rs[0]))                            # deltaTij <= 0
    R = Rs[0].copy(); R[3, 3] = -1.0
    refused(lambda: b.set_imu(1, recs[0], R))                         # non-positive diagonal
    R = Rs[0].copy(); R[0, 5] = np.nan
    refused(lambda: b.set_imu(1, recs[0], R))                         # not finite
    b.close()
    # IMU on some frames but not on others
    b = GraphBuilder(); _feed(b, X_fe)
    for k in (1, 2, 4, 5, 6, 7):
        b.set_imu(k, recs[k - 1], Rs[k - 1])
    refused(b.problem); b.close()
    # frame ids not consecutive while IMU is present
    b = GraphBuilder()
    b.add_frame(0, X_fe[0], None); b.add_frame(2, X_fe[2], lie.identity()[0]); b.set_imu(2, recs[0], Rs[0])
    refused(b.problem); b.close()
    # a measurement on a frame that was not added
    b = GraphBuilder(); b.add_frame(0, X_fe[0], None); b.add_frame(1, X_fe[1], lie.identity()[0])
    b.set_imu(1, recs[0], Rs[0]); b.set_imu(5, recs[1], Rs[1])
    refused(b.problem); b.close()
