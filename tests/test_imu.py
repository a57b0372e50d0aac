"""Visual-inertial graphs on the host: the numpy preintegration (dynosam_b200/synth_imu.py) against exact kinematics and
re-preintegration, the independent residual (imu_reference.py) against its own derivatives, and the problem tables."""
import numpy as np
import pytest

import imu_reference as IR
from dynosam_b200 import lie, synth, synth_imu as SI
from dynosam_b200.problem import ARITY, COMBINED_IMU15, DIM, JCOLS, MEAS_DIM, PRIOR_BIAS6, PRIOR_VEL3

XI = np.array([0.03, 0.02, -0.05, 0.4, -0.1, 1.0])      # per-frame twist with a large rotation rate


def _exact_delta(R0, T, g=SI.GRAVITY):
    """ground-truth (dR, dp, dv) over [0, T] of the constant-twist motion starting at rotation R0, gravity included"""
    X0 = np.concatenate([R0.reshape(9), np.zeros(3)])
    X1 = lie.compose(X0[None], lie.se3_exp((T/SI.FRAME_DT)*XI[None]))[0]
    w, v = SI.body_rates(XI)
    R1, p1 = X1[:9].reshape(3, 3), X1[9:]
    v0, v1 = R0@v, R1@v
    dR = R0.T@R1
    dp = R0.T@(p1 - v0*T - 0.5*g*T*T)
    dv = R0.T@(v1 - v0 - g*T)
    return dR, dp, dv


@pytest.mark.parametrize("seed", [0, 1])
def test_preintegration_matches_exact_kinematics(seed):
    R0 = IR.exp3(np.random.default_rng(seed).normal(0, 1.0, 3))
    errs = []
    for n in (20, 40, 80):
        acc, gyro = SI.imu_samples(R0, XI, n, SI.FRAME_DT/n)
        rec = IR.unpack(SI.preintegrate(acc, gyro, SI.FRAME_DT/n))
        dR, dp, dv = _exact_delta(R0, SI.FRAME_DT)
        assert rec["dt"] == pytest.approx(SI.FRAME_DT, abs=1e-15)
        assert np.abs(rec["dR"] - dR).max() < 1e-13          # constant angular rate: the rotation is exact
        errs.append(max(np.abs(rec["dp"] - dp).max(), np.abs(rec["dv"] - dv).max()))
    # the acceleration is integrated with one sample per step: first order, the error halves with the step
    assert 1.8 < errs[0]/errs[1] < 2.2 and 1.8 < errs[1]/errs[2] < 2.2
    assert errs[2] < 1e-3


def test_bias_correction_second_order():
    rng = np.random.default_rng(3)
    R0 = IR.exp3(rng.normal(0, 1.0, 3))
    n, dt = 50, SI.FRAME_DT/50
    acc, gyro = SI.imu_samples(R0, XI, n, dt, bias=np.array([0.2, -0.1, 0.05, 0.01, -0.02, 0.015]))
    hat = np.array([0.1, 0.0, 0.1, 0.0, -0.01, 0.01])
    rec = SI.preintegrate(acc, gyro, dt, hat)
    P = IR.unpack(rec)
    d0 = rng.normal(0, 1, 6)*np.array([0.05, 0.05, 0.05, 0.02, 0.02, 0.02])
    errs = []
    for s in (1.0, 0.25):
        db = s*d0
        Q = IR.unpack(SI.preintegrate(acc, gyro, dt, hat + db))
        dRc = P["dR"]@IR.exp3(P["JRw"]@db[3:])
        dpc = P["dp"] + P["JPa"]@db[:3] + P["JPw"]@db[3:]
        dvc = P["dv"] + P["JVa"]@db[:3] + P["JVw"]@db[3:]
        errs.append(max(np.linalg.norm(IR.log3(dRc.T@Q["dR"])), np.abs(dpc - Q["dp"]).max(), np.abs(dvc - Q["dv"]).max()))
    assert 12.0 < errs[0]/errs[1] < 20.0


def test_residual_zero_on_exact_data():
    """noise-free samples, zero bias, many samples: the residual at the true states is the integration error only"""
    N = 4
    X = lie.se3_exp(np.arange(N)[:, None]*XI[None])
    w, v = SI.body_rates(XI)
    n = 4000
    for k in range(N - 1):
        acc, gyro = SI.imu_samples(X[k, :9].reshape(3, 3), XI, n, SI.FRAME_DT/n)
        rec = SI.preintegrate(acc, gyro, SI.FRAME_DT/n)
        vi, vj = X[k, :9].reshape(3, 3)@v, X[k + 1, :9].reshape(3, 3)@v
        r = IR.imu_residual(X[k], vi, X[k + 1], vj, np.zeros(6), np.zeros(6), rec)
        assert np.abs(r).max() < 1e-3


def test_reference_bias_rows_and_velocity_sign():
    """r[9:15] = b_i - b_j (Between(b_j, b_i)); the velocity rows move with +v_j"""
    rng = np.random.default_rng(5)
    rec = SI.preintegrate(*SI.imu_samples(np.eye(3), XI, 10, 0.01), 0.01)
    Xi = lie.se3_exp(rng.normal(0, 1, (1, 6)))[0]; Xj = lie.se3_exp(rng.normal(0, 1, (1, 6)))[0]
    vi, vj, bi, bj = rng.normal(0, 1, 3), rng.normal(0, 1, 3), rng.normal(0, 0.1, 6), rng.normal(0, 0.1, 6)
    r = IR.imu_residual(Xi, vi, Xj, vj, bi, bj, rec)
    assert np.allclose(r[9:], bi - bj)
    J = IR.imu_numeric_jacobian([Xi, vi, Xj, vj, bi, bj], rec)
    assert np.allclose(J[9:, 18:24], np.eye(6), atol=1e-8) and np.allclose(J[9:, 24:30], -np.eye(6), atol=1e-8)
    # d r_v / d v_j = R_p^T is a rotation
    Dv = J[6:9, 15:18]
    assert np.allclose(Dv@Dv.T, np.eye(3), atol=1e-7) and np.linalg.det(Dv) > 0


def test_problem_tables():
    assert ARITY[COMBINED_IMU15] == 6 and DIM[COMBINED_IMU15] == 15 and JCOLS[COMBINED_IMU15] == 30 and MEAS_DIM[COMBINED_IMU15] == 70
    assert (ARITY[PRIOR_VEL3], DIM[PRIOR_VEL3], JCOLS[PRIOR_VEL3]) == (1, 3, 3)
    assert (ARITY[PRIOR_BIAS6], DIM[PRIOR_BIAS6], JCOLS[PRIOR_BIAS6]) == (1, 6, 6)


def test_make_problem_imu_chain():
    base = synth.make_problem(n_frames=8, n_static=60, n_dynamic=20, seed=4)
    p = synth.make_problem(n_frames=8, n_static=60, n_dynamic=20, seed=4, imu=True)
    assert p.n_vel == 8 and p.n_bias == 8
    types = [b.type for b in p.blocks]
    assert types.count(COMBINED_IMU15) == 1 and PRIOR_VEL3 in types and PRIOR_BIAS6 in types
    imu = p.blocks[types.index(COMBINED_IMU15)]
    assert np.array_equal(imu.idx, np.stack([np.arange(7), np.arange(7), np.arange(1, 8), np.arange(1, 8), np.arange(7), np.arange(1, 8)], 1))
    # the IMU chain replaces the odometry; every other block and every variable is the graph without IMU
    assert np.array_equal(p.pose, base.pose) and np.array_equal(p.point, base.point)
    nb = [b for b in base.blocks if b.type != 1]
    for a, b in zip([b for b in p.blocks if b.type < PRIOR_VEL3], nb):
        assert a.type == b.type and np.array_equal(a.idx, b.idx)
    # the square-root information is upper triangular and positive on the diagonal
    R = imu.sigma.reshape(-1, 15, 15)
    assert np.allclose(np.tril(R, -1), 0) and (np.diagonal(R, axis1=1, axis2=2) > 0).all()


def test_reference_closed_form_jacobian_matches_central_differences():
    """imu_reference.imu_jacobian (the 1e-9 bar of the device's Jacobians) against central differences: random states with
    large rotations, non-zero velocities and bias != biasHat; every one of the six blocks"""
    rng = np.random.default_rng(1)
    for _ in range(30):
        acc, gyro = SI.imu_samples(IR.exp3(rng.normal(0, 1, 3)), XI, 10, 0.01, bias=rng.normal(0, 0.05, 6))
        rec = SI.preintegrate(acc, gyro, 0.01, rng.normal(0, 0.05, 6))
        a = [lie.se3_exp(rng.normal(0, 1, (1, 6)))[0], rng.normal(0, 1, 3), lie.se3_exp(rng.normal(0, 1, (1, 6)))[0],
             rng.normal(0, 1, 3), rng.normal(0, 0.1, 6), rng.normal(0, 0.1, 6)]
        Ja, Jn = IR.imu_jacobian(*a, rec), IR.imu_numeric_jacobian(a, rec)
        for c0, d in zip((0, 6, 9, 15, 18, 24), (6, 3, 6, 3, 6, 6)):
            assert np.abs(Ja[:, c0:c0 + d] - Jn[:, c0:c0 + d]).max() <= 1e-6*np.abs(Ja).max()


def test_gtsam_adapter_maps_visual_inertial_graphs():
    """the adapter compiles against the GTSAM 4.2 API stubs with the navigation headers, and tells a velocity from a
    landmark by the key character (Vector3 == Point3 in GTSAM 4.2)"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DDYNOBA_WITH_GTSAM", "-DDYNOBA_FLOWPROJ_ACCESSORS",
                        "-I", os.path.join(root, "tests", "stubs"), "-I", os.path.join(root, "include"), "-x", "c++",
                        os.path.join(root, "include", "dynoba_gtsam_adapter.hpp")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    src = open(os.path.join(root, "include", "dynoba_gtsam_adapter.hpp")).read()
    for t in ("DYNOBA_COMBINED_IMU15", "DYNOBA_PRIOR_VEL3", "DYNOBA_PRIOR_BIAS6", "DYNOBA_VEL3", "DYNOBA_BIAS6",
              "dynoba_set_variable_order", "chr() == 'V'", "->R()", "omegaCoriolis"):
        assert t in src, t
    # the velocity branch comes before the landmark branch of the same value type
    assert src.index("isVelocityKey(kv.key)") < src.index("point_index_[kv.key]")
