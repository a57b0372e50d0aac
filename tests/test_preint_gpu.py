"""dynoba_imu_preintegrate_batch on the device: every case of tests/preint_cases.py against the 50-digit reference within
the a-priori bound, the same bits for an interval alone, in a batch of 10 000 ragged intervals, at batch sizes around the
CTA's warp count and on a repeated call, the host build of preint.cuh within the bound, and raw samples through the
preintegration and the graph builder into an LM solve."""
import numpy as np
import pytest

import preint_cases as PC
import test_preint as TP
from dynosam_b200 import binding, synth, synth_imu
from dynosam_b200.binding import Solver, imu_preintegrate_batch
from dynosam_b200.problem import COMBINED_IMU15, PRIOR_BIAS6, PRIOR_VEL3, FactorBlock, Problem

pytestmark = pytest.mark.gpu
CASES = TP.CASES


def _card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception:                                   # noqa: BLE001 -- the card name is a label only
        return "unknown card"


def _one(c):
    return imu_preintegrate_batch(c.P, [c.stamps], [c.acc_gyr], None if c.bh is None else [c.bh])


def test_device_equals_the_reference():
    res = {}
    for name, c in CASES.items():
        o = _one(c)
        res[name] = TP.errors(name, o["record"][0], o["cov"][0], o["sqrt_info"][0], o["status"][0])
    worst = max(((n, q, v) for n, r in res.items() for q, v in r.items()), key=lambda t: t[2])
    print(f"preint device worst: {worst[0]} {worst[1]} {worst[2]:.3g} of the tolerance ({_card()})")
    bad = {(n, q): v for n, r in res.items() for q, v in r.items() if not v <= 1.0}
    assert not bad, bad


def _ragged(n, seed=1):
    """n intervals of 2..40 samples with jittered dt around 5 ms, rotating, with bias_hat"""
    rng = np.random.default_rng(seed)
    st, ag = [], []
    for _ in range(n):
        m = int(rng.integers(2, 41))
        st.append(np.cumsum(np.concatenate([[rng.uniform(0, 10)], rng.uniform(0.004, 0.006, m - 1)])))
        ag.append(np.concatenate([rng.normal(0, 3, (m, 3)) + [0, 0, 9.81], rng.normal(0, 0.5, (m, 3))], 1))
    return st, ag, rng.normal(0, 0.01, (n, 6))


def _params():
    T = np.eye(4); T[:3, :3] = PC._rot((1, 2, -1), 0.7); T[:3, 3] = [0.1, -0.05, 0.2]
    return binding.imu_frontend_params((0.0, 9.8, 0.0), 0.2, 0.05, 0.02, 4e-5, 1e-3, T)


def test_same_bits_alone_in_batches_and_repeated():
    P = _params()
    st, ag, bh = _ragged(10000)
    full = imu_preintegrate_batch(P, st, ag, bh)
    again = imu_preintegrate_batch(P, st, ag, bh)
    for k in full:
        assert np.array_equal(full[k], again[k]), k
    assert (full["status"] == 0).all()
    for i in (0, 1, 3, 4, 5, 4999, 9999):
        o = imu_preintegrate_batch(P, [st[i]], [ag[i]], bh[i:i + 1])
        for k in full:
            assert np.array_equal(o[k][0], full[k][i]), (i, k)
    for n in (1, 2, 3, 4, 5, 7, 8, 9, 31, 33):                # around the 4 warps of a CTA
        for off in (0, 6):
            o = imu_preintegrate_batch(P, st[off:off + n], ag[off:off + n], bh[off:off + n])
            for k in full:
                assert np.array_equal(o[k], full[k][off:off + n]), (n, off, k)
    z = imu_preintegrate_batch(P, [], [])
    assert z["record"].shape == (0, 70) and z["status"].shape == (0,)


def test_device_equals_the_host_build(tmp_path):
    lib = TP.build_shim(tmp_path)
    P = _params()
    st, ag, bh = _ragged(500, seed=2)
    d = imu_preintegrate_batch(P, st, ag, bh)
    h = TP.host_batch(lib, P, list(zip(st, ag, bh)))
    assert np.array_equal(d["status"], h["status"])
    worst = 0.0
    for i in range(500):
        n = len(st[i]) - 1
        z = h["record"][i]
        for _, lo, hi in TP.BLOCKS:
            tol = 16*PC.EPS*(n + 1)*max(1.0, np.abs(z[lo:hi]).max())
            worst = max(worst, np.abs(d["record"][i, lo:hi] - z[lo:hi]).max()/tol)
        S = h["cov"][i]; dg = np.sqrt(np.diag(S))
        worst = max(worst, (np.abs(d["cov"][i] - S)/(32*PC.EPS*(n + 1)*np.outer(dg, dg))).max())
        kappa = np.linalg.cond(S/np.outer(dg, dg))
        R = h["sqrt_info"][i]
        worst = max(worst, np.abs(d["sqrt_info"][i] - R).max()/(32*PC.EPS*(n + 15)*kappa*np.abs(R).max()))
    print(f"preint device vs host worst {worst:.3g} of the tolerance")
    assert worst <= 1.0


def _vio_problem(base, X_gt, records, Rs, vel0):
    N = X_gt.shape[0]
    k = np.arange(1, N)
    blocks = [b for b in base.blocks if b.type != 1]                    # no odometry BetweenFactor: the IMU replaces it
    blocks += [FactorBlock(PRIOR_VEL3, np.array([[0]]), vel0[:1], np.array([synth_imu.VEL_PRIOR_SIGMA])),
               FactorBlock(PRIOR_BIAS6, np.array([[0]]), np.zeros((1, 6)), synth_imu.BIAS_PRIOR_SIGMA),
               FactorBlock(COMBINED_IMU15, np.stack([k - 1, k - 1, k, k, k - 1, k], 1), records, Rs.reshape(-1, 225))]
    return Problem(base.pose, base.point, calib=base.calib, blocks=blocks, pose_order=base.pose_order, vel=vel0,
                   bias=np.zeros((N, 6)), vel_order=np.arange(N, dtype=np.int32), bias_order=np.arange(N, dtype=np.int32))


def _builder_graph(base, records, Rs):
    """the base problem's frames and static observations through the graph builder with one preintegrated measurement per
    frame after the first (Gaussian point noise, so that the dense statement of tests/test_imu_gpu.py applies)"""
    import test_builder as TB
    from dynosam_b200.builder import GraphBuilder
    b = GraphBuilder(huber_k=0.0)
    TB._feed(base, b)
    for k in range(1, base.meta["n_frames"]):
        b.set_imu(k, records[k - 1], Rs[k - 1])
    return b


def test_raw_samples_to_builder_to_lm():
    """raw samples -> dynoba_imu_preintegrate_batch -> dynoba_builder_set_imu -> dynoba_builder_emit -> dynoba_optimize on a
    seeded stream, against (1) the same graph built from the 50-digit reference's records and R: the same LM iteration and
    inner-iteration counts and chi^2 to 1e-9; (2) GTSAM's LM stated in dense fp64 over tests/imu_reference.py's factor
    (tests/test_imu_gpu.py's _lm_host) on the emitted graph: the same counts, chi^2 to 1e-6, velocities and biases to 1e-6"""
    import preint_reference as PR
    import test_imu_gpu as TIG
    xi = np.array([0.0, 0.004, 0.0, 0.02, 0.0, 1.0])
    base = synth.make_problem(n_frames=20, n_objects=0, n_static=150, n_dynamic=0, seed=23, robust=False)
    X_gt = base.meta["gt_camera"]
    st, ag = synth_imu.imu_stream(X_gt, xi, samples_per_frame=10, bias_true=np.array([0.02, -0.01, 0.03, 1e-3, -2e-3, 5e-4]), seed=4)
    P = binding.imu_frontend_params(synth_imu.GRAVITY, 0.2, 0.05, 0.02, 4e-5, 1e-3)
    d = imu_preintegrate_batch(P, st, ag)
    assert (d["status"] == 0).all()
    Pm = PR.params(P); ref_rec, ref_R = [], []
    for s_, a_ in zip(st, ag):
        z, _, R = PR.preintegrate(Pm, s_, a_)
        ref_rec.append([float(x) for x in z]); ref_R.append(np.array([[float(R[i, j]) for j in range(15)] for i in range(15)]))
    runs = []
    for rec, Rs in ((d["record"], d["sqrt_info"]), (np.array(ref_rec), np.array(ref_R))):
        b = _builder_graph(base, rec, Rs)
        s = Solver(); b.emit(s)
        runs.append(s.optimize())
        n = base.meta["n_frames"]; vel = np.zeros((n, 3)); bias = np.zeros((n, 6))
        assert s.lib.dynoba_get_variables(s.h, binding.VEL3, n, binding._dp(vel)) == 0
        assert s.lib.dynoba_get_variables(s.h, binding.BIAS6, n, binding._dp(bias)) == 0
        s.close()
        if len(runs) == 1:
            q = b.problem(); dev_nav = (vel, bias)
        b.close()
    a, r = runs
    assert a["iterations"] == r["iterations"] and a["inner_iterations"] == r["inner_iterations"], (a, r)
    assert abs(a["error_final"] - r["error_final"]) <= 1e-9*abs(r["error_final"]), (a, r)
    assert abs(a["error_initial"] - r["error_initial"]) <= 1e-9*abs(r["error_initial"]), (a, r)
    xh, eh, ith, innh = TIG._lm_host(q, (q.pose.copy(), q.point.copy(), q.vel.copy(), q.bias.copy()))
    assert (a["iterations"], a["inner_iterations"]) == (ith, innh), (a, ith, innh)
    assert a["error_final"] == pytest.approx(eh, rel=1e-6)
    assert np.abs(dev_nav[0] - xh[2]).max() <= 1e-6*max(1.0, np.abs(xh[2]).max()) and np.abs(dev_nav[1] - xh[3]).max() <= 1e-6


def test_noise_free_samples_recover_velocities_and_bias():
    """noise-free samples at 400 per frame and noise-free points: the minimum is the true trajectory, velocities and zero
    bias, to the preintegration's first-order integration error (2e-3, as tests/test_imu_gpu.py states it)"""
    xi = np.array([0.0, 0.004, 0.0, 0.02, 0.0, 1.0])
    base = synth.make_problem(n_frames=10, n_objects=0, n_static=150, n_dynamic=0, seed=17, robust=False, meas_noise=0.0)
    X_gt = base.meta["gt_camera"]
    R = X_gt[:, :9].reshape(-1, 3, 3)
    vel_gt = np.einsum("nij,j->ni", R, synth_imu.body_rates(xi)[1])
    st, ag = synth_imu.imu_stream(X_gt, xi, samples_per_frame=400, bias_true=np.zeros(6), noise=False)
    P = binding.imu_frontend_params(synth_imu.GRAVITY, 0.2, 0.05, 0.02, 4e-5, 1e-3)
    d = imu_preintegrate_batch(P, st, ag)
    assert (d["status"] == 0).all()
    p = _vio_problem(base, X_gt, d["record"], d["sqrt_info"], vel_gt + 0.05*np.random.default_rng(1).normal(size=vel_gt.shape))
    p.vel[0] = vel_gt[0]
    s = Solver(p)
    s.optimize(relative_error_tol=1e-14, absolute_error_tol=1e-14)
    vel, bias = s.nav_values()
    pose, _, _ = s.values()
    s.close()
    assert np.abs(vel - vel_gt).max() < 2e-3 and np.abs(bias).max() < 2e-3
    assert np.abs(pose[:, 9:] - X_gt[:, 9:]).max() < 2e-3
