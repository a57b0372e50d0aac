"""Visual-inertial graphs on the device: COMBINED_IMU15, PRIOR_VEL3 / PRIOR_BIAS6 and the velocity / bias variables of the
reduced system, against the independent numpy statement (imu_reference.py), dense fp64 algebra and scipy."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg
import scipy.optimize

import imu_reference as IR
from dynosam_b200 import lie, synth
from dynosam_b200.binding import BIAS6, ERR_BAD_ARG, ERR_UNSUPPORTED, VEL3, DynobaError, Solver
from dynosam_b200.problem import (CLASS_DIM, COMBINED_IMU15, JCOLS, POSE2POINT3, PRIOR6, PRIOR_BIAS6, PRIOR_VEL3, SLOT_CLASS,
                                  FactorBlock, Problem)

pytestmark = pytest.mark.gpu


def _vio(seed=11, **kw):
    cfg = dict(n_frames=12, n_objects=1, n_static=120, n_dynamic=60, seed=seed, imu=True)
    cfg.update(kw)
    p = synth.make_problem(**cfg)
    rng = np.random.default_rng(seed)
    p.bias = p.bias + rng.normal(0, 1, p.bias.shape)*np.array([0.05]*3 + [0.01]*3)    # bias != biasHat
    p.vel = p.vel + rng.normal(0, 0.5, p.vel.shape)
    return p


def _imu_args(p, row):
    i0, v0, i1, v1, b0, b1 = row
    return [p.pose[i0], p.vel[v0], p.pose[i1], p.vel[v1], p.bias[b0], p.bias[b1]]


def test_imu_linearization_against_reference():
    p = _vio()
    # large rotations on the camera poses (the landmarks do not matter here)
    rng = np.random.default_rng(2)
    p.pose[:12] = lie.compose(p.pose[:12], lie.se3_exp(np.concatenate([rng.normal(0, 0.5, (12, 3)), rng.normal(0, 1, (12, 3))], 1)))
    s = Solver(p)
    s.linearize()
    for bi, blk in enumerate(p.blocks):
        if blk.type not in (COMBINED_IMU15, PRIOR_VEL3, PRIOR_BIAS6):
            continue
        A, b = s.linearization(bi)
        err = s.factor_errors(bi)
        if blk.type == COMBINED_IMU15:
            R = blk.sigma.reshape(-1, 15, 15)
            for f in range(blk.n):
                args = _imu_args(p, blk.idx[f])
                r = IR.imu_residual(*args, blk.meas[f])
                bw = -R[f]@r
                assert np.abs(b[f] - bw).max() <= 1e-9*np.abs(bw).max()
                Jw = R[f]@IR.imu_jacobian(*args, blk.meas[f])              # closed form, pinned to central differences on the CPU
                Jn = R[f]@IR.imu_numeric_jacobian(args, blk.meas[f])
                for c0, d in zip((0, 6, 9, 15, 18, 24), (6, 3, 6, 3, 6, 6)):      # every Jacobian block
                    assert np.abs(A[f][:, c0:c0 + d] - Jw[:, c0:c0 + d]).max() <= 1e-9*np.abs(Jw).max(), (f, c0)
                    assert np.abs(A[f][:, c0:c0 + d] - Jn[:, c0:c0 + d]).max() <= 1e-6*np.abs(Jn).max(), (f, c0)
                Sigma = np.linalg.inv(R[f].T@R[f])
                e_ref = 0.5*r@scipy.linalg.solve(Sigma, r, assume_a="pos")
                assert err[f] == pytest.approx(e_ref, rel=1e-6)
        else:
            x = p.vel if blk.type == PRIOR_VEL3 else p.bias
            isig = 1.0/np.broadcast_to(blk.sigma, (blk.n, blk.sigma.shape[-1]))
            for f in range(blk.n):
                r = (x[blk.idx[f, 0]] - blk.meas[f])*isig[f]
                assert np.allclose(b[f], -r, rtol=1e-12, atol=0) and np.allclose(A[f], np.diag(isig[f]*np.ones(x.shape[1])), rtol=1e-15, atol=0)
                assert err[f] == pytest.approx(0.5*r@r, rel=1e-12)


def _dense_system(p, s, lam):
    """J^T J + lam I and J^T b over [poses 6 | points 3 | flows 2 | velocities 3 | biases 6] from the device's own Jacobians"""
    counts = [p.n_pose, p.n_point, p.n_flow, p.n_vel, p.n_bias]
    base = np.concatenate([[0], np.cumsum([n*d for n, d in zip(counts, (6, 3, 2, 3, 6))])])
    cls_base = {0: (base[0], 6), 1: (base[1], 3), 2: (base[2], 2), 3: (base[3], 3), 4: (base[4], 6)}
    n = base[-1]
    H = np.zeros((n, n)); g = np.zeros(n)
    for bi, blk in enumerate(p.blocks):
        A, b = s.linearization(bi)
        cols = []
        for f in range(blk.n):
            idx = []
            for k, c in enumerate(SLOT_CLASS[blk.type]):
                o, d = cls_base[c]
                idx.extend(range(o + d*blk.idx[f, k], o + d*blk.idx[f, k] + d))
            cols.append(idx)
        cols = np.array(cols)
        for f in range(blk.n):
            H[np.ix_(cols[f], cols[f])] += A[f].T@A[f]
            g[cols[f]] += A[f].T@b[f]
    H += lam*np.eye(n)
    return H, g, base


@pytest.mark.parametrize("ncells", [-1, 0, 2, 4])
def test_imu_reduced_system_and_step(ncells):
    p = _vio(seed=5, n_frames=40, n_objects=2, n_static=400, n_dynamic=200)
    s = Solver(p)
    s.set_partition(ncells)
    s.linearize()
    lam = 1e-3
    H, g, base = _dense_system(p, s, lam)
    P = np.r_[0:base[1], base[3]:base[5]]          # poses, velocities, biases
    L = np.r_[base[1]:base[3]]                     # points, flows
    Hll = H[np.ix_(L, L)]
    S_ref = H[np.ix_(P, P)] - H[np.ix_(P, L)]@np.linalg.solve(Hll, H[np.ix_(L, P)])
    g_ref = g[P] - H[np.ix_(P, L)]@np.linalg.solve(Hll, g[L])
    S, gS = s.reduced_system(lam)
    d = np.sqrt(np.diag(S_ref))
    assert (np.abs(S - S_ref)/np.outer(d, d)).max() <= 1e-11
    assert (np.abs(gS - g_ref)/d).max() <= 1e-11*max(1.0, (np.abs(g_ref)/d).max())
    delta = s.solve(lam)
    ref = np.linalg.solve(H, g)
    dd = np.sqrt(np.diag(H))
    assert (np.abs(delta - ref)*dd).max() <= 1e-6*(np.abs(ref)*dd).max()
    info = s.info()
    assert info["reduced_dim"] == 6*(p.n_pose + p.n_vel + p.n_bias)


def _graph_residual(p, x):
    """whitened residual of a graph of POSE2POINT3 / PRIOR6 / PRIOR_VEL3 / PRIOR_BIAS6 / COMBINED_IMU15 factors (Gaussian)"""
    pose, point, vel, bias = x
    out = []
    for blk in p.blocks:
        isig = None if blk.type == COMBINED_IMU15 else 1.0/np.broadcast_to(blk.sigma, (blk.n, blk.sigma.shape[-1]))
        if blk.type == POSE2POINT3:
            X = pose[blk.idx[:, 0]]
            q = lie.transform_to(X, point[blk.idx[:, 1]])
            out.append(((q - blk.meas)*isig).ravel())
        elif blk.type == PRIOR6:
            for f in range(blk.n):
                X = pose[blk.idx[f, 0]]; M = blk.meas[f]
                d = lie.compose(lie.inverse(X[None]), M[None])[0]
                out.append(-np.concatenate([IR.log3(d[:9].reshape(3, 3)), _se3_log_t(d)])*isig[f])
        elif blk.type in (PRIOR_VEL3, PRIOR_BIAS6):
            v = vel if blk.type == PRIOR_VEL3 else bias
            out.append(((v[blk.idx[:, 0]] - blk.meas)*isig).ravel())
        elif blk.type == COMBINED_IMU15:
            R = blk.sigma.reshape(-1, 15, 15)
            for f in range(blk.n):
                i0, v0, i1, v1, b0, b1 = blk.idx[f]
                out.append(R[f]@IR.imu_residual(pose[i0], vel[v0], pose[i1], vel[v1], bias[b0], bias[b1], blk.meas[f]))
        else:
            raise AssertionError(blk.type)
    return np.concatenate(out)


def _se3_log_t(d):
    w = IR.log3(d[:9].reshape(3, 3)); t = d[9:]
    th = np.linalg.norm(w)
    if th < 1e-10:
        return t
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])/th
    return t - 0.5*th*W@t + (1 - th/(2*np.tan(0.5*th)))*W@W@t


def test_imu_lm_minimum_against_scipy_least_squares():
    p = synth.make_problem(n_frames=6, n_objects=0, n_static=40, n_dynamic=0, seed=8, robust=False, imu=True)
    x0 = (p.pose.copy(), p.point.copy(), p.vel.copy(), p.bias.copy())
    npo, npt, nv, nb = p.n_pose, p.n_point, p.n_vel, p.n_bias

    def unpack(d):
        o = 0
        pose = np.stack([IR.retract_pose(x0[0][i], d[o + 6*i:o + 6*i + 6]) for i in range(npo)]); o += 6*npo
        point = x0[1] + d[o:o + 3*npt].reshape(-1, 3); o += 3*npt
        vel = x0[2] + d[o:o + 3*nv].reshape(-1, 3); o += 3*nv
        bias = x0[3] + d[o:o + 6*nb].reshape(-1, 6)
        return pose, point, vel, bias
    res = scipy.optimize.least_squares(lambda d: _graph_residual(p, unpack(d)), np.zeros(6*npo + 3*npt + 3*nv + 6*nb),
                                       method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=20000)
    e_min = 0.5*float(res.fun@res.fun)
    s = Solver(p)
    e0 = s.error()
    assert e0 == pytest.approx(0.5*float(_graph_residual(p, x0)@_graph_residual(p, x0)), rel=1e-9)
    st = s.optimize(relative_error_tol=1e-14, absolute_error_tol=1e-14, max_iterations=200)
    assert st["error_final"] == pytest.approx(e_min, rel=1e-6)
    vel, bias = s.nav_values()
    _, _, vref, bref = unpack(res.x)
    assert np.abs(vel - vref).max() < 1e-5 and np.abs(bias - bref).max() < 1e-5


def _graph_linearize(p, x):
    """whitened (r, J) of the Gaussian POSE2POINT3 / PRIOR6 / PRIOR_VEL3 / PRIOR_BIAS6 / COMBINED_IMU15 graph over
    [poses 6 | points 3 | velocities 3 | biases 6], the Jacobians as the device forms them (PRIOR6: H = I, GTSAM's)"""
    pose, point, vel, bias = x
    o_pt = 6*p.n_pose; o_v = o_pt + 3*p.n_point; o_b = o_v + 3*p.n_vel; n = o_b + 6*p.n_bias
    rows, Js = [], []
    for blk in p.blocks:
        for f in range(blk.n):
            Jr = np.zeros((0, n))
            if blk.type == POSE2POINT3:
                i, l = blk.idx[f]; X = pose[i]; R = X[:9].reshape(3, 3); isg = 1.0/blk.sigma[0]
                q = R.T@(point[l] - X[9:]); r = (q - blk.meas[f])*isg
                Jr = np.zeros((3, n)); Jr[:, 6*i:6*i + 3] = IR._skew(q)*isg; Jr[:, 6*i + 3:6*i + 6] = -np.eye(3)*isg
                Jr[:, o_pt + 3*l:o_pt + 3*l + 3] = R.T*isg
            elif blk.type == PRIOR6:
                i = blk.idx[f, 0]; isg = 1.0/blk.sigma
                d = lie.compose(lie.inverse(pose[i][None]), blk.meas[f][None])[0]
                r = -np.concatenate([IR.log3(d[:9].reshape(3, 3)), _se3_log_t(d)])*isg
                Jr = np.zeros((6, n)); Jr[:, 6*i:6*i + 6] = np.diag(isg*np.ones(6))
            elif blk.type in (PRIOR_VEL3, PRIOR_BIAS6):
                dim, o, v = (3, o_v, vel) if blk.type == PRIOR_VEL3 else (6, o_b, bias)
                i = blk.idx[f, 0]; isg = 1.0/blk.sigma*np.ones(dim)
                r = (v[i] - blk.meas[f])*isg
                Jr = np.zeros((dim, n)); Jr[:, o + dim*i:o + dim*i + dim] = np.diag(isg)
            else:
                Rs = blk.sigma.reshape(-1, 15, 15)[f]
                i0, v0, i1, v1, b0, b1 = blk.idx[f]
                args = [pose[i0], vel[v0], pose[i1], vel[v1], bias[b0], bias[b1]]
                r = Rs@IR.imu_residual(*args, blk.meas[f]); J = Rs@IR.imu_jacobian(*args, blk.meas[f])
                Jr = np.zeros((15, n))
                for c0, d, off in zip((0, 6, 9, 15, 18, 24), (6, 3, 6, 3, 6, 6),
                                      (6*i0, o_v + 3*v0, 6*i1, o_v + 3*v1, o_b + 6*b0, o_b + 6*b1)):
                    Jr[:, off:off + d] += J[:, c0:c0 + d]
            rows.append(r); Js.append(Jr)
    return np.concatenate(rows), np.concatenate(Js)


def _retract_all(p, x, d):
    pose, point, vel, bias = x
    o_pt = 6*p.n_pose; o_v = o_pt + 3*p.n_point; o_b = o_v + 3*p.n_vel
    return (np.stack([IR.retract_pose(pose[i], d[6*i:6*i + 6]) for i in range(p.n_pose)]), point + d[o_pt:o_v].reshape(-1, 3),
            vel + d[o_v:o_b].reshape(-1, 3), bias + d[o_b:].reshape(-1, 6))


def _lm_host(p, x, lambda_initial=1e-5, lambda_factor=10.0, lambda_upper=1e5, min_fidelity=1e-3, rel_tol=1e-5, abs_tol=1e-5,
             max_iterations=100):
    """GTSAM 4.2.0 LevenbergMarquardtOptimizer (iterate / tryLambda / defaultOptimize, lambda * I damping) with dense
    fp64 algebra, on the graph of _graph_linearize"""
    err = lambda y: 0.5*float(_graph_residual(p, y)@_graph_residual(p, y))
    e, lam, it, inner = err(x), lambda_initial, 0, 0
    new = e
    while True:
        cur = new
        r, J = _graph_linearize(p, x)
        H, g = J.T@J, -J.T@r
        while True:
            try:
                L = np.linalg.cholesky(H + lam*np.eye(H.shape[0]))
                d = scipy.linalg.cho_solve((L, True), g); solved = True
            except np.linalg.LinAlgError:
                solved = False
            success = stop = False
            if solved:
                xc = _retract_all(p, x, d); ne = err(xc)
                lin = 0.5*g@d + 0.5*lam*d@d
                if lin >= 0:
                    cost = e - ne
                    if lin > np.finfo(float).eps*0.5*float(r@r):
                        success = cost/lin > min_fidelity
                    stop = abs(cost) < rel_tol*e
            if success:
                x, e, lam = xc, ne, lam/lambda_factor; it += 1; inner += 1; break
            elif not stop:
                lam *= lambda_factor; inner += 1
                if lam >= lambda_upper:
                    break
            else:
                break
        new = e
        if not (it < max_iterations and not (new <= 0.0 or (cur - new)/cur <= rel_tol or (cur - new) <= abs_tol) and np.isfinite(cur)):
            break
    return x, e, it, inner


@pytest.mark.parametrize("n_frames,n_static", [(20, 120), (60, 400)])
def test_imu_lm_trace_against_host_lm(n_frames, n_static):
    """full LM on VIO graphs: equal outer / inner iteration counts and final chi^2 <= 1e-6 against the host statement"""
    p = synth.make_problem(n_frames=n_frames, n_objects=0, n_static=n_static, n_dynamic=0, seed=13, robust=False, imu=True)
    x0 = (p.pose.copy(), p.point.copy(), p.vel.copy(), p.bias.copy())
    xh, eh, ith, innh = _lm_host(p, x0)
    s = Solver(p)
    st = s.optimize()
    assert (st["iterations"], st["inner_iterations"]) == (ith, innh)
    assert st["error_final"] == pytest.approx(eh, rel=1e-6)
    vel, bias = s.nav_values()
    assert np.abs(vel - xh[2]).max() <= 1e-6*max(1.0, np.abs(xh[2]).max()) and np.abs(bias - xh[3]).max() <= 1e-6


def test_imu_recovers_true_states_on_noise_free_data():
    """noise-free IMU samples and points, zero true bias: the minimum is the true trajectory, velocities and biases"""
    from dynosam_b200 import synth_imu as SI
    base = synth.make_problem(n_frames=10, n_objects=0, n_static=150, n_dynamic=0, seed=17, robust=False, meas_noise=0.0)
    X_gt = base.meta["gt_camera"]
    vel0, bias0, blocks, meta = SI.add_imu_chain(X_gt, np.array([0.0, 0.004, 0.0, 0.02, 0.0, 1.0]), 99, samples_per_frame=400,
                                                 bias_true=np.zeros(6), noise=False)
    odo = [b for b in base.blocks if b.type != 1]
    p = Problem(base.pose, base.point, calib=base.calib, blocks=odo + blocks, pose_order=base.pose_order, vel=vel0, bias=bias0,
                vel_order=np.arange(10, dtype=np.int32), bias_order=np.arange(10, dtype=np.int32))
    s = Solver(p)
    s.optimize(relative_error_tol=1e-14, absolute_error_tol=1e-14)
    vel, bias = s.nav_values()
    pose, _, _ = s.values()
    # what is left is the preintegration's first-order integration error at 400 samples per frame
    assert np.abs(vel - meta["vel_gt"]).max() < 2e-3 and np.abs(bias).max() < 2e-3
    assert np.abs(pose[:, 9:] - X_gt[:, 9:]).max() < 2e-3


def _plain(seed=3):
    return synth.make_problem(n_frames=20, n_objects=1, n_static=300, n_dynamic=100, seed=seed)


def _same_run(x, y, tol=1e-8):
    """Equal up to the order of the fp64 RED atomics that accumulate S and g_S.  With no velocity / bias the host takes
    exactly the code path it took before those kinds existed (NP == np), but the device sums S with fire-and-forget
    atomics whose order changes from run to run of the SAME handle -- so two handles are compared at that run-to-run
    level, not bit for bit: S and g_S to 1e-12 in units of diag S; the step and the LM result, in which the condition
    number of S amplifies that reassociation, to `tol` relative."""
    return np.abs(x - y).max(initial=0.0) <= tol*max(np.abs(x).max(initial=0.0), 1e-300)


def _same_system(a, b, lam=1e-3):
    Sa, ga = a.reduced_system(lam); Sb, gb = b.reduced_system(lam)
    d = np.sqrt(np.diag(Sa))
    return Sa.shape == Sb.shape and (np.abs(Sa - Sb)/np.outer(d, d)).max() <= 1e-12 and (np.abs(ga - gb)/d).max() <= 1e-12*max(1.0, (np.abs(ga)/d).max())


def test_empty_nav_sets_change_nothing():
    p = _plain()
    a = Solver(p)
    b = Solver(p)
    b.set_variables(VEL3, np.zeros((0, 3))); b.set_variables(BIAS6, np.zeros((0, 6)))
    b.set_variable_order(VEL3, np.zeros(0)); b.set_variable_order(BIAS6, np.zeros(0))
    assert a.info() == b.info()
    assert _same_system(a, b)
    assert _same_run(a.solve(1e-3), b.solve(1e-3))
    sa, sb = a.optimize(), b.optimize()
    for k in ("iterations", "inner_iterations", "lambda_final", "reduced_dim", "bandwidth"):
        assert sa[k] == sb[k], k
    assert sa["error_initial"] == sb["error_initial"]
    assert sa["error_final"] == pytest.approx(sb["error_final"], rel=1e-10)
    for x, y in zip(a.values(), b.values()):
        assert _same_run(x, y)


@pytest.mark.parametrize("cfg", ["C1", "C1_wide"])
def test_imu_lm_runs_at_c1_size(cfg):
    kw = dict(n_frames=20, n_objects=1, n_static=700, n_dynamic=300) if cfg == "C1" else dict(n_frames=120, n_objects=3, n_static=4000, n_dynamic=1500)
    p = synth.make_problem(seed=21, imu=True, **kw)
    s = Solver(p)
    st = s.optimize()
    assert st["iterations"] > 0 and st["error_final"] < st["error_initial"]
    assert st["reduced_dim"] == 6*(p.n_pose + p.n_vel + p.n_bias)
    vel, bias = s.nav_values()
    assert np.isfinite(vel).all() and np.isfinite(bias).all()
    assert not np.array_equal(vel, p.vel) and not np.array_equal(bias, p.bias)
    # one reduced solve, with the step taken by dynoba_retract, lowers the error like the LM's first step
    s2 = Solver(p)
    d = s2.solve(1e-5)
    assert d.shape[0] == 6*p.n_pose + 3*p.n_point + 2*p.n_flow + 3*p.n_vel + 6*p.n_bias
    s2.retract(d)
    assert s2.error() < st["error_initial"]


def _expect(status, fn, *a):
    with pytest.raises(DynobaError) as e:
        fn(*a)
    assert e.value.status == status


def test_refusals():
    p = _vio()
    s = Solver(p)
    lib, h = s.lib, s.h
    # the linear prior, the marginal, shard and reduce with velocity / bias variables
    _expect(ERR_UNSUPPORTED, s.add_linear_prior, np.array([0]), p.pose[:1], np.eye(6), np.zeros(6))
    _expect(ERR_UNSUPPORTED, s.marginal, np.array([p.n_pose - 1]))
    _expect(ERR_UNSUPPORTED, s.set_shard, 0, 2, lambda *a: None)
    _expect(ERR_UNSUPPORTED, s.set_reduce, lambda *a: None)
    imu = next(b for b in p.blocks if b.type == COMBINED_IMU15)
    # robust_k on the IMU type
    _expect(ERR_UNSUPPORTED, s.add_factors, FactorBlock(COMBINED_IMU15, imu.idx, imu.meas, imu.sigma, robust_k=1.0))
    # sigma_dim 225 on another type; an IMU block with Isotropic noise
    _expect(ERR_BAD_ARG, s.add_factors, FactorBlock(PRIOR_BIAS6, np.array([[0]]), np.zeros((1, 6)), np.ones(225)))
    _expect(ERR_BAD_ARG, s.add_factors, FactorBlock(COMBINED_IMU15, imu.idx, imu.meas, np.array([1.0])))
    # a non-finite R
    bad = imu.sigma.copy(); bad[0, 3] = np.nan
    _expect(ERR_BAD_ARG, s.add_factors, FactorBlock(COMBINED_IMU15, imu.idx, imu.meas, bad))
    # an order hint for poses through the variable-kind entry point
    st = lib.dynoba_set_variable_order(h, 0, 0, C.cast(None, C.POINTER(C.c_int32)))
    assert st == ERR_BAD_ARG
    # nav variables added after a linear prior: refused when the graph is built
    q = _plain()
    t = Solver(q)
    t.add_linear_prior(np.array([0]), q.pose[:1], np.eye(6), np.zeros(6))
    t.set_variables(VEL3, np.zeros((2, 3)))
    _expect(ERR_UNSUPPORTED, t.finalize)
    # the handle that refused still solves its graph
    s.optimize(max_iterations=2)


def test_problem_without_pose_order_keeps_frame_interleaving():
    """no hints at all: every kind ranks by index, so X_k, V_k, b_k of the synthetic chain stay adjacent"""
    p = _vio(n_objects=0, n_dynamic=0)
    hinted = Solver(p).info()
    p.pose_order = None; p.vel_order = None; p.bias_order = None
    s = Solver(p)
    assert s.info() == hinted
    assert _same_system(s, Solver(_vio(n_objects=0, n_dynamic=0)))


def test_value_refresh_keeps_other_kinds():
    p = _vio(n_objects=0, n_dynamic=0)
    s = Solver(p)
    s.finalize()
    s.set_variables(VEL3, p.vel + 1.0)
    vel, bias = s.nav_values()
    assert np.array_equal(vel, p.vel + 1.0) and np.array_equal(bias, p.bias)
    pose, _, _ = s.values()
    assert np.array_equal(pose, p.pose)
    s.set_variables(0, p.pose)
    vel2, bias2 = s.nav_values()
    assert np.array_equal(vel2, p.vel + 1.0) and np.array_equal(bias2, p.bias)


def test_problem_copy_keeps_nav():
    p = _vio(n_objects=0, n_dynamic=0)
    q = p.copy()
    assert isinstance(q, Problem) and np.array_equal(q.vel, p.vel) and np.array_equal(q.bias, p.bias)
    assert CLASS_DIM[3] == 3 and CLASS_DIM[4] == 6 and JCOLS[COMBINED_IMU15] == 30
