"""The sliding window (dynoba_add_linear_prior_vars + dynoba_marginal_vars) on visual-inertial graphs: a
gtsam::LinearContainerFactor(HessianFactor) whose slots are poses, velocities and biases, and the Schur marginal of the
last frames' X, H, V, b with the HessianFactor constant f, against dense fp64 algebra over the device's own Jacobians
(test_imu_gpu._dense_system) and the LinearContainerFactor algebra [GTSAM-ext LinearContainerFactor::{error,linearize}]:
    error(x) = 1/2 d^T G d - g^T d + 1/2 f,  d = linPoint.localCoordinates(x);   linearize -> HessianFactor(G, g - G d)
with d = Logmap(lin^-1 x) for a Pose3 and x - lin for a Vector3 velocity or an imuBias::ConstantBias [acc; gyro]."""
import dataclasses

import numpy as np
import pytest

import imu_reference as IR
import selinv_reference as SI
from test_imu_gpu import _dense_system, _se3_log_t, _vio
from dynosam_b200 import lie, synth
from dynosam_b200.binding import (BIAS6, ERR_BAD_ARG, ERR_UNSUPPORTED, POSE6, VEL3, DynobaError, Solver, TANGENT_DIM)
from dynosam_b200.problem import SLOT_CLASS, FactorBlock, Problem

pytestmark = pytest.mark.gpu

KIND_CLASS = {POSE6: 0, VEL3: 3, BIAS6: 4}       # variable kind -> column class of _dense_system


def _cols(base, kinds, idx):
    """columns of the slots (kinds[i], idx[i]) in _dense_system's layout, in slot order"""
    out = []
    for k, i in zip(kinds, idx):
        d = TANGENT_DIM[k]
        out.extend(range(base[KIND_CLASS[k]] + d*i, base[KIND_CLASS[k]] + d*i + d))
    return np.array(out)


def _value(p, k, i):
    return (p.pose, p.vel, p.bias)[(POSE6, VEL3, BIAS6).index(k)][i]


def _local(p, kinds, idx, lin):
    """localCoordinates of the slots at p's values from the packed linearisation point"""
    out, o = [], 0
    for k, i in zip(kinds, idx):
        x = _value(p, k, i)
        if k == POSE6:
            d = lie.compose(lie.inverse(lin[o:o + 12][None]), x[None])[0]
            out.append(np.concatenate([IR.log3(d[:9].reshape(3, 3)), _se3_log_t(d)])); o += 12
        else:
            w = x.size
            out.append(x - lin[o:o + w]); o += w
    return np.concatenate(out)


def _last_frames(p, k):
    """(kinds, idx) of every pose (camera and object motion), velocity and bias of the last k frames"""
    F = p.meta["n_frames"]
    kinds, idx = [], []
    for kind, order in ((POSE6, p.pose_order), (VEL3, p.vel_order), (BIAS6, p.bias_order)):
        sel = np.flatnonzero(order >= F - k)
        kinds += [kind]*sel.size; idx += list(sel)
    return np.array(kinds, np.int32), np.array(idx, np.int32)


def _random_prior(rng, p, kinds, idx, f=0.7):
    D = sum(TANGENT_DIM[int(k)] for k in kinds)
    A = rng.normal(0, 1, (D + 4, D)); G = A.T @ A*30.0 + 5.0*np.eye(D)
    lin = []
    for k, i in zip(kinds, idx):
        x = _value(p, k, i)
        lin.append(lie.retract(x[None], rng.normal(0, 0.02, (1, 6)))[0] if k == POSE6 else x + rng.normal(0, 0.02, x.size))
    return dict(kind=np.asarray(kinds, np.int32), idx=np.asarray(idx, np.int32), lin=np.concatenate(lin), G=G,
                g=rng.normal(0, 3.0, D), f=f)


def _with_values(p, s):
    pose, point, flow = s.values(); vel, bias = s.nav_values()
    return dataclasses.replace(p, pose=pose, point=point, flow=flow, vel=vel, bias=bias, linear_priors=[])


def _prior_error(p, pr):
    d = _local(p, pr["kind"], pr["idx"], pr["lin"])
    return 0.5*d @ pr["G"] @ d - pr["g"] @ d + 0.5*pr["f"], d


def test_typed_prior_error_step_and_lm():
    rng = np.random.default_rng(3)
    p = _vio()
    kinds, idx = _last_frames(p, 3)
    perm = rng.permutation(kinds.size)                                   # kinds interleaved in the slot order
    pr = _random_prior(rng, p, kinds[perm], idx[perm])
    s = Solver(dataclasses.replace(p, linear_priors=[pr]))
    s0 = Solver(p)
    e_prior, d0 = _prior_error(p, pr)
    e_ref = s0.error() + e_prior
    assert abs(s.error() - e_ref) <= 1e-9*abs(e_ref)
    # damped step: dense normal equations of the graph plus the relinearised Hessian factor (G, g - G d)
    lam = 1e-3
    s0.linearize()
    H, g, base = _dense_system(p, s0, lam)
    cols = _cols(base, pr["kind"], pr["idx"])
    H[np.ix_(cols, cols)] += pr["G"]; g[cols] += pr["g"] - pr["G"] @ d0
    ref = np.linalg.solve(H, g)
    d = s.solve(lam)
    assert np.linalg.norm(d - ref) <= 1e-6*np.linalg.norm(ref), np.linalg.norm(d - ref)/np.linalg.norm(ref)
    # LM lowers the error and its final error counts the prior
    st = s.optimize(max_iterations=8)
    q = _with_values(p, s)
    e1 = Solver(q).error() + _prior_error(q, pr)[0]
    assert st["error_final"] < st["error_initial"]
    assert abs(st["error_final"] - e1) <= 1e-8*abs(e1)


def test_pose_only_typed_prior_equals_the_legacy_prior():
    """the typed entry point with POSE6 slots builds the table the legacy one implies: the error is bit for bit the same,
    the step and the LM result agree to the spread that the order of the band's fp64 atomics gives two legacy handles"""
    rng = np.random.default_rng(4)
    p = synth.make_problem(n_frames=20, n_objects=1, n_static=300, n_dynamic=100, seed=3)
    idx = np.flatnonzero(p.pose_order >= 15).astype(np.int32)
    pr = _random_prior(rng, p, np.full(idx.size, POSE6, np.int32), idx)
    legacy = dict(idx=pr["idx"], lin=pr["lin"].reshape(-1, 12), G=pr["G"], g=pr["g"], f=pr["f"])
    a1, a2 = (Solver(dataclasses.replace(p, linear_priors=[legacy])) for _ in range(2))
    b = Solver(dataclasses.replace(p, linear_priors=[pr]))
    assert a1.error() == b.error()

    def rel(x, y):
        return np.abs(x - y).max()/np.abs(x).max()
    lam = 1e-3
    da1, da2, db = a1.solve(lam), a2.solve(lam), b.solve(lam)
    spread = rel(da1, da2)
    assert spread <= 1e-10 and rel(da1, db) <= max(2*spread, 1e-10), (spread, rel(da1, db))
    sa1, sa2, sb = a1.optimize(), a2.optimize(), b.optimize()
    assert sb["iterations"] == sa1["iterations"] and sb["inner_iterations"] == sa1["inner_iterations"]
    es = abs(sa1["error_final"] - sa2["error_final"])/sa1["error_final"]
    assert abs(sb["error_final"] - sa1["error_final"])/sa1["error_final"] <= max(2*es, 1e-10)
    xa1, xa2, xb = (s.values()[0] for s in (a1, a2, b))
    vs = rel(xa1, xa2)
    assert vs <= 1e-8 and rel(xa1, xb) <= max(2*vs, 1e-8)


def _check_marginal(p, s, kinds, idx):
    """G, g, f of marginal_vars against the dense Schur complement of the device's own linearisation"""
    s.linearize()
    H, gd, base = _dense_system(p, s, 0.0)
    sum_b2 = sum(float(np.sum(s.linearization(bi)[1]**2)) for bi in range(len(p.blocks)))
    G, g, f = s.marginal_vars(kinds, idx)
    K = _cols(base, kinds, idx)
    E = np.setdiff1d(np.arange(H.shape[0]), K)
    X = np.linalg.solve(H[np.ix_(E, E)], np.concatenate([H[np.ix_(E, K)], gd[E, None]], 1))
    Gk = H[np.ix_(K, K)] - H[np.ix_(K, E)] @ X[:, :-1]
    gk = gd[K] - H[np.ix_(K, E)] @ X[:, -1]
    assert G.shape == (K.size, K.size) and g.shape == (K.size,)        # sum of 6 / 3 / 6: no inert scalar
    assert np.abs(G - Gk).max() <= 1e-7*np.abs(Gk).max()
    assert np.abs(g - gk).max() <= 1e-6*max(np.abs(gk).max(), 1e-12)
    f_ref = sum_b2 - gd[E] @ X[:, -1]
    assert abs(f - f_ref) <= 1e-8*sum_b2, (f, f_ref, sum_b2)
    return G, g, f


@pytest.mark.parametrize("k", [1, 3])
def test_typed_marginal_equals_the_dense_schur_complement(k):
    rng = np.random.default_rng(5 + k)
    p = _vio(seed=7, n_objects=1)
    assert (p.pose_order >= 0).all() and len(p.blocks) and p.n_vel and p.n_bias
    kinds, idx = _last_frames(p, k)
    assert (kinds == POSE6).sum() > k                                   # an object motion among the kept poses
    perm = rng.permutation(kinds.size)
    kinds, idx = kinds[perm], idx[perm]
    s = Solver(p)
    _check_marginal(p, s, kinds, idx)                                   # at the initial values (g != 0)
    s.optimize()
    _check_marginal(p, s, kinds, idx)                                   # at the optimum, where the reference takes it
    with pytest.raises(DynobaError) as ei:                              # not the most recent variables
        s.marginal_vars(np.array([POSE6, VEL3]), np.array([0, 0]))
    assert ei.value.status == ERR_UNSUPPORTED


def _frames_of(p, b):
    """[n, slots] frame of every pose-like slot of block b (-1 for landmarks)"""
    order = {0: p.pose_order, 3: p.vel_order, 4: p.bias_order}
    return np.stack([order[c][b.idx[:, s]] if c in order else np.full(b.n, -1) for s, c in enumerate(SLOT_CLASS[b.type])], 1)


def _subproblem(p, blocks, keep):
    """the variables of classes 0 (pose), 1 (point), 3 (velocity), 4 (bias) kept by the masks keep[class], re-indexed"""
    new = {c: np.cumsum(m) - 1 for c, m in keep.items()}
    out = []
    for b in blocks:
        idx = b.idx.copy()
        for s_, c in enumerate(SLOT_CLASS[b.type]):
            idx[:, s_] = new[c][idx[:, s_]]
        out.append(FactorBlock(b.type, idx, b.meas, b.sigma, b.robust_k, b.aux_idx))
    return Problem(p.pose[keep[0]], p.point[keep[1]], calib=p.calib, blocks=out, pose_order=p.pose_order[keep[0]],
                   vel=p.vel[keep[3]], bias=p.bias[keep[4]], vel_order=p.vel_order[keep[3]], bias_order=p.bias_order[keep[4]])


def test_two_windows_with_typed_marginal_prior_equal_the_joint_solve():
    """Marginalisation consistency with the IMU chain across the cut.  Window A: the factors of the landmarks last seen
    before f_cut and every factor without a landmark (IMU, priors) whose frames all lie before f_cut -- so the IMU factors
    inside the kept frames constrain their velocities and biases.  Window B: the rest, which starts with the
    COMBINED_IMU15 from frame f_cut - 1 to f_cut.  Kept block: X, V, b of frames [f_cut - k, f_cut).  The Gauss-Newton step
    of window B plus the typed marginal prior of A (linearised at the current values) equals the joint step on B's
    variables."""
    p = synth.make_problem(n_frames=40, n_objects=0, n_static=1000, n_dynamic=0, seed=12, max_static_age=3, imu=True)
    f_cut, k = 20, 4                                                    # k >= max track age: no landmark of B reaches behind the kept block
    last = np.full(p.n_point, -1)
    for b in p.blocks:
        cls = SLOT_CLASS[b.type]
        if 1 in cls:
            np.maximum.at(last, b.idx[:, cls.index(1)], _frames_of(p, b).max(1))
    in_a_pt = last < f_cut
    A, B = [], []
    for b in p.blocks:
        cls = SLOT_CLASS[b.type]
        sel = in_a_pt[b.idx[:, cls.index(1)]] if 1 in cls else _frames_of(p, b).max(1) < f_cut
        for dst, m in ((A, sel), (B, ~sel)):
            if m.any():
                dst.append(FactorBlock(b.type, b.idx[m], None if b.meas is None else b.meas[m], b.sigma if b.sigma_bcast else b.sigma[m],
                                       b.robust_k, None if b.aux_idx is None else b.aux_idx[m]))
    assert any(b.type == 13 for b in B) and any(b.type == 13 for b in A)
    in_a = {0: p.pose_order < f_cut, 1: in_a_pt, 3: p.vel_order < f_cut, 4: p.bias_order < f_cut}
    in_b = {0: p.pose_order >= f_cut - k, 1: ~in_a_pt, 3: p.vel_order >= f_cut - k, 4: p.bias_order >= f_cut - k}
    pa, pb = _subproblem(p, A, in_a), _subproblem(p, B, in_b)
    assert pa.n_factors + pb.n_factors == p.n_factors
    pa.meta = dict(n_frames=f_cut)
    kinds, idx_a = _last_frames(pa, k)
    sa = Solver(pa)
    G, g, _ = sa.marginal_vars(kinds, idx_a)
    sa.close()
    # the same variables in window B: its first k frames, kind by kind in the same order
    first = {POSE6: np.flatnonzero(pb.pose_order < f_cut), VEL3: np.flatnonzero(pb.vel_order < f_cut), BIAS6: np.flatnonzero(pb.bias_order < f_cut)}
    idx_b = np.concatenate([first[kk] for kk in (POSE6, VEL3, BIAS6)]).astype(np.int32)
    assert np.array_equal(kinds, np.repeat([POSE6, VEL3, BIAS6], [first[kk].size for kk in (POSE6, VEL3, BIAS6)]))
    lin = np.concatenate([_value(pb, kk, i) for kk, i in zip(kinds, idx_b)])
    assert np.array_equal(lin, np.concatenate([_value(pa, kk, i) for kk, i in zip(kinds, idx_a)]))
    pb2 = dataclasses.replace(pb, linear_priors=[dict(kind=kinds, idx=idx_b, lin=lin, G=G, g=g, f=0.0)])
    lam = 1e-9
    sj = Solver(p); dj = sj.solve(lam); sj.close()
    sb = Solver(pb2); db = sb.solve(lam); sb.close()
    o = np.cumsum([0, 6*p.n_pose, 3*p.n_point, 2*p.n_flow, 3*p.n_vel, 6*p.n_bias])
    ref = np.concatenate([dj[o[0]:o[1]].reshape(-1, 6)[in_b[0]].ravel(), dj[o[1]:o[2]].reshape(-1, 3)[in_b[1]].ravel(),
                          dj[o[3]:o[4]].reshape(-1, 3)[in_b[3]].ravel(), dj[o[4]:o[5]].reshape(-1, 6)[in_b[4]].ravel()])
    assert np.linalg.norm(db - ref) <= 1e-5*np.linalg.norm(ref), np.linalg.norm(db - ref)/np.linalg.norm(ref)


def test_covariance_with_typed_prior():
    rng = np.random.default_rng(9)
    p = _vio(seed=13, n_objects=1)
    kinds, idx = _last_frames(p, 2)
    pr = _random_prior(rng, p, kinds, idx)
    s = Solver(dataclasses.replace(p, linear_priors=[pr]))
    s.linearize()
    H, _, base = _dense_system(p, s, 0.0)                               # the prior adds G; its g does not enter H
    cols = _cols(base, pr["kind"], pr["idx"])
    H[np.ix_(cols, cols)] += pr["G"]
    pcols = np.concatenate([np.arange(base[0], base[1]), np.arange(base[3], base[5])])
    for kind in (POSE6, VEL3, BIAS6):
        n = {POSE6: p.n_pose, VEL3: p.n_vel, BIAS6: p.n_bias}[kind]; d = TANGENT_DIM[kind]
        C = s.marginal_covariance(kind)
        blocks = base[KIND_CLASS[kind]] + d*np.arange(n)[:, None] + np.arange(d)[None, :]
        ref, kappa = SI.schur_inverse_blocks(H, pcols, blocks)
        assert SI.cov_error(C, ref) <= 40.0*kappa*np.finfo(float).eps, (kind, SI.cov_error(C, ref), kappa)


def _expect(status, fn, *a):
    with pytest.raises(DynobaError) as e:
        fn(*a)
    assert e.value.status == status, e.value


def test_argument_checks():
    p = _vio(n_objects=0, n_dynamic=0)
    s = Solver(p)
    v = p.n_vel - 1
    G6, G3 = np.eye(6), np.eye(3)
    _expect(ERR_BAD_ARG, s.add_linear_prior_vars, [7], [0], np.zeros(6), G6, np.zeros(6))                       # bad kind
    _expect(ERR_BAD_ARG, s.add_linear_prior_vars, [VEL3, VEL3], [v, v], np.zeros(6), np.eye(6), np.zeros(6))   # listed twice
    _expect(ERR_BAD_ARG, s.add_linear_prior_vars, [VEL3], [v], np.zeros(6), G3, np.zeros(3))                  # lin size
    _expect(ERR_BAD_ARG, s.add_linear_prior_vars, [BIAS6], [0], np.zeros(6), G3, np.zeros(3))                 # G size
    A = np.eye(9); A[0, 7] = 0.5
    _expect(ERR_BAD_ARG, s.add_linear_prior_vars, [BIAS6, VEL3], [0, v], np.zeros(9), A, np.zeros(9))          # asymmetric
    _expect(ERR_BAD_ARG, s.marginal_vars, [2], [0])                                                            # bad kind
    _expect(ERR_BAD_ARG, s.marginal_vars, [VEL3, VEL3], [v, v])                                                # listed twice
    # a valid typed prior is taken on this graph, and the handle still solves it; shard and reduce stay refused
    s.add_linear_prior_vars([VEL3, BIAS6], [v, p.n_bias - 1], np.concatenate([p.vel[v], p.bias[-1]]), np.eye(9), np.zeros(9))
    s.optimize(max_iterations=2)
    _expect(ERR_UNSUPPORTED, s.set_shard, 0, 2, lambda *a: None)
    _expect(ERR_UNSUPPORTED, s.set_reduce, lambda *a: None)
    # a velocity index out of range: refused when the graph is built
    t = Solver(p)
    t.add_linear_prior_vars([VEL3], [p.n_vel], np.zeros(3), G3, np.zeros(3))
    _expect(ERR_BAD_ARG, t.finalize)
