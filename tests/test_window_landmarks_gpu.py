"""The sliding window that keeps the last frames' landmarks: the linearised landmark factors LINEAR_PP3 / LINEAR_PPP3
(gtsam::LinearContainerFactor holding a 3-row JacobianFactor) and dynoba_marginal_keep_points, which hands the kept
points' factors to the next window and takes them out of the Schur marginal.

GTSAM semantics [GTSAM-ext LinearContainerFactor::{error,linearize}], restated in numpy here:
    d = lin.localCoordinates(x)   (Logmap(lin^-1 x) per pose, x - lin for the point)
    error(x) = 1/2 |A d - b|^2,   linearize(x) = JacobianFactor(A, b - A d)
The decisive test is test_two_windows_keep_points_equal_the_joint_solve: a window marginalised with its last frames'
points kept, followed by the next window with the HessianFactor prior and the exported factors, takes the joint graph's
Gauss-Newton step."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
from mpmath import mpf

import factor_cases as FC
import lie_reference as LR
from test_imu_gpu import _dense_system
from dynosam_b200 import synth
from dynosam_b200.binding import (BIAS6, ERR_BAD_ARG, ERR_UNSUPPORTED, FLOW2, POINT3, POSE6, VEL3, DynobaError, Solver,
                                  TANGENT_DIM, _dp, _ip, c_dp, c_ip)
from dynosam_b200.problem import (HYBRID3, LINEAR_PP3, LINEAR_PPP3, POSE2POINT3, PRIOR6, SLOT_CLASS, STEREO3, FactorBlock,
                                  Problem, linear_block)

pytestmark = pytest.mark.gpu
EPS = 2.0**-52


# ---------------------------------------------------------------------------------------------------- 1. the factor kernel
ANGLES = ["0", "1e-5", "0.3", "2.5", "pi-1e-4"]
AXES = [(0, 0, 1), (0.6, 0.8, 0), (1, 1, 1), (-0.6, 0, -0.8)]


def _linear_case(n, seed):
    """one anchor PRIOR6, a LINEAR_PP3 block and a LINEAR_PPP3 block of n factors each; factor f's linearisation point is
    its variables composed with a relative rotation of angle ANGLES[f % 5] (the Logmap branches: identity, Taylor, acos, acos
    near pi) and a translation of 0, 1 or 1e3"""
    rng = np.random.default_rng(seed)
    poses, lins, rels = [], [], []
    for f in range(3*n):                                                # pose slots: PP3 f -> f, PPP3 f -> n + 2f, n + 2f + 1
        x = FC.random_pose(rng, 2.0, 2.0)
        rel = FC.pose12(FC.rotation(ANGLES[f % 5], AXES[f % 4]), rng.normal(size=3)*[0.0, 1.0, 1e3][f % 3])
        lins.append(FC.compose12(x, np.array(LR.to_float(LR.pose_flat(LR.inverse(LR.pose(rel)))))))
        poses.append(x); rels.append(rel)
    pose = np.array(poses).reshape(-1, 12) if n else FC.IDENT[None]
    point = rng.normal(0, 5.0, (2*n, 3)); point[::3] *= 200.0
    lin_pt = point + rng.normal(0, 0.1, point.shape)
    blocks = [FactorBlock(PRIOR6, np.array([[0]]), pose[:1], np.array([1.0]))]
    for t, npose in ((LINEAR_PP3, 1), (LINEAR_PPP3, 2)):
        jc = 6*npose + 3
        pi = np.arange(n)[:, None]*npose + (0 if t == LINEAR_PP3 else n) + np.arange(npose)[None]
        li = np.arange(n) + (0 if t == LINEAR_PP3 else n)
        A = rng.normal(0, 1, (n, 3, jc))*np.where(np.arange(n) % 7 == 0, 1e3, 1.0)[:, None, None]
        b = rng.normal(0, 1, (n, 3))
        blocks.append(linear_block(t, np.concatenate([pi, li[:, None]], 1), A, b, np.array(lins).reshape(-1, 12)[pi] if n else np.zeros((0, npose, 12)), lin_pt[li]))
    return Problem(pose, point, blocks=blocks)


def _reference(p, blk):
    """50-digit b - A d and 1/2 |b - A d|^2 per factor, and the a-priori bound of |b_dev - b_ref| per row: the Logmap
    error (lie_reference.log_rot_bound, scaled by the translations) and the point difference's rounding propagated through
    |A|, plus (jcols + 1) roundings of the dot product"""
    npose = 1 if blk.type == LINEAR_PP3 else 2
    jc = 6*npose + 3
    bref, eref, bound = [], [], []
    for f in range(blk.n):
        m = blk.meas[f]; A = m[:3*jc].reshape(3, jc); b = m[3*jc:3*jc + 3]
        d, derr = [], []
        for s in range(npose):
            lin = m[3*jc + 3 + 12*s:3*jc + 15 + 12*s]; x = p.pose[blk.idx[f, s]]
            d += LR.g_local(LR.pose(lin), LR.pose(x))
            B = float(LR.log_rot_bound(LR.between(LR.pose(lin), LR.pose(x))[0]))
            derr += [EPS*B*(1 + np.abs(x[9:]).max() + np.abs(lin[9:]).max())]*6
        lp = m[3*jc + 3 + 12*npose:]; xp = p.point[blk.idx[f, npose]]
        d += [mpf(float(u)) - mpf(float(v)) for u, v in zip(xp, lp)]
        derr += list(EPS*np.abs(xp - lp))
        r = [mpf(float(b[i])) - sum(mpf(float(A[i, c]))*d[c] for c in range(jc)) for i in range(3)]
        bref.append(LR.to_float(r)); eref.append(float(sum(q*q for q in r)/2))
        df = np.abs(np.array(LR.to_float(d)))
        bound.append(np.abs(A) @ np.array(derr) + (jc + 1)*EPS*(np.abs(b) + np.abs(A) @ df))
    return np.array(bref).reshape(-1, 3), np.array(eref), np.array(bound).reshape(-1, 3)


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 2500])
def test_linear_factor_kernel(n):
    """J = A bit for bit; b - A d and the error within 8 units of the a-priori bound of _reference (a unit: a faithful
    fp64 Logmap of the pose slots and one rounding per product of the dot product, propagated through |A|; 8 units as
    test_factors_gpu.py::test_linear_prior_logmap allows the prior's Logmap)"""
    p = _linear_case(n, seed=n)
    s = Solver(p)
    s.linearize()
    worst_b = worst_e = 0.0
    for bi in (1, 2):
        blk = p.blocks[bi]
        J, b = s.linearization(bi)
        if n == 0:                                                      # an empty block launches nothing
            assert J.shape[0] == b.shape[0] == 0 and s.error() == 0.0
            continue
        e = s.factor_errors(bi)
        jc = J.shape[2]
        assert np.array_equal(J.reshape(n, -1), blk.meas[:, :3*jc])
        bref, eref, bound = _reference(p, blk)
        worst_b = max(worst_b, (np.abs(b - bref)/bound).max())
        ebound = (np.abs(bref)*bound).sum(1) + 4*EPS*eref
        worst_e = max(worst_e, (np.abs(e - eref)/ebound).max())
    print(f"LINEAR H100 n={n}: |b - b_ref| {worst_b:.3g}, |e - e_ref| {worst_e:.3g} (units of the bound)")
    assert worst_b <= 8 and worst_e <= 8
    # the graph error sums the per-factor errors with the anchor prior (zero residual)
    if n:
        tot = sum(s.factor_errors(bi).sum() for bi in (1, 2))
        assert abs(s.error() - tot) <= 1e-12*tot
    s.close()


def test_linear_factor_noise_model_refused():
    p = _linear_case(3, seed=1)
    blk = p.blocks[1]
    for sigma, k in ((np.array([2.0]), 0.0), (np.ones(3)*0.5, 0.0), (np.array([1.0]), 1e-3)):
        s = Solver()
        with pytest.raises(DynobaError) as e:
            s.add_factors(dataclasses.replace(blk, sigma=sigma, robust_k=k))
        assert e.value.status == ERR_BAD_ARG
        s.close()


# ---------------------------------------------------------------------------------------------------- shared algebra
def _local_pose(lin, x):
    """Logmap(lin^-1 x) from the 50-digit reference, rounded once"""
    return np.array(LR.to_float(LR.g_local(LR.pose(lin), LR.pose(x))))


def _linear_d(p, blk):
    """d of every factor of a linear block at p's values, in the block's column order"""
    npose = 1 if blk.type == LINEAR_PP3 else 2
    jc = 6*npose + 3
    out = []
    for f in range(blk.n):
        m = blk.meas[f]
        d = [_local_pose(m[3*jc + 3 + 12*s:3*jc + 15 + 12*s], p.pose[blk.idx[f, s]]) for s in range(npose)]
        d.append(p.point[blk.idx[f, npose]] - m[3*jc + 3 + 12*npose:])
        out.append(np.concatenate(d))
    return np.array(out).reshape(-1, jc)


def _ab(blk):
    jc = 9 if blk.type == LINEAR_PP3 else 15
    return blk.meas[:, :3*jc].reshape(-1, 3, jc), blk.meas[:, 3*jc:3*jc + 3]


# ---------------------------------------------------------------------------------------------------- 2. damped step
def test_damped_step_with_linear_factors():
    """a hybrid graph plus LINEAR_PP3 factors on (camera pose, static point) and LINEAR_PPP3 factors on (camera pose, motion,
    dynamic point) linearised away from the current values (d != 0): the error and the damped step against the oracle's
    dense normal equations plus the numpy LinearContainerFactor algebra"""
    from oracle import oracle as O
    rng = np.random.default_rng(4)
    base = synth.make_config("C1")
    blocks = list(base.blocks)
    for t, src in ((LINEAR_PP3, POSE2POINT3), (LINEAR_PPP3, HYBRID3)):
        sb = next(b for b in base.blocks if b.type == src)
        sel = rng.choice(sb.n, 60, replace=False)
        idx = sb.idx[sel]; npose = 1 if t == LINEAR_PP3 else 2; jc = 6*npose + 3
        lin_pose = np.stack([FC.compose12(base.pose[i], FC.pose12(FC.rotation(mpf(0.02), tuple(rng.normal(size=3))), rng.normal(0, 0.05, 3)))
                             for i in idx[:, :npose].ravel()]).reshape(-1, npose, 12)
        blocks.append(linear_block(t, idx, rng.normal(0, 2.0, (60, 3, jc)), rng.normal(0, 1.0, (60, 3)), lin_pose,
                                   base.point[idx[:, npose]] + rng.normal(0, 0.05, (60, 3))))
    p = dataclasses.replace(base, blocks=blocks)
    s = Solver(p); o = O.OracleProblem(base)
    H, g = o.dense_normal()
    e_lin = 0.0
    for blk in blocks[len(base.blocks):]:
        A, b = _ab(blk); d = _linear_d(p, blk)
        r = b - np.einsum("nij,nj->ni", A, d)
        e_lin += 0.5*float((r*r).sum())
        for f in range(blk.n):
            cols = np.concatenate([6*blk.idx[f, k] + np.arange(6) if c == 0 else 6*p.n_pose + 3*blk.idx[f, k] + np.arange(3)
                                   for k, c in enumerate(SLOT_CLASS[blk.type])])
            H[np.ix_(cols, cols)] += A[f].T @ A[f]; g[cols] += A[f].T @ r[f]
    e_ref = o.error() + e_lin
    assert abs(s.error() - e_ref) <= 1e-9*e_ref
    lam = 1e-3
    ref = np.linalg.solve(H + lam*np.eye(H.shape[0]), g)
    dd = s.solve(lam)
    assert np.linalg.norm(dd - ref) <= 1e-6*np.linalg.norm(ref), np.linalg.norm(dd - ref)/np.linalg.norm(ref)
    st = s.optimize(max_iterations=6)
    assert st["error_final"] < st["error_initial"]
    s.close()


# ---------------------------------------------------------------------------------------------------- window splits
def _frames(p):
    return {0: p.pose_order, 3: p.vel_order, 4: p.bias_order}


def _slot_frames(p, b):
    fr = _frames(p)
    return np.stack([fr[c][b.idx[:, s]] if c in fr else np.full(b.n, -1) for s, c in enumerate(SLOT_CLASS[b.type])], 1)


def _take(b, m):
    return FactorBlock(b.type, b.idx[m], None if b.meas is None else b.meas[m], b.sigma if b.sigma_bcast else b.sigma[m],
                       b.robust_k, None if b.aux_idx is None else b.aux_idx[m])


def _reindex(p, blocks, keep):
    """the variables of p kept by the masks keep[class] (0 pose, 1 point, 3 velocity, 4 bias), blocks re-indexed"""
    new = {c: np.cumsum(m) - 1 for c, m in keep.items()}
    out = []
    for b in blocks:
        idx = b.idx.copy()
        for s_, c in enumerate(SLOT_CLASS[b.type]):
            assert keep[c][idx[:, s_]].all()
            idx[:, s_] = new[c][idx[:, s_]]
        out.append(FactorBlock(b.type, idx, b.meas, b.sigma, b.robust_k, b.aux_idx))
    imu = p.n_vel > 0
    return Problem(p.pose[keep[0]], p.point[keep[1]], aux_pose=p.aux_pose, calib=p.calib, blocks=out,
                   pose_order=p.pose_order[keep[0]], vel=p.vel[keep[3]] if imu else np.zeros((0, 3)),
                   bias=p.bias[keep[4]] if imu else np.zeros((0, 6)), vel_order=p.vel_order[keep[3]] if imu else None,
                   bias_order=p.bias_order[keep[4]] if imu else None)


def _window_split(p, f_cut, k):
    """The reference's split (SlidingWindowOptimization.cc:64-130, isRecentKey): window 1 holds the factors of frames
    < f_cut and keeps every key inserted in frames [f_cut - k, f_cut) -- camera poses, motions, velocities, biases and the
    points first observed there (a point is inserted at its first observation; without backtracking it is observed only
    later).  Tracks are longer than k, so kept points are observed again in window 2.  Observations at frames >= f_cut of
    points inserted before f_cut - k are dropped from the joint graph: the reference's window has no such keys."""
    first = np.full(p.n_point, 1 << 30)
    for b in p.blocks:
        if 1 in SLOT_CLASS[b.type]:
            np.minimum.at(first, b.idx[:, SLOT_CLASS[b.type].index(1)], _slot_frames(p, b).max(1))
    joint, w1, w2 = [], [], []
    for b in p.blocks:
        fr = _slot_frames(p, b).max(1)
        m = np.ones(b.n, bool)
        if 1 in SLOT_CLASS[b.type]:
            m = ~((first[b.idx[:, SLOT_CLASS[b.type].index(1)]] < f_cut - k) & (fr >= f_cut))
        if m.any():
            joint.append(_take(b, m))
    for b in joint:
        fr = _slot_frames(p, b)
        a = fr.max(1) < f_cut
        pos = fr[:, [c in (0, 3, 4) for c in SLOT_CLASS[b.type]]]
        assert (pos[~a] >= f_cut - k).all()                               # window 2 touches no eliminated variable
        if a.any(): w1.append(_take(b, a))
        if (~a).any(): w2.append(_take(b, ~a))
    pj = dataclasses.replace(p, blocks=joint, linear_priors=[])
    fr = _frames(p)
    cls = (0, 3, 4) if p.n_vel else (0,)
    K1 = {c: fr[c] < f_cut for c in cls}; K1[1] = first < f_cut
    K2 = {c: fr[c] >= f_cut - k for c in cls}; K2[1] = (first >= f_cut - k) & (first < (1 << 30))
    if not p.n_vel:
        for c in (3, 4): K1[c] = K2[c] = np.zeros(0, bool)
    return pj, w1, w2, K1, K2, first


def _kept_vars(pa, f_cut, k):
    kinds, idx = [], []
    for kind, order in ((POSE6, pa.pose_order), (VEL3, pa.vel_order), (BIAS6, pa.bias_order)):
        if order is None:
            continue
        sel = np.flatnonzero(order >= f_cut - k)
        kinds += [kind]*sel.size; idx += list(sel)
    return np.array(kinds, np.int32), np.array(idx, np.int32)


def _to_stereo(p, rng):
    """every POSE2POINT3 factor whose point lies well in front of the camera becomes a STEREO3 factor on (uL, uR, v)"""
    from dynosam_b200 import lie
    out = []
    for b in p.blocks:
        if b.type != POSE2POINT3:
            out.append(b); continue
        q = lie.transform_to(p.pose[b.idx[:, 0]], p.point[b.idx[:, 1]])
        m = q[:, 2] > 1.0
        K = p.calib
        z = np.stack([K[3] + K[0]*q[:, 0]/q[:, 2], K[3] + K[0]*(q[:, 0] - K[5])/q[:, 2], K[4] + K[1]*q[:, 1]/q[:, 2]], 1)
        z += rng.normal(0, 0.5, z.shape)
        if m.any():
            out.append(FactorBlock(STEREO3, b.idx[m], z[m], np.array([1.0]), b.robust_k))
        if (~m).any():
            out.append(_take(b, ~m))
    return dataclasses.replace(p, blocks=out)


def _case(name):
    if name == "static":
        return synth.make_problem(n_frames=16, n_objects=0, n_static=400, n_dynamic=0, seed=21, max_static_age=6)
    if name == "stereo":
        p = synth.make_problem(n_frames=16, n_objects=0, n_static=400, n_dynamic=0, seed=22, max_static_age=6)
        return _to_stereo(p, np.random.default_rng(0))
    if name == "hybrid":
        return synth.make_problem(n_frames=16, n_objects=1, n_static=300, n_dynamic=160, seed=23, max_static_age=6,
                                  max_dynamic_age=6)
    return synth.make_problem(n_frames=16, n_objects=0, n_static=400, n_dynamic=0, seed=24, max_static_age=6, imu=True)


def _w1(name, f_cut=10, k=3):
    p = _case(name)
    pj, w1, w2, K1, K2, first = _window_split(p, f_cut, k)
    pa = _reindex(pj, w1, K1)
    kinds, idx = _kept_vars(pa, f_cut, k)
    pts = np.flatnonzero((first[K1[1]] >= f_cut - k)).astype(np.int32)
    return p, pj, w1, w2, K1, K2, first, pa, kinds, idx, pts


def _drop_points(pa, pts):
    """pa without the points pts and their factors (every other index unchanged but the points')"""
    keep_pt = np.ones(pa.n_point, bool); keep_pt[pts] = False
    blocks = []
    for b in pa.blocks:
        if 1 in SLOT_CLASS[b.type]:
            m = keep_pt[b.idx[:, SLOT_CLASS[b.type].index(1)]]
            if m.any(): blocks.append(_take(b, m))
        else:
            blocks.append(b)
    keep = {0: np.ones(pa.n_pose, bool), 1: keep_pt, 3: np.ones(pa.n_vel, bool), 4: np.ones(pa.n_bias, bool)}
    return _reindex(pa, blocks, keep)


def _cols(base, kinds, idx):
    kc = {POSE6: 0, VEL3: 3, BIAS6: 4}
    return np.concatenate([base[kc[k]] + TANGENT_DIM[k]*i + np.arange(TANGENT_DIM[k]) for k, i in zip(kinds, idx)])


# ---------------------------------------------------------------------------------------------------- 3. exclusion
@pytest.mark.parametrize("name", ["hybrid", "imu"])
def test_keep_points_excludes_their_factors(name):
    """(G, g, f) of marginal_keep_points = marginal_vars of the graph without the kept points and their factors, and
    = the dense Schur complement of that graph; the exported A / b = the rows of dynoba_get_linearization"""
    _, _, _, _, _, _, _, pa, kinds, idx, pts = _w1(name)
    assert pts.size > 20
    s = Solver(pa)
    G, g, f, blocks = s.marginal_keep_points(kinds, idx, pts)
    q = _drop_points(pa, pts)
    sq = Solver(q)
    Gq, gq, fq = sq.marginal_vars(kinds, idx)
    sq.linearize()
    H, gd, base = _dense_system(q, sq, 0.0)
    sum_b2 = sum(float(np.sum(sq.linearization(bi)[1]**2)) for bi in range(len(q.blocks)))
    Kc = _cols(base, kinds, idx); E = np.setdiff1d(np.arange(H.shape[0]), Kc)
    X = np.linalg.solve(H[np.ix_(E, E)], np.concatenate([H[np.ix_(E, Kc)], gd[E, None]], 1))
    Gk = H[np.ix_(Kc, Kc)] - H[np.ix_(Kc, E)] @ X[:, :-1]; gk = gd[Kc] - H[np.ix_(Kc, E)] @ X[:, -1]
    fk = sum_b2 - gd[E] @ X[:, -1]
    assert np.abs(G - Gq).max() <= 1e-9*np.abs(Gq).max() and np.abs(g - gq).max() <= 1e-9*np.abs(gq).max()
    assert abs(f - fq) <= 1e-8*sum_b2, (f, fq, sum_b2)
    assert np.abs(G - Gk).max() <= 1e-7*np.abs(Gk).max() and np.abs(g - gk).max() <= 1e-6*np.abs(gk).max()
    assert abs(f - fk) <= 1e-8*sum_b2, (f, fk, sum_b2)
    # the exported factors: every factor of a kept point, block by block in caller order, A and b bit for bit
    s.linearize()
    kept = np.zeros(pa.n_point, bool); kept[pts] = True
    want_A, want_b, want_idx, want_t = [], [], [], []
    for bi, b in enumerate(pa.blocks):
        if 1 not in SLOT_CLASS[b.type]:
            continue
        m = kept[b.idx[:, SLOT_CLASS[b.type].index(1)]]
        if m.any():
            A, bb = s.linearization(bi)
            want_A += list(A[m]); want_b += list(bb[m]); want_idx += list(b.idx[m])
            want_t += [LINEAR_PP3 if SLOT_CLASS[b.type] == [0, 1] else LINEAR_PPP3]*int(m.sum())
    got = [(blk.type, i, *(x[j] for x in _ab(blk))) for blk in blocks for j, i in enumerate(blk.idx)]
    assert len(got) == len(want_t)
    pose, point, _ = s.values()
    for (t, i, A, bb), wt, wi, wa, wb in zip(got, want_t, want_idx, want_A, want_b):
        assert t == wt and np.array_equal(i, wi) and np.array_equal(A, wa) and np.array_equal(bb, wb)
    for blk in blocks:                                                  # linearisation point: the current values
        npose = 1 if blk.type == LINEAR_PP3 else 2; jc = 6*npose + 3
        assert np.array_equal(blk.meas[:, 3*jc + 3:3*jc + 3 + 12*npose].reshape(-1, npose, 12), pose[blk.idx[:, :npose]])
        assert np.array_equal(blk.meas[:, 3*jc + 3 + 12*npose:], point[blk.idx[:, npose]])
    s.close(); sq.close()


# ---------------------------------------------------------------------------------------------------- 4. two windows
@pytest.mark.parametrize("name", ["static", "stereo", "hybrid", "imu"])
def test_two_windows_keep_points_equal_the_joint_solve(name):
    f_cut, k = 10, 3
    p, pj, w1, w2, K1, K2, first, pa, kinds, idx, pts = _w1(name, f_cut, k)
    sa = Solver(pa)
    G, g, f, blocks = sa.marginal_keep_points(kinds, idx, pts)
    sa.close()
    assert sum(b.n for b in blocks) > 0
    if name == "stereo":
        assert any(b.type == STEREO3 for b in pa.blocks)
    if name == "hybrid":
        assert {b.type for b in blocks} == {LINEAR_PP3, LINEAR_PPP3}
    # exported factors in joint indices, then window 2's
    w1_of = {c: np.flatnonzero(m) for c, m in K1.items()}
    lin2 = []
    for b in blocks:
        jidx = b.idx.copy()
        for s_, c in enumerate(SLOT_CLASS[b.type]):
            jidx[:, s_] = w1_of[c][b.idx[:, s_]]
        lin2.append(FactorBlock(b.type, jidx, b.meas, b.sigma))
    pb = _reindex(pj, w2 + lin2, K2)
    pb_new = _reindex(pj, w2, K2)
    # some kept points are observed again in window 2
    kept_joint = w1_of[1][pts]
    seen2 = np.concatenate([b.idx[:, SLOT_CLASS[b.type].index(1)] for b in w2 if 1 in SLOT_CLASS[b.type]])
    assert np.isin(kept_joint, seen2).sum() > 5
    # the kept variables in window 2: same variables, same order
    w2_new = {c: np.cumsum(m) - 1 for c, m in K2.items()}
    kc = {POSE6: 0, VEL3: 3, BIAS6: 4}
    idx_b = np.array([w2_new[kc[kk]][w1_of[kc[kk]][i]] for kk, i in zip(kinds, idx)], np.int32)
    lin = np.concatenate([(pb.pose, None, None, pb.vel, pb.bias)[kc[kk]][i] for kk, i in zip(kinds, idx_b)])
    pb2 = dataclasses.replace(pb, linear_priors=[dict(kind=kinds, idx=idx_b, lin=lin, G=G, g=g, f=f)])
    lam = 1e-9
    sj = Solver(pj); dj = sj.solve(lam); sj.close()
    sb = Solver(pb2); db = sb.solve(lam)
    o = np.cumsum([0, 6*p.n_pose, 3*p.n_point, 0, 3*p.n_vel, 6*p.n_bias])
    parts = [dj[o[0]:o[1]].reshape(-1, 6)[K2[0]].ravel(), dj[o[1]:o[2]].reshape(-1, 3)[K2[1]].ravel()]
    if p.n_vel:
        parts += [dj[o[3]:o[4]].reshape(-1, 3)[K2[3]].ravel(), dj[o[4]:o[5]].reshape(-1, 6)[K2[4]].ravel()]
    ref = np.concatenate(parts)
    rel = np.linalg.norm(db - ref)/np.linalg.norm(ref)
    print(f"WINDOW H100 {name}: {sum(b.n for b in blocks)} exported factors, step relative difference {rel:.3g}")
    assert rel <= 1e-5, rel
    # window 2's error at d = 0: its new factors, 1/2 f of the prior and 1/2 |b|^2 of the exported factors
    sn = Solver(pb_new)
    e_ref = sn.error() + 0.5*f + 0.5*sum(float((_ab(b)[1]**2).sum()) for b in lin2)
    sn.close()
    assert abs(sb.error() - e_ref) <= 1e-10*e_ref
    sb.close()


# ---------------------------------------------------------------------------------------------------- 5. state, refusals
def _spread(a, b):
    return max(np.abs(a - b).max()/max(np.abs(a).max(), 1e-300), 0.0)


def test_state_refusals_and_a_third_window():
    p, pj, w1, w2, K1, K2, first, pa, kinds, idx, pts = _w1("hybrid")
    s = Solver(pa)
    G0, g0, f0 = s.marginal_vars(kinds, idx)
    G1, g1, f1 = s.marginal_vars(kinds, idx)
    Gz, gz, fz, bz = s.marginal_keep_points(kinds, idx, [])
    assert bz == []
    if np.array_equal(G0, G1) and np.array_equal(g0, g1) and f0 == f1:  # two calls agree bit for bit: so does n_pts = 0
        assert np.array_equal(Gz, G0) and np.array_equal(gz, g0) and fz == f0
    else:                                                               # the band's fp64 atomics flush in varying order
        assert _spread(G0, Gz) <= 2*_spread(G0, G1) + 1e-15 and _spread(g0, gz) <= 2*_spread(g0, g1) + 1e-15

    def expect(status, *a, **kw):
        with pytest.raises(DynobaError) as e:
            s.marginal_keep_points(*a, **kw)
        assert e.value.status == status, e.value
    old = np.flatnonzero(first[K1[1]] < 10 - 3 - 1)[:1].astype(np.int32)   # inserted before the kept frames: backtracking
    expect(ERR_UNSUPPORTED, kinds, idx, np.concatenate([pts[:3], old]))
    expect(ERR_BAD_ARG, kinds, idx, np.concatenate([pts[:3], pts[:1]]))       # listed twice
    expect(ERR_BAD_ARG, kinds, idx, np.array([pa.n_point], np.int32))         # out of range
    expect(ERR_BAD_ARG, kinds, idx, pts[:2], pt_kinds=[POINT3, FLOW2])         # a flow variable
    # capacity below the number of exported factors: BAD_ARG, and n_out still counts them
    n = C.c_int64(); Gb = np.zeros_like(G0); gb = np.zeros_like(g0); fb = C.c_double()
    typ = np.zeros(1, np.int32); vid = np.zeros(3, np.int32); Ab = np.zeros(48)
    st = s.lib.dynoba_marginal_keep_points(s.h, kinds.size, _ip(kinds), _ip(idx), pts.size, C.cast(None, c_ip), _ip(pts),
                                           _dp(Gb), _dp(gb), C.byref(fb), 1, C.byref(n), _ip(typ), _ip(vid), _dp(Ab))
    assert st == ERR_BAD_ARG and n.value > 1
    # a successful call in between: the handle optimises as a fresh one
    s.marginal_keep_points(kinds, idx, pts)
    r = [Solver(pa).optimize(max_iterations=5) for _ in range(2)]
    st_s = s.optimize(max_iterations=5)
    es = abs(r[0]["error_final"] - r[1]["error_final"])/r[0]["error_final"]
    assert st_s["iterations"] == r[0]["iterations"]
    assert abs(st_s["error_final"] - r[0]["error_final"])/r[0]["error_final"] <= max(2*es, 1e-10)
    s.close()
    # a WCME graph: a kept point chained to others by LandmarkMotionTernaryFactor
    w = synth.make_problem(n_frames=12, n_objects=1, n_static=100, n_dynamic=60, seed=5, formulation="wcme")
    sw = Solver(w)
    t = next(b for b in w.blocks if b.type == 4)
    kw_, iw = np.array([POSE6], np.int32), np.array([int(np.argmax(w.pose_order))], np.int32)
    with pytest.raises(DynobaError) as e:
        sw.marginal_keep_points(kw_, iw, t.idx[:1, 0])
    assert e.value.status == ERR_UNSUPPORTED
    sw.close()


def test_third_window_eliminates_the_kept_points():
    """window 2 -- new factors, the prior and window 1's exported factors -- is itself marginalised keeping its own last
    frames' points: window 1's kept points are eliminated with their linear factors (a landmark whose factors span two
    blocks takes the general path), and the marginal equals the dense Schur complement of window 2"""
    f_cut, k = 10, 3
    p, pj, w1, w2, K1, K2, first, pa, kinds, idx, pts = _w1("hybrid", f_cut, k)
    sa = Solver(pa)
    G, g, f, blocks = sa.marginal_keep_points(kinds, idx, pts)
    sa.close()
    w1_of = {c: np.flatnonzero(m) for c, m in K1.items()}
    lin2 = []
    for b in blocks:
        jidx = b.idx.copy()
        for s_, c in enumerate(SLOT_CLASS[b.type]):
            jidx[:, s_] = w1_of[c][b.idx[:, s_]]
        lin2.append(FactorBlock(b.type, jidx, b.meas, b.sigma))
    pb = _reindex(pj, w2 + lin2, K2)
    w2_new = np.cumsum(K2[0]) - 1
    idx_b = w2_new[w1_of[0][idx]].astype(np.int32)
    pb = dataclasses.replace(pb, linear_priors=[dict(kind=kinds, idx=idx_b, lin=pb.pose[idx_b].ravel(), G=G, g=g, f=f)])
    f2 = int(pb.pose_order.max()) + 1
    kinds2, idx2 = _kept_vars(pb, f2, k)
    first2 = first[K2[1]]
    pts2 = np.flatnonzero(first2 >= f2 - k).astype(np.int32)
    sb = Solver(pb)
    sb.optimize(max_iterations=3)
    G2, g2, f2v, blocks2 = sb.marginal_keep_points(kinds2, idx2, pts2)
    assert sum(b.n for b in blocks2) > 0
    # against the dense Schur complement of window 2 without its kept points' factors (the prior added by hand)
    q = _drop_points(dataclasses.replace(pb, pose=sb.values()[0], point=sb.values()[1], linear_priors=[]), pts2)
    sq = Solver(q); sq.linearize()
    H, gd, base = _dense_system(q, sq, 0.0)
    pr = pb.linear_priors[0]
    from test_sliding_window import _local
    d0 = _local(pr["lin"].reshape(-1, 12), q.pose[pr["idx"]])
    c = _cols(base, pr["kind"], pr["idx"])
    H[np.ix_(c, c)] += pr["G"]; gd[c] += pr["g"] - pr["G"] @ d0
    Kc = _cols(base, kinds2, idx2); E = np.setdiff1d(np.arange(H.shape[0]), Kc)
    X = np.linalg.solve(H[np.ix_(E, E)], np.concatenate([H[np.ix_(E, Kc)], gd[E, None]], 1))
    Gk = H[np.ix_(Kc, Kc)] - H[np.ix_(Kc, E)] @ X[:, :-1]; gk = gd[Kc] - H[np.ix_(Kc, E)] @ X[:, -1]
    assert np.abs(G2 - Gk).max() <= 1e-7*np.abs(Gk).max() and np.abs(g2 - gk).max() <= 1e-6*np.abs(gk).max()
    sb.close(); sq.close()
