"""dynoba_joint_marginal_covariance (csrc/kernels_cov.cu: the band sweeps; csrc/kernels_chain.cu: the landmark strips)
against dense fp64 inverses, against dynoba_marginal_covariance on the same handle, and through its state machine.

Errors are in units of sqrt(Sigma_aa Sigma_bb) of the reference (selinv_reference.cov_error), the tolerance that of
test_covariance_gpu.py: 40 kappa eps, kappa = kappa(D^-1/2 S D^-1/2) of the graph's reduced system; C2's last three
pose-like variables against the inverse of dynoba_marginal's G within TOL_C2.
"""
import dataclasses

import numpy as np
import pytest

import selinv_reference as SI
from dynosam_b200.binding import (BIAS6, ERR_BAD_ARG, ERR_INDETERMINATE, FLOW2, POINT3, POSE6, VEL3, DynobaError,
                                  Solver)
from dynosam_b200.problem import CLASS_DIM, SLOT_CLASS
from test_covariance_gpu import TOL_C2, TOL_GRAPH_KAPPA, _information

pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps
CLS = {POSE6: 0, POINT3: 1, FLOW2: 2, VEL3: 3, BIAS6: 4}


def _touched(p, cls):
    """indices of variables of class cls that some factor touches, in first-seen order"""
    seen = []
    for b in p.blocks:
        for k, c in enumerate(SLOT_CLASS[b.type]):
            if c == cls:
                seen.extend(int(v) for v in b.idx[:, k])
    return list(dict.fromkeys(seen))


def _keys(p):
    """(kinds, idx): a key set that mixes every kind the graph has -- the first and last pose (beyond the band) and two
    neighbours, two points sharing a pose and two far apart, two points of one chain, a flow, X / V / b of one frame"""
    keys = [(POSE6, 0), (POSE6, 1), (POSE6, p.n_pose - 1), (POSE6, p.n_pose // 2)]
    pts = _touched(p, 1)
    for b in p.blocks:        # two points seen from one pose
        cl = SLOT_CLASS[b.type]
        if 1 in cl and 0 in cl:
            kp, kl = cl.index(0), cl.index(1)
            same = np.flatnonzero(b.idx[:, kp] == b.idx[0, kp])
            other = [int(b.idx[i, kl]) for i in same if b.idx[i, kl] != b.idx[0, kl]]
            if other:
                keys += [(POINT3, int(b.idx[0, kl])), (POINT3, other[0])]
                break
    if pts:
        keys += [(POINT3, pts[-1]), (POINT3, pts[len(pts) // 2])]
    for b in p.blocks:        # two points of one chain
        cl = SLOT_CLASS[b.type]
        if cl.count(1) == 2:
            keys += [(POINT3, int(b.idx[0, 0])), (POINT3, int(b.idx[0, 1]))]
            break
    fl = _touched(p, 2)
    if fl:
        keys += [(FLOW2, fl[0]), (FLOW2, fl[-1])]
    if p.n_vel:
        k = min(p.n_vel, p.n_bias, p.n_pose) // 2
        keys += [(VEL3, k), (BIAS6, k), (VEL3, 0)]
        if (POSE6, k) not in keys:
            keys.append((POSE6, k))
    keys = list(dict.fromkeys(keys))
    return np.array([k for k, _ in keys], np.int32), np.array([i for _, i in keys], np.int32)


def _tol(p):
    """40 kappa eps of the graph's reduced system"""
    s = Solver(p)
    s.linearize()
    H, _, base = _information(p, s)
    s.close()
    pcols = np.concatenate([np.arange(base[0], base[1]), np.arange(base[3], base[5])])
    return TOL_GRAPH_KAPPA*SI.schur_inverse_blocks(H, pcols, [])[1]*EPS


def _reference(p, s, kinds, idx):
    H, counts, base = _information(p, s)
    pcols = np.concatenate([np.arange(base[0], base[1]), np.arange(base[3], base[5])])
    _, kappa = SI.schur_inverse_blocks(H, pcols, [])
    Hi = SI.equilibrated_inverse(H.toarray())
    cols = np.concatenate([base[CLS[k]] + CLASS_DIM[CLS[k]]*i + np.arange(CLASS_DIM[CLS[k]]) for k, i in zip(kinds, idx)])
    return Hi[np.ix_(cols, cols)], kappa


@pytest.mark.parametrize("name", list(SI.cov_graphs()))
def test_graph_joint_covariance(name):
    p = SI.cov_graphs()[name]()
    s = Solver(p)
    kinds, idx = _keys(p)
    C, off = s.joint_marginal_covariance(kinds, idx)
    assert np.array_equal(C, C.T)
    s.linearize()
    ref, kappa = _reference(p, s, kinds, idx)
    tol = TOL_GRAPH_KAPPA*kappa*EPS
    err = SI.cov_error(C, ref)
    print(f"JOINT {name}: {err:.2e} = {err/(kappa*EPS):.2f} kappa eps, kappa {kappa:.2e}, D {C.shape[0]}, "
          f"kinds {sorted(set(kinds.tolist()))}")
    assert err <= tol, (err, kappa)
    # the diagonal blocks against dynoba_marginal_covariance of the same handle (the selected inversion's route)
    for k, i, o in zip(kinds, idx, off):
        d = CLASS_DIM[CLS[int(k)]]
        m = s.marginal_covariance(int(k), [int(i)])[0]
        e = SI.cov_error(C[o:o + d, o:o + d], m)
        assert e <= tol, (int(k), int(i), e)
    # a one-variable joint call equals the marginal
    for k, i in zip(kinds[:3], idx[:3]):
        one, _ = s.joint_marginal_covariance([k], [i])
        assert SI.cov_error(one, s.marginal_covariance(int(k), [int(i)])[0]) <= tol
    s.close()


def test_c2_last_pose_likes_match_marginal_information():
    """C2 at full size: the joint covariance of the last three pose-like variables in solver order, off-diagonal blocks
    included, is the inverse of dynoba_marginal's G"""
    from dynosam_b200 import synth
    p = synth.make_config("C2", formulation="hybrid")
    s = Solver(p)
    order = p.pose_order if p.pose_order is not None else np.arange(p.n_pose)
    keep = np.argsort(order, kind="stable")[-3:]
    G, _ = s.marginal(keep)
    C, _ = s.joint_marginal_covariance(np.full(3, POSE6, np.int32), keep)
    err = SI.cov_error(C, np.linalg.inv(G))
    print(f"JOINTC2 last 3 poses: {err:.2e}")
    assert err <= TOL_C2, err
    s.close()


def test_independent_of_partition():
    p = SI.cov_graphs()["hybrid"]()
    kinds, idx = _keys(p)
    got = []
    for cells in (-1, 1, 2, 4):
        s = Solver(p)
        s.set_partition(cells)
        got.append(s.joint_marginal_covariance(kinds, idx)[0])
        s.close()
    tol = _tol(p)
    for C in got[1:]:
        assert SI.cov_error(C, got[0]) <= tol


def _stats(st):
    return {k: st[k] for k in ("iterations", "inner_iterations", "error_initial", "error_final", "lambda_final")}


def test_optimize_after_joint_is_unchanged():
    p = SI.cov_graphs()["hybrid"]()
    kinds, idx = _keys(p)
    runs = []
    for with_cov in (False, False, True):
        s = Solver(p)
        if with_cov:
            s.joint_marginal_covariance(kinds, idx)
        st = s.optimize()
        runs.append((_stats(st), s.values()))
        s.close()
    (st0, v0), (st1, v1), (st2, v2) = runs
    assert st0 == st1 and all(np.array_equal(a, b) for a, b in zip(v0, v1)), "optimize is not repeatable"
    assert st2 == st0, (st2, st0)
    assert all(np.array_equal(a, b) for a, b in zip(v2, v0))


def test_call_orders_match_fresh_handles():
    """marginal -> joint -> marginal, joint -> marginal, and a retract between two calls all give what fresh handles give"""
    p = SI.cov_graphs()["wcme"]()
    kinds, idx = _keys(p)
    f = Solver(p)
    J = f.joint_marginal_covariance(kinds, idx)[0]
    f.close()
    f = Solver(p)
    Mp, Ml = f.marginal_covariance(POSE6), f.marginal_covariance(POINT3)
    f.close()
    tol = _tol(p)
    s = Solver(p)
    assert SI.cov_error(s.marginal_covariance(POSE6), Mp) <= tol
    assert SI.cov_error(s.joint_marginal_covariance(kinds, idx)[0], J) <= tol
    assert SI.cov_error(s.marginal_covariance(POSE6), Mp) <= tol
    assert SI.cov_error(s.marginal_covariance(POINT3), Ml) <= tol
    s.close()
    s = Solver(p)
    assert SI.cov_error(s.joint_marginal_covariance(kinds, idx)[0], J) <= tol
    assert SI.cov_error(s.marginal_covariance(POINT3), Ml) <= tol
    assert SI.cov_error(s.marginal_covariance(POSE6), Mp) <= tol
    # a retract between two calls: the second follows the new values
    rng = np.random.default_rng(4)
    delta = np.concatenate([rng.normal(0, 0.05, 6*p.n_pose), rng.normal(0, 0.2, 3*p.n_point)])
    s.retract(delta)
    J1 = s.joint_marginal_covariance(kinds, idx)[0]
    pose, point, flow = s.values()
    s.close()
    f = Solver(dataclasses.replace(p, pose=pose, point=point, flow=flow))
    Jf = f.joint_marginal_covariance(kinds, idx)[0]
    f.close()
    assert SI.cov_error(J1, Jf) <= tol
    assert SI.cov_error(J, Jf) > 1e-6


def _status(s, kinds, idx, cov=True):
    import ctypes as C
    k = np.ascontiguousarray(kinds, np.int32); i = np.ascontiguousarray(idx, np.int32)
    out = np.zeros(4096)
    cp = out.ctypes.data_as(C.POINTER(C.c_double)) if cov else C.cast(None, C.POINTER(C.c_double))
    return s.lib.dynoba_joint_marginal_covariance(s.h, k.size, k.ctypes.data_as(C.POINTER(C.c_int32)),
                                                 i.ctypes.data_as(C.POINTER(C.c_int32)), cp)


def test_error_statuses():
    p = SI.cov_graphs()["simple"]()
    s = Solver(p)
    s.marginal_covariance(POSE6, [0])          # finalized and holding Sigma: a refusal must leave it usable
    assert _status(s, [], []) == ERR_BAD_ARG
    assert _status(s, [7], [0]) == ERR_BAD_ARG
    assert _status(s, [POSE6], [p.n_pose]) == ERR_BAD_ARG
    assert _status(s, [POINT3], [-1]) == ERR_BAD_ARG
    assert _status(s, [POSE6, POINT3, POSE6], [1, 0, 1]) == ERR_BAD_ARG
    assert _status(s, [POSE6], [0], cov=False) == ERR_BAD_ARG
    assert _status(s, [POSE6], [0]) == 0
    s.close()
    # a landmark no factor touches
    q = dataclasses.replace(p, point=np.concatenate([p.point, [[1.0, 2.0, 3.0]]]))
    s = Solver(q)
    with pytest.raises(DynobaError) as ei:
        s.joint_marginal_covariance([POSE6, POINT3], [0, q.n_point - 1])
    assert ei.value.status == ERR_INDETERMINATE
    s.close()
    # an indefinite reduced system
    import band_reference as BR
    case = BR.CASES["wb3"]
    sysm = BR.build(case)
    neg, _ = BR.negative_prior(sysm, 0)
    s = Solver(sysm.problem([neg]))
    with pytest.raises(DynobaError) as ei:
        s.joint_marginal_covariance([POSE6], [1])
    assert ei.value.status == ERR_INDETERMINATE
    s.close()


def test_singular_group_is_indeterminate():
    """the WCPE graph without unit pose priors: a requested chain's own block is singular"""
    from dynosam_b200 import synth
    import schur_reference as SR
    p = synth.make_problem(n_frames=40, n_objects=1, n_static=300, n_dynamic=200, formulation="wcpe", seed=5,
                           object_span=(40, 40), max_dynamic_age=SR.GG_MAXL)
    s = Solver(p)
    with pytest.raises(DynobaError) as ei:
        s.joint_marginal_covariance([POINT3], [_touched(p, 1)[-1]])
    assert ei.value.status == ERR_INDETERMINATE
    s.close()
