"""dynoba_marginal_covariance (csrc/kernels_cov.cu: band selected inversion, pose-like gather, landmark kernels) against
dense fp64 inverses.  Errors are in units of sqrt(Sigma_aa Sigma_bb) of the reference (selinv_reference.cov_error).

Band level: the pose blocks of S^-1 on band_reference's systems (dense priors only, so H = S), inverted equilibrated.
Full graphs: every variable of every kind against H^-1, H = J^T J from the device's own Jacobians (Solver.linearization,
as schur_reference.Reference builds it; the blocks through the Schur-complement identity, selinv_reference), and the
pose blocks against oracle.dense_normal()'s inverse as well.

Tolerances, from the worst values measured on an H100 80GB HBM3 at 700 W:

    band family          worst / tolerance
    dominant, graded     5.7e-15 (wb35) / 1e-13
    nearsing             2.2e-7 (nearsing_wb3) / 3e-6
    laplacian            9.8e-8 (laplacian_kend15) / 2e-6
    full graphs          err / (kappa eps) <= 1.3 (wcme: 6.3e-10 at kappa 2.2e6) / 40 kappa eps, kappa = kappa(D^-1/2 S D^-1/2)
                         of the graph's reduced system: the error of a backward-stable inverse, the reference's included
    C2 last poses        1.2e-6 / 1e-5 (against the inverse of dynoba_marginal's G; two runs gave 1.0e-6 and 1.2e-6)

Partitions of the handle do not change a bit of the result: the covariances always come from the plain layout.
"""
import dataclasses

import numpy as np
import pytest
import scipy.sparse as sp

import band_reference as BR
import selinv_reference as SI
from dynosam_b200.binding import BIAS6, ERR_INDETERMINATE, FLOW2, POINT3, POSE6, VEL3, DynobaError, Solver
from dynosam_b200.problem import CLASS_DIM, SLOT_CLASS

pytestmark = pytest.mark.gpu

TOL_BAND = {"dominant": 1e-13, "graded": 1e-13, "nearsing": 3e-6, "laplacian": 2e-6}
TOL_GRAPH_KAPPA = 40.0    # x kappa eps
TOL_C2 = 1e-5
ORACLE_MAX_DIM = 6000     # dense oracle inverse only on graphs this small

_cache = {}


def _system(case):
    if case.name not in _cache:
        _cache[case.name] = BR.build(case)
    return _cache[case.name]


def _band_solver(sysm, cells, extra=()):
    c = sysm.case
    s = Solver(sysm.problem(extra))
    s.set_partition(cells)
    if c.outer_weight:
        s.set_tuning("outer_weight", c.outer_weight)
    if c.min_bandwidth:
        s.set_shard(0, 1, lambda *a: None, c.min_bandwidth)
    return s


def _band_reference(sysm):
    """pose blocks of S^-1 in user order"""
    S = BR.dense(sysm.band(0.0)[0])
    ref = SI.equilibrated_inverse(S)
    pos = np.argsort(sysm.s2u)                    # solver position of every user pose
    cols = 6*pos[:, None] + np.arange(6)[None, :]
    return ref[cols[:, :, None], cols[:, None, :]]


@pytest.mark.parametrize("name", [c.name for c in BR.PLAIN + BR.CELLS])
def test_band_pose_covariances(name):
    """every plain band layout and every cell case: the covariances come from the plain layout whatever the partition"""
    case = BR.CASES[name]
    sysm = _system(case)
    s = _band_solver(sysm, case.cells)
    C = s.marginal_covariance(POSE6)
    assert np.array_equal(C, C.transpose(0, 2, 1))
    err = SI.cov_error(C, _band_reference(sysm))
    print(f"COVBAND {case.family} {name}: {err:.2e}")
    assert err <= TOL_BAND[case.family], err
    idx = np.random.default_rng(1).permutation(case.n_pose)[:7]
    assert np.array_equal(s.marginal_covariance(POSE6, idx), C[idx])
    s.close()


@pytest.mark.parametrize("name", ["wb9_permuted", "c2_kend17", "c4_wb17", "c16_wb1", "c8_wb7"])
def test_band_covariances_independent_of_partition(name):
    case = BR.CASES[name]
    sysm = _system(case)
    got = []
    for cells in (-1, 1, 2, 4, 8):
        s = _band_solver(sysm, cells)
        got.append(s.marginal_covariance(POSE6))
        s.close()
    for cells, C in zip((1, 2, 4, 8), got[1:]):
        assert np.array_equal(C, got[0]), cells


@pytest.mark.parametrize("name,where", [("wb3", 0), ("wb3", -1), ("c2_kend17", 0), ("c2_kend17", 40)])
def test_indefinite_is_reported_then_optimized(name, where):
    case = BR.CASES[name]
    sysm = _system(case)
    neg, _ = BR.negative_prior(sysm, where % case.n_pose)
    s = _band_solver(sysm, case.cells, extra=[neg])
    with pytest.raises(DynobaError) as ei:
        s.marginal_covariance(POSE6)
    assert ei.value.status == ERR_INDETERMINATE
    st = s.optimize(max_iterations=3)
    assert np.isfinite(st["error_final"])
    s.close()


# ------------------------------------------------------------------------------------------------------------ full graphs
def _information(p, s):
    """sparse H = J^T J over [poses 6 | points 3 | flows 2 | velocities 3 | biases 6] from the device's Jacobians"""
    counts = (p.n_pose, p.n_point, p.n_flow, p.n_vel, p.n_bias)
    base = np.concatenate([[0], np.cumsum([c*d for c, d in zip(counts, CLASS_DIM)])])
    rows, cols, vals = [], [], []
    r0 = 0
    for bi, b in enumerate(p.blocks):
        A, _ = s.linearization(bi)
        d = A.shape[1]
        r = r0 + np.arange(b.n)[:, None]*d + np.arange(d)[None, :]
        c0 = 0
        for k, cls in enumerate(SLOT_CLASS[b.type]):
            w = CLASS_DIM[cls]
            var = base[cls] + w*b.idx[:, k].astype(np.int64)
            for c in range(w):
                rows.append(r.reshape(-1)); cols.append(np.repeat(var + c, d)); vals.append(A[:, :, c0 + c].reshape(-1))
            c0 += w
        r0 += b.n*d
    J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(r0, base[-1]))
    return (J.T @ J).tocsr(), counts, base


KINDS = [(POSE6, 0), (POINT3, 1), (FLOW2, 2), (VEL3, 3), (BIAS6, 4)]


@pytest.mark.parametrize("name", list(SI.cov_graphs()))
def test_graph_covariances(name):
    p = SI.cov_graphs()[name]()
    s = Solver(p)
    s.linearize()
    H, counts, base = _information(p, s)
    pcols = np.concatenate([np.arange(base[0], base[1]), np.arange(base[3], base[5])])
    for kind, cls in KINDS:
        if counts[cls] == 0:
            continue
        d = CLASS_DIM[cls]
        C = s.marginal_covariance(kind)
        blocks = base[cls] + d*np.arange(counts[cls])[:, None] + np.arange(d)[None, :]
        ref, kappa = SI.schur_inverse_blocks(H, pcols, blocks)
        tol = TOL_GRAPH_KAPPA*kappa*np.finfo(float).eps
        assert np.array_equal(C, C.transpose(0, 2, 1))
        err = SI.cov_error(C, ref)
        print(f"COVGRAPH {name} kind {kind}: {err:.2e} = {err/(kappa*np.finfo(float).eps):.2f} kappa eps, kappa {kappa:.2e} "
              f"({counts[cls]} variables)")
        assert err <= tol, (kind, err, kappa)
        if kind == POSE6 and p.n_vel == 0 and base[3] <= ORACLE_MAX_DIM:
            # the oracle linearises on its own: its Jacobians differ from the device's by rounding, amplified by kappa
            from oracle.oracle import OracleProblem
            Ho, _ = OracleProblem(p).dense_normal()
            oref = SI.marginal_blocks(SI.equilibrated_inverse(Ho), counts, 0)
            eo = SI.cov_error(C, oref)
            print(f"COVORACLE {name}: {eo:.2e}")
            assert eo <= 10*tol, eo
    s.close()


def test_singular_wcpe_is_indeterminate():
    """schur_reference's WCPE graph without the unit pose priors of cov_graphs: its information matrix is singular (LM
    only solves it damped), as gtsam::Marginals finds with IndeterminantLinearSystemException"""
    from dynosam_b200 import synth
    import schur_reference as SR
    p = synth.make_problem(n_frames=40, n_objects=1, n_static=300, n_dynamic=200, formulation="wcpe", seed=5,
                           object_span=(40, 40), max_dynamic_age=SR.GG_MAXL)
    s = Solver(p)
    with pytest.raises(DynobaError) as ei:
        s.marginal_covariance(POINT3)
    assert ei.value.status == ERR_INDETERMINATE
    s.close()


def test_last_poses_match_marginal_information():
    """C2: the covariance of the last pose-like variables is the inverse of dynoba_marginal's G (an independent path:
    a factorisation stopped before the kept block)"""
    from dynosam_b200 import synth
    p = synth.make_config("C2", formulation="hybrid")
    s = Solver(p)
    order = p.pose_order if p.pose_order is not None else np.arange(p.n_pose)
    s2u = np.argsort(order, kind="stable")          # user pose at each solver position
    k = 3
    keep = s2u[-k:]
    G, _ = s.marginal(keep)
    ref = np.linalg.inv(G)
    C = s.marginal_covariance(POSE6, keep)
    refb = np.array([ref[6*i:6*i + 6, 6*i:6*i + 6] for i in range(k)])
    err = SI.cov_error(C, refb)
    print(f"COVC2 last {k} poses: {err:.2e}")
    assert err <= TOL_C2, err
    s.close()


def _stats(st):
    return {k: st[k] for k in ("iterations", "inner_iterations", "error_initial", "error_final", "lambda_final")}


def test_optimize_after_covariance_is_unchanged():
    p = SI.cov_graphs()["hybrid"]()
    runs = []
    for with_cov in (False, False, True):
        s = Solver(p)
        if with_cov:
            s.marginal_covariance(POSE6); s.marginal_covariance(POINT3)
        st = s.optimize()
        runs.append((_stats(st), s.values()))
        s.close()
    (st0, v0), (st1, v1), (st2, v2) = runs
    assert st0 == st1 and all(np.array_equal(a, b) for a, b in zip(v0, v1)), "optimize is not repeatable"
    assert st2 == st0, (st2, st0)
    assert all(np.array_equal(a, b) for a, b in zip(v2, v0))


def test_covariance_follows_the_values():
    """after retract the covariances are recomputed at the new values (a fresh handle at those values agrees)"""
    p = SI.cov_graphs()["hybrid"]()
    s = Solver(p)
    C0 = s.marginal_covariance(POSE6); P0 = s.marginal_covariance(POINT3)
    rng = np.random.default_rng(4)
    delta = np.concatenate([rng.normal(0, 0.05, 6*p.n_pose), rng.normal(0, 0.2, 3*p.n_point)])
    s.retract(delta)
    C1 = s.marginal_covariance(POSE6); P1 = s.marginal_covariance(POINT3)
    pose, point, flow = s.values()
    s.close()
    f = Solver(dataclasses.replace(p, pose=pose, point=point, flow=flow))
    Cf = f.marginal_covariance(POSE6); Pf = f.marginal_covariance(POINT3)
    f.close()
    assert SI.cov_error(C1, Cf) <= 1e-12 and SI.cov_error(P1, Pf) <= 1e-12
    assert SI.cov_error(C0, Cf) > 1e-6 and SI.cov_error(P0, Pf) > 1e-6
