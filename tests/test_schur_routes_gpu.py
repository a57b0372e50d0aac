"""Landmark elimination on the device, route by route, against the dense fp64 reference (schur_reference.py) built from
the device's own whitened Jacobians.  Errors are in the scaled units of schur_reference's comparator.

Tolerance 1e-11 for S, g_S and the landmark / flow step; the device sums in another order (RED atomics, warp
shuffles), so the expected difference is fp64 reassociation.  Worst measured on an H100 80GB HBM3 (400 W), over both
lambdas and every cell layout:

    route graph     S        g_S      dl
    window_np1      1.4e-13  5.3e-14  1.3e-12   (once-seen stereo points: landmark blocks conditioned ~3e3)
    window_np2      3.0e-15  4.2e-16  1.3e-15
    simple          2.6e-15  1.1e-15  1.1e-16
    general_wcme    1.9e-15  1.0e-15  1.8e-15
    general_wcpe    2.1e-15  1.4e-15  2.8e-16
    all_types       1.7e-15  3.9e-15  1.4e-14
"""
import numpy as np
import pytest

import schur_reference as SR
from dynosam_b200.binding import Solver

pytestmark = pytest.mark.gpu

TOL = 1e-11
LAMBDAS = (1e-4, 1e-1)
GRAPHS = sorted(SR.ROUTE_GRAPHS)
_cache = {}


def _problem(name):
    if name not in _cache:
        _cache[name] = SR.ROUTE_GRAPHS[name]()
    return _cache[name]


def _reference(s, p, lam):
    s.linearize()
    return SR.Reference(p, s.linearization, lam)


def _max_cells(s):
    """the most cells the band layout can cut this reduced system into (kernels_band.cu band_plan_layout)"""
    info = s.info()
    NT = (info["reduced_dim"] + 31)//32
    WB = min(max((info["bandwidth"] + 31)//32, 1), NT - 1)
    return (NT + WB)//(2*WB + 2*max(WB, 2))


def _check_solve(s, p, R, lam):
    d = s.solve(lam)
    npz = 6*p.n_pose
    dp, dl = d[:npz], d[npz:]
    el = R.l_err(dl, dp)
    # the pose step solves the reference system: backward error in the comparator's units, and the dense solve
    sc = np.sqrt(R.Hdiag[:npz])
    back = float((np.abs(R.S @ dp - R.gS)/(sc*(R.r + np.abs(sc*dp).max()))).max())
    ref = R.pose_step()
    fwd = np.linalg.norm(dp - ref)/np.linalg.norm(ref)
    return el, back, fwd


@pytest.mark.parametrize("name", GRAPHS)
def test_reduced_system_matches_reference(name):
    p = _problem(name)
    s = Solver(p)
    for lam in LAMBDAS:
        R = _reference(s, p, lam)
        S, g = s.reduced_system(lam)
        es, eg = R.s_err(S), R.g_err(g)
        print(f"{name} lambda {lam:g}: S {es:.2e} g_S {eg:.2e}")
        assert es <= TOL and eg <= TOL, (es, eg)
    s.close()


@pytest.mark.parametrize("name", GRAPHS)
def test_damped_solve_matches_reference(name):
    """dynoba_solve: landmark and flow steps against the reference back-substitution of the device's own pose step,
    the pose step against the reference S; one plain band factorisation, the default layout, and 2 and 4 cells where
    the graph is long enough for them (window_np1 is built to be)."""
    p = _problem(name)
    for cells in (-1, 0, 2, 4):
        s = Solver(p); s.set_partition(cells)
        if cells > 0 and _max_cells(s) < cells:
            assert name != "window_np1", _max_cells(s)
            s.close()
            continue
        for lam in LAMBDAS:
            R = _reference(s, p, lam)
            el, back, fwd = _check_solve(s, p, R, lam)
            print(f"{name} cells {cells} lambda {lam:g}: dl {el:.2e} pose backward {back:.2e} forward {fwd:.2e}")
            assert el <= TOL and back <= TOL and fwd <= 1e-6, (cells, lam, el, back, fwd)
        s.close()


@pytest.mark.parametrize("name", GRAPHS)
def test_shuffled_factors_match_reference(name):
    """every factor listed in a random order: the general sort of the symbolic phase"""
    q = SR.permuted(_problem(name), 7, landmark_runs=False)
    s = Solver(q)
    lam = LAMBDAS[0]
    R = _reference(s, q, lam)
    S, g = s.reduced_system(lam)
    assert R.s_err(S) <= TOL and R.g_err(g) <= TOL, (R.s_err(S), R.g_err(g))
    el, back, fwd = _check_solve(s, q, R, lam)
    assert el <= TOL and back <= TOL and fwd <= 1e-6, (el, back, fwd)
    s.close()


@pytest.mark.parametrize("name", GRAPHS)
def test_lm_matches_oracle(name):
    """five LM iterations: every accepted and rejected step goes through the back-substitution and model decrease of
    each route.  The WCPE motion-pose factor is differentiated numerically (1e-6 apart between device and oracle)."""
    from oracle import oracle as O
    p = _problem(name)
    s = Solver(p); o = O.OracleProblem(p)
    st = s.optimize(max_iterations=5); so = o.optimize(max_iterations=5)
    tol = 1e-3 if name == "general_wcpe" else 1e-6
    assert st["iterations"] == so["iterations"] and st["inner_iterations"] == so["inner_iterations"], (st, so)
    assert abs(st["error_final"] - so["error_final"]) <= tol*so["error_final"], (st, so)
    s.close()


def test_chain_past_general_kernel_is_refused():
    from dynosam_b200.binding import DynobaError, ERR_UNSUPPORTED
    s = Solver(SR.refused_chain_graph())
    with pytest.raises(DynobaError) as ei:
        s.solve(1e-4)
    assert ei.value.status == ERR_UNSUPPORTED
    s.close()
