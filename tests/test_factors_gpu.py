"""The factor kernels, the pose retraction and the dense prior's Logmap on the device, case by case (tests/factor_cases.py)
against the 50-digit reference (tests/lie_reference.py), through dynosam_b200.binding.Solver only.

Every error is in units of its a-priori bound (factor_cases' docstring: closed forms a few eps in the units of the
inputs; the acos branch of Logmap pi eps/(pi - theta)^2 towards pi; the numerically differentiated Jacobians
eps max|h|/delta; the pi branch equals GTSAM's formula to rounding and the true map to pi - theta), so a tolerance of 64
means 64 x that bound's unit.  Cheirality (zero Jacobian rows, 2 fx exactly) and a Huber weight of exactly 1 at n <= k
are compared bit for bit.  Each case prints `FACTOR H100 <case>: ...`.

Worst measured / tolerance, NVIDIA H100 80GB HBM3, power limit 700 W:

    family                                   b           A           A (numeric)   factor error   chi^2 (relative)
    rot (Logmap factors, every branch)       0.70 / 16   1.6 / 64    0.19 / 16     0.22 / 8       4.2e-8 (pi eps/(pi - theta)^2 cases)
    zero (exactly-zero residuals)            0 (bits)    0           0.12 / 16     0 (bits)       0
    straddle                                 0.05 / 16   0           -             0.03 / 8       2.3e-7 (theta = pi - 1e-5)
    cheirality, flowproj                     0.23 / 16   0.86 / 64   -             0.05 / 8       2.3e-16
    huber                                    0 (bits)    0           -             0 (bits)       1.8e-16
    sigma                                    0.42 / 16   1.3 / 64    -             0.17 / 8       1.8e-16
    blocks, gather                           0.42 / 16   3.2 / 64    0.59 / 16     0.21 / 8       2.6e-16
    big (131 072 / 131 073 factors)          0.71 / 16   5.8 / 64    -             0.21 / 8       1.2e-16 (bound: 1025 eps)
    retract                                  R 3 eps, t 0.7 of the bound, R^T R - I 4 eps / 8 each; 39 eps after 100 steps of 1e-3
    linear prior                             error 0.008 / 64, gradient 0.021 / 64

chi^2 is held to n_partials eps plus the summed per-factor differences (which the factor-error column bounds).
"""
import numpy as np
import pytest
from mpmath import mpf

import factor_cases as FC
import lie_reference as LR
from dynosam_b200.problem import PRIOR6, FactorBlock, Problem

pytestmark = pytest.mark.gpu

CASES = FC.cases()
PROBLEM_CASES = [n for n, c in CASES.items() if c.delta is None]
EPS = 2.0**-52


def _solver(p):
    from dynosam_b200.binding import Solver
    return Solver(p)


@pytest.mark.parametrize("name", PROBLEM_CASES)
def test_linearization_and_errors(name):
    c = CASES[name]
    s = _solver(c.problem)
    s.linearize()
    e = [s.error() for _ in range(3)]
    assert e[0] == e[1] == e[2] or not np.isfinite(e[0]), e          # the reduction order is fixed: same bits call to call
    FC.check_problem(c, s.linearization, s.factor_errors, e[0], "H100")
    s.close()


def test_retract():
    c = CASES["retract"]
    s = _solver(c.problem)
    s.retract(c.delta)
    pose, point, flow = s.values()
    err = FC.retract_errors(c, pose, point, flow)
    print(f"FACTOR H100 retract: R {err[0]:.2g} t {err[1]:.2g} orthonormality {err[2]:.2g} (units of eps and of the bound)")
    # the stored R is a product of two rotations rounded once each: orthonormal to 4 eps after one step
    assert err[0] <= 8 and err[1] <= 8 and err[2] <= 8 and err[3] == 0, err
    # nothing re-orthonormalises: what 100 retractions of 1e-3 rad leave, measured (a random walk of roundings)
    n = c.problem.n_pose
    d = np.zeros_like(c.delta); d[:6*n] = np.tile([6e-4, -8e-4, 0.0, 1e-3, 0.0, 0.0], n)
    for _ in range(100):
        s.retract(d)
    R = s.values()[0][:, :9].reshape(n, 3, 3)
    drift = np.abs(np.einsum("nij,nik->njk", R, R) - np.eye(3)).max()
    print(f"FACTOR H100 retract x100: |R^T R - I| = {drift/EPS:.3g} eps")
    assert drift <= 400*EPS                                            # 100 steps of at most 4 eps each
    s.close()


@pytest.mark.parametrize("offset", ["0", "1e-9", "pi-5e-6"])
def test_linear_prior_logmap(offset):
    """gtsam::LinearContainerFactor on one pose whose linearisation point is `offset` radians away: error
    1/2 d^T G d - g^T d + 1/2 f and gradient g - G d with d = Logmap(lin^-1 x) from the formula maps in 50 digits"""
    rng = np.random.default_rng(21)
    x = FC.random_pose(rng, 1.0, 2.0)
    rel = FC.pose12(FC.rotation(offset, (0.6, 0.8, 0.0)), [0.3, -0.2, 0.1] if offset != "0" else [0.0, 0.0, 0.0])
    lin = FC.compose12(x, np.array(LR.to_float(LR.pose_flat(LR.inverse(LR.pose(rel))))))
    A = rng.normal(size=(8, 6)); G = A.T @ A + np.eye(6); g = rng.normal(size=6)
    blk = FactorBlock(PRIOR6, np.array([[0]]), x[None], np.array([10.0]))                # (zero residual: the prior is all)
    p = Problem(x[None], np.zeros((0, 3)), blocks=[blk], linear_priors=[dict(idx=np.array([0], np.int32), lin=lin[None], G=G, g=g, f=0.7)])
    s = _solver(p)
    d = LR.g_local(LR.pose(lin), LR.pose(x))
    Gm = [[mpf(float(v)) for v in row] for row in G]; gm = LR.vec(g)
    Gd = [LR.dot(row, d) for row in Gm]
    e_ref = float(LR.dot(d, Gd)/2 - LR.dot(gm, d) + mpf("0.35"))
    grad_ref = np.array(LR.to_float([a - b for a, b in zip(gm, Gd)]))
    B = float(LR.log_rot_bound(LR.between(LR.pose(lin), LR.pose(x))[0]))/8
    unit = EPS*B*(1 + np.abs(x[9:]).max() + np.abs(lin[9:]).max())*np.abs(G).sum(1).max()*3
    e = s.error()
    _, gd = s.reduced_system(1e-3)
    err_e = abs(e - e_ref)/(unit*(np.abs(LR.to_float(d)).max() + 1)); err_g = np.abs(gd - grad_ref).max()/unit
    print(f"FACTOR H100 linear_prior {offset}: error {err_e:.2g} gradient {err_g:.2g}")
    assert err_e <= 64 and err_g <= 64
    s.close()
