"""The two scalars of each LM decision, read back from the device (Solver.last_model after Solver.solve), against their
exact values from the device's own J, b, delta and the dense priors (tests/lm_reference.py), on every case of
tests/lm_cases.py and every lambda it names.

Errors are in units of u sum|terms| (u = 2^-53), the a-priori scale of the rounding of a sum of those terms in any
order.  The priors of the cases are linearised at the current values, so their local coordinates d are 0 up to the
rounding of the device's Logmap; |d| <= 16 u is added to the scale through the terms |delta_r G_rc| 16 u.  The tolerance
TOL is a fixed multiple of the worst value measured on an H100 (DESIGN.md section 4)."""
import numpy as np
import pytest

import lm_cases as LC
import lm_reference as LR
from dynosam_b200 import binding

pytestmark = pytest.mark.gpu
TOL = 16.0          # 4x the worst measured on an H100 80GB HBM3 at 700 W (4.02, lin of used_1024)


def _measure(s, p, lam, priors):
    try:
        delta = s.solve(lam)
    except binding.DynobaError as e:
        assert e.status == binding.ERR_INDETERMINATE
        assert s.last_model()[2] != 0.0
        return None
    oldLin, lin, fail = s.last_model()
    assert fail == 0.0
    J, b = LR.jacobian(p, s.linearization)
    M = LR.ExactModel(J, b, priors)
    o_ex, o_terms = M.old_lin()
    c_ex, c_terms = M.model(delta, lam)
    for q in priors:                 # |d| <= 16 u: g^T d in oldLin, 1/2 delta^T G d in lin
        o_terms += 16*float(np.abs(q.g).sum())
        c_terms += 8*float(np.abs(delta[q.cols]) @ np.abs(q.G).sum(1))
    e_old = abs(oldLin - o_ex)/(LR.U*max(o_terms, 1e-300))
    e_lin = abs(lin - c_ex)/(LR.U*max(c_terms, 1e-300))
    return e_old, e_lin, oldLin, lin


@pytest.mark.parametrize("case", LC.cases(), ids=lambda c: c.name)
def test_model_scalars_exact(case):
    p = case.problem
    s = binding.Solver(p)
    try:
        if case.partition:
            s.set_partition(case.partition)
        priors = LR.priors_at_lin(p)
        worst = [0.0, 0.0]
        solved = 0
        for lam in case.lambdas:
            r = _measure(s, p, lam, priors)
            if r is None:
                continue
            solved += 1
            e_old, e_lin, oldLin, lin = r
            worst = [max(worst[0], e_old), max(worst[1], e_lin)]
            assert e_old <= TOL, (case.name, lam, e_old, oldLin)
            assert e_lin <= TOL, (case.name, lam, e_lin, lin)
        assert solved >= 1
        # a solve right after calls that leave other partials in the shared buffer: an error evaluation and a single
        # block's linearisation
        s.error()
        s.linearize_block(0)
        r = _measure(s, p, case.lambdas[-1], priors)
        if r is not None:
            assert r[0] <= TOL and r[1] <= TOL, (case.name, r)
            worst = [max(worst[0], r[0]), max(worst[1], r[1])]
        print(f"lm-model {case.name}: oldLin {worst[0]:.3g}, lin {worst[1]:.3g} u sum|terms|")
    finally:
        s.close()


def test_literal_decrease_identity():
    """on a small graph: GTSAM's literal L(delta) = linear.error(0) - linear.error(delta) and the closed form C(delta) the
    device sums differ by exactly 1/2 delta^T ((H + lambda I) delta - g), which is the damped system's residual against
    the device's delta (difference (i) of DESIGN.md section 4); the device's lin is C, not L"""
    from dynosam_b200 import synth
    p = synth.make_problem(n_frames=4, n_objects=0, n_static=12, n_dynamic=0, seed=3, robust=False)
    s = binding.Solver(p)
    try:
        lam = 1e-3
        delta = s.solve(lam)
        oldLin, lin, _ = s.last_model()
        J, b = LR.jacobian(p, s.linearization)
        M = LR.ExactModel(J, b, [])
        assert M.identity_holds(delta, lam)
        L = M.literal_decrease(delta, lam)
        c_ex, c_terms = M.model(delta, lam)
        assert abs(lin - c_ex) <= TOL*LR.U*c_terms
        assert abs(L - c_ex) <= 1e-6*abs(c_ex)          # delta solves the damped system to about 1e-10 here
    finally:
        s.close()
