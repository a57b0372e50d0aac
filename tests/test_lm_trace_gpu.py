"""dynoba_optimize's LM trace (Solver.lm_trace) on small graphs, with parameters that force each exit, against
lm_reference.replay (GTSAM 4.2.0 restated): fed the trace's scalars, the restatement re-derives every decision, every
lambda, (iterations, inner), lambda_final and error_final.  Each trial's scalars are then reproduced on a second handle
walked through the accepted steps with solve / last_model / retract / error.  oldLin is bit-identical until the first
accepted step (fixed-order sums at the same values); lin and nerr follow a damped step whose reduced system is scattered
with fp64 RED atomics, so they agree to the run-to-run rounding of that scatter (DESIGN.md section 4 (ii)), and so do
later values of oldLin.  Parameters under which the outer loop need not end are
refused before any launch."""
import math

import numpy as np
import pytest

import lm_reference as LR
from dynosam_b200 import binding, synth
from dynosam_b200.binding import POSE6, POINT3, FLOW2, VEL3, BIAS6

pytestmark = pytest.mark.gpu
# relative difference allowed between the two handles' lin and nerr (and oldLin after the first accepted step).  Measured
# on an H100 80GB HBM3 (700 W): 0 on every row of every case, the two handles agree bit for bit.  The bound leaves room
# only for a reordered RED scatter of the reduced system.
SPREAD_TOL = dict(oldLin=1e-12, lin=1e-12, nerr=1e-12)


def _rel(a, b):
    if a == b or (math.isnan(a) and math.isnan(b)):
        return 0.0
    return abs(a - b)/max(abs(b), 1e-300)


def _graph(seed=3):
    return synth.make_problem(n_frames=6, n_objects=1, n_static=60, n_dynamic=30, seed=seed)


def _indefinite():
    """a negative dense prior over two poses: the damped system is indefinite until lambda outweighs it"""
    import dataclasses
    p = _graph(5)
    G = -50.0*np.eye(12)
    return dataclasses.replace(p, linear_priors=[dict(idx=np.array([4, 5], np.int32), lin=p.pose[[4, 5]].copy(), G=G, g=np.zeros(12), f=0.0)])


def _nonfinite():
    p = _graph(7)
    p.point[0] = [0.0, 0.0, np.nan]
    return p


EXITS = [
    ("error_tol", _graph, dict(error_tol=1e300), ([], "error_tol")),
    ("max_iterations_zero", _graph, dict(max_iterations=0), ([], "max_iterations")),
    ("all_rejected", _graph, dict(min_model_fidelity=1e300, relative_error_tol=0.0, absolute_error_tol=0.0), (["giveup"], "absolute")),
    ("stop_without_success", _graph, dict(relative_error_tol=1e3, min_model_fidelity=1e300), (["stop"], "relative")),
    ("lower_clamp", _graph, dict(lambda_initial=1e-3, lambda_lower_bound=3e-5, max_iterations=4), None),
    ("rel_zero_abs", _graph, dict(relative_error_tol=0.0, absolute_error_tol=1e-9, max_iterations=30), None),
    ("max_iterations_cap", _graph, dict(max_iterations=2, relative_error_tol=0.0, absolute_error_tol=0.0), None),
    ("indefinite", _indefinite, dict(max_iterations=3), None),
    ("nonfinite", _nonfinite, dict(), None),
]


def _values(s, p):
    pose, point, flow = s.values()
    vel, bias = s.nav_values()
    return pose, point, flow, vel, bias


def _restore(s, v):
    for kind, a in zip((POSE6, POINT3, FLOW2, VEL3, BIAS6), v):
        if a.shape[0]:
            s.set_variables(kind, a)


@pytest.mark.parametrize("case", EXITS, ids=[c[0] for c in EXITS])
def test_trace_replays_and_reproduces(case):
    name, make, over, want = case
    p = make()
    P = LR.params(**over)
    s = binding.Solver(p)
    s2 = binding.Solver(p)
    try:
        st = s.optimize(binding.default_params(**P))
        tr = s.lm_trace()
        E = LR.effective(P)
        rp = LR.replay([tuple(r[[7, 3, 4, 6]]) for r in tr], st["error_initial"], E)
        assert len(rp.rows) == tr.shape[0], name
        for r, (it, inner, lam, err, succ, stop) in zip(tr, rp.rows):
            assert (r[0], r[1], r[2]) == (it, inner, lam), (name, r)
            assert r[5] == err or (math.isnan(r[5]) and math.isnan(err)), (name, r)
            assert (bool(r[8]), bool(r[9])) == (succ, stop), (name, r)
        assert (st["iterations"], st["inner_iterations"]) == (rp.iterations, rp.inner), name
        assert st["lambda_final"] == rp.lambda_final, name
        assert st["error_final"] == rp.error_final or (math.isnan(st["error_final"]) and math.isnan(rp.error_final)), name
        if want is not None:
            assert (rp.exits, rp.reason) == want, (name, rp.exits, rp.reason)
        if name == "lower_clamp":
            # an accepted step whose lambda / factor falls below the lower bound, followed by lambda == the bound
            lam_next = list(tr[1:, 2]) + [st["lambda_final"]]
            clamped = [i for i, r in enumerate(tr) if r[8] and r[2]/E["lambda_factor"] < E["lambda_lower_bound"]]
            assert clamped and all(lam_next[i] == E["lambda_lower_bound"] for i in clamped), tr[:, [2, 8]]
        if name == "indefinite":
            assert tr[0, 7] == 0.0 and any(tr[:, 8] == 1.0), tr[:, [2, 7, 8]]
        if name == "nonfinite":
            assert not math.isfinite(st["error_initial"]) and rp.reason == "nonfinite"
        # the same trials on a second handle, walked through the accepted steps.  Until the first accepted step both
        # handles linearise at the same values, so oldLin is bit-identical; after it the values differ by the rounding
        # of the step
        moved = False
        spread = dict(oldLin=0.0, lin=0.0, nerr=0.0)
        for r in tr:
            v = _values(s2, p)
            try:
                d = s2.solve(r[2])
            except binding.DynobaError as e:
                assert e.status == binding.ERR_INDETERMINATE and r[7] == 0.0, (name, r)
                continue
            oldLin, lin, fail = s2.last_model()
            assert r[7] == 1.0 and fail == 0.0
            if moved:
                spread["oldLin"] = max(spread["oldLin"], _rel(oldLin, r[3]))
            else:
                assert oldLin == r[3] or (math.isnan(oldLin) and math.isnan(r[3])), (name, oldLin, r[3])
            if not (math.isfinite(r[4]) and r[4] >= 0):
                continue
            spread["lin"] = max(spread["lin"], _rel(lin, r[4]))
            s2.retract(d)
            nerr = s2.error()
            spread["nerr"] = max(spread["nerr"], _rel(nerr, r[6]))
            if r[8]:
                moved = True
            else:
                _restore(s2, v)
        print(f"lm-trace {name}: relative spread " + ", ".join(f"{k} {v:.3g}" for k, v in spread.items()))
        for k, v in spread.items():
            assert v <= SPREAD_TOL[k], (name, k, v)
    finally:
        s.close(); s2.close()


REFUSED = [dict(relative_error_tol=0.0, absolute_error_tol=-1.0), dict(relative_error_tol=math.nan, absolute_error_tol=math.nan),
           dict(relative_error_tol=1e-5, absolute_error_tol=-1.0, error_tol=-1.0)]


@pytest.mark.parametrize("bad", REFUSED, ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_endless_parameters_refused_before_any_launch(bad):
    """on a handle that has optimised before: the refused call changes no value and leaves an empty trace"""
    p = _graph()
    s = binding.Solver(p)
    try:
        s.optimize(max_iterations=1)
        assert s.lm_trace().shape[0] >= 1
        before = s.values()
        with pytest.raises(binding.DynobaError) as e:
            s.optimize(**bad)
        assert e.value.status == binding.ERR_BAD_ARG
        assert s.lm_trace().shape[0] == 0
        assert all(np.array_equal(a, b) for a, b in zip(before, s.values()))
    finally:
        s.close()
