"""The LM decisions of csrc/lm_control.cuh, built for the host, against lm_reference.replay (GTSAM 4.2.0 restated), on
scripted trial scalars at every decision's exact threshold; and the refusal of parameters under which the outer loop
need not end, with a scripted run of endless give-ups that shows the loop the refusal prevents."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import lm_reference as LR
from dynosam_b200.binding import LmParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")
NAN, INF = math.nan, math.inf


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    so = str(tmp_path_factory.mktemp("lm_control") / "lm_control_host.so")
    r = subprocess.run([nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets",
                        "-I", CSRC, os.path.join(ROOT, "tests", "capi", "lm_control_host.cu"), "-o", so],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.host_lm_params_usable.argtypes = [C.POINTER(LmParams), C.POINTER(LmParams)]
    L.host_lm_converged.argtypes = [C.c_double, C.c_double, C.POINTER(LmParams)]
    L.host_lm_run.argtypes = [C.POINTER(LmParams), C.c_double, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _lm(P):
    q = LmParams()
    for k in LR.PARAM_NAMES:
        setattr(q, k, P[k])
    q.verbosity = 0
    return q


def usable(lib, P):
    out = LmParams()
    ok = lib.host_lm_params_usable(C.byref(_lm(P)), C.byref(out))
    return bool(ok), LR.params(out)


def run(lib, P, err0, script, cap=200):
    s = np.ascontiguousarray(script, np.float64).reshape(-1, 4)
    rows = np.zeros((cap, 10)); out = np.zeros(4, np.int64); outd = np.zeros(2)
    lib.host_lm_run(C.byref(_lm(P)), err0, s.ctypes.data, s.shape[0], cap, rows.ctypes.data, out.ctypes.data, outd.ctypes.data)
    return rows[:out[2]], dict(iterations=int(out[0]), inner=int(out[1]), ended=bool(out[3]), lambda_final=outd[0], error_final=outd[1])


def same(a, b):
    return a == b or (math.isnan(a) and math.isnan(b))


def check_against_replay(lib, P, err0, script, cap=200):
    """the host loop and the GTSAM restatement take the same decisions, bit for bit, from the same scalars"""
    rows, st = run(lib, P, err0, script, cap)
    s = np.asarray(script, np.float64).reshape(-1, 4)
    rp = LR.replay(lambda t: tuple(s[min(t, len(s) - 1)]), err0, P, cap=cap)
    assert len(rp.rows) == len(rows)
    for r, (it, inner, lam, err, succ, stop) in zip(rows, rp.rows):
        assert (r[0], r[1]) == (it, inner) and same(r[2], lam) and same(r[5], err), (r, rp.rows)
        assert (bool(r[8]), bool(r[9])) == (succ, stop), (r, succ, stop)
    assert (st["iterations"], st["inner"]) == (rp.iterations, rp.inner)
    assert same(st["lambda_final"], rp.lambda_final) and same(st["error_final"], rp.error_final)
    assert st["ended"] == (rp.reason != "cap")
    return rows, st, rp


ULP = lambda x: np.nextafter(x, INF) - x
# (name, parameter overrides, initial error, script rows (solved, oldLin, lin, nerr), expected (exits, reason))
CASES = [
    # modelFidelity == min_model_fidelity is a rejection; one ulp more cost is a success
    ("fidelity_equal", dict(min_model_fidelity=0.25, relative_error_tol=0.0), 1.0, [(1, 1.0, 0.5, 0.875)], None),
    ("fidelity_above", dict(min_model_fidelity=0.25, relative_error_tol=0.0, max_iterations=1), 1.0,
     [(1, 1.0, 0.5, np.nextafter(0.875, 0.0))], (["accepted"], "max_iterations")),
    # lin == eps oldLin: no fidelity test, the step is rejected although the cost fell
    ("lin_at_eps", dict(relative_error_tol=0.0), 1.0, [(1, 1.0, 2.0**-52, 0.5)], None),
    ("lin_above_eps", dict(relative_error_tol=0.0, max_iterations=1, min_model_fidelity=-INF), 1.0,
     [(1, 1.0, 2.0**-52 + 2.0**-104, 0.5)], (["accepted"], "max_iterations")),
    # |cost| == rel err does not stop; one ulp less does
    ("stop_equal", dict(relative_error_tol=0.25, min_model_fidelity=1e300), 1.0, [(1, 1.0, 0.5, 0.75)], None),
    ("stop_below", dict(relative_error_tol=0.25, min_model_fidelity=1e300), 1.0, [(1, 1.0, 0.5, 0.75 + ULP(0.75))],
     (["stop"], "relative")),
    # lambda * factor == upper exactly gives up; upper one ulp higher takes one more trial
    ("upper_exact", dict(lambda_initial=1.0, lambda_factor=2.0, lambda_upper_bound=8.0), 1.0, [(0, 0, 0, 0)],
     (["giveup"], "relative")),
    ("upper_above", dict(lambda_initial=1.0, lambda_factor=2.0, lambda_upper_bound=8.0 + ULP(8.0)), 1.0, [(0, 0, 0, 0)],
     (["giveup"], "relative")),
    # lambda / factor below the lower bound is clamped to it
    ("lower_clamp", dict(lambda_initial=1.0, lambda_factor=10.0, lambda_lower_bound=0.5, max_iterations=2, min_model_fidelity=0.0),
     4.0, [(1, 4.0, 1.0, 3.0), (1, 3.0, 1.0, 2.0)], (["accepted", "accepted"], "max_iterations")),
    # a decrease equal to absolute_error_tol converges; one ulp larger tolerance too, one ulp smaller does not
    ("abs_equal", dict(relative_error_tol=0.0, absolute_error_tol=0.25, min_model_fidelity=0.0), 1.0,
     [(1, 1.0, 0.25, 0.75), (0, 0, 0, 0)], (["accepted"], "absolute")),
    ("abs_below", dict(relative_error_tol=0.0, absolute_error_tol=np.nextafter(0.25, 0.0), min_model_fidelity=0.0, max_iterations=2), 1.0,
     [(1, 1.0, 0.25, 0.75), (1, 0.75, 0.25, 0.5)], (["accepted", "accepted"], "max_iterations")),
    # relative decrease at the tolerance
    ("rel_equal", dict(relative_error_tol=0.25, absolute_error_tol=-1.0, min_model_fidelity=0.0), 1.0,
     [(1, 1.0, 0.25, 0.75)], (["accepted"], "relative")),
    # currentError == 0 (error_tol < 0): the relative test is 0/0, the absolute test ends the loop
    ("error_zero", dict(error_tol=-1.0, absolute_error_tol=0.0), 0.0, [(1, 0.0, 0.0, 0.0)], (["giveup"], "absolute")),
    # error_tol at or above the initial error, max_iterations 0: no trial
    ("error_tol_initial", dict(error_tol=1.0), 1.0, [(1, 1.0, 1.0, 0.0)], ([], "error_tol")),
    ("max_iterations_zero", dict(max_iterations=0), 1.0, [(1, 1.0, 1.0, 0.0)], ([], "max_iterations")),
    # lin = -0.0 is a valid step (>= 0) without a fidelity test; NaN lin is a failed solve; NaN nerr is a rejection
    ("lin_negative_zero", dict(relative_error_tol=0.5), 1.0, [(1, 1.0, -0.0, 0.75)], (["stop"], "relative")),
    ("lin_negative", dict(relative_error_tol=0.5), 1.0, [(1, 1.0, -1e-300, 0.75)], (["giveup"], "relative")),
    ("lin_nan", dict(), 1.0, [(1, 1.0, NAN, 0.5)], (["giveup"], "relative")),
    ("lin_inf", dict(min_model_fidelity=-1.0), 1.0, [(1, 1.0, INF, 0.5)], (["giveup"], "relative")),
    ("nerr_nan", dict(), 1.0, [(1, 1.0, 0.5, NAN)], (["giveup"], "relative")),
    ("unsolved", dict(), 1.0, [(0, 1.0, 0.5, 0.5)], (["giveup"], "relative")),
    # an infinite initial error: one step is taken, then the loop ends on !isfinite(currentError)
    ("initial_inf", dict(), INF, [(1, 1.0, 0.5, 0.5)], (["accepted"], "nonfinite")),
    ("initial_nan", dict(), NAN, [(1, 1.0, 0.5, 0.5)], (["giveup"], "nonfinite")),
    # rejected, then accepted at a larger lambda (an indefinite system at small lambda)
    ("fail_then_accept", dict(max_iterations=1), 2.0, [(0, 0, 0, 0), (0, 0, 0, 0), (1, 2.0, 1.0, 1.0)],
     (["accepted"], "max_iterations")),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_decisions_match_gtsam_restatement(lib, case):
    name, over, err0, script, want = case
    ok, P = usable(lib, LR.params(**over))
    assert ok, name
    rows, st, rp = check_against_replay(lib, P, err0, script)
    if want is not None:
        assert (rp.exits, rp.reason) == want, (name, rp.exits, rp.reason)


def test_threshold_pairs_differ(lib):
    """each threshold pair above really sits on the boundary: the two sides take different first decisions"""
    first = {c[0]: check_against_replay(lib, usable(lib, LR.params(**c[1]))[1], c[2], c[3])[2].rows[:1] for c in CASES}
    for a, b in [("fidelity_equal", "fidelity_above"), ("lin_at_eps", "lin_above_eps"), ("stop_equal", "stop_below")]:
        assert first[a] != first[b], (a, b)
    up = {c[0]: check_against_replay(lib, usable(lib, LR.params(**c[1]))[1], c[2], c[3])[1] for c in CASES}
    assert up["upper_exact"]["inner"] == 3 and up["upper_above"]["inner"] == 4
    assert up["lower_clamp"]["lambda_final"] == 0.5


def test_dbl_min_raise(lib):
    """a lower bound below DBL_MIN is raised to it, and a run of accepted steps stops dividing lambda there"""
    ok, P = usable(lib, LR.params(lambda_initial=1e-300, lambda_factor=1e10, lambda_lower_bound=0.0, max_iterations=3,
                                  min_model_fidelity=0.0, relative_error_tol=0.0, absolute_error_tol=0.0))
    assert ok and P["lambda_lower_bound"] == LR.DBL_MIN == LR.effective(LR.params())["lambda_lower_bound"]
    rows, st, rp = check_against_replay(lib, P, 8.0, [(1, 8.0, 1.0, 4.0), (1, 4.0, 1.0, 2.0), (1, 2.0, 1.0, 1.0)])
    assert st["lambda_final"] == LR.DBL_MIN and st["iterations"] == 3
    assert usable(lib, LR.params(lambda_lower_bound=1e-200))[1]["lambda_lower_bound"] == 1e-200


def test_climb_limit(lib):
    """factors that need more than 10^4 rejected steps from min(initial, lower) to upper are refused, fewer accepted"""
    span = math.log(1e5) - math.log(LR.DBL_MIN)          # from the raised lower bound
    f_edge = math.exp(span/1e4)
    assert usable(lib, LR.params(lambda_factor=f_edge*(1 + 1e-9)))[0]
    assert not usable(lib, LR.params(lambda_factor=f_edge*(1 - 1e-9)))[0]
    span = math.log(1e5) - math.log(1e-5)                # lower bound above lambda_initial: from lambda_initial
    f_edge = math.exp(span/1e4)
    assert usable(lib, LR.params(lambda_factor=f_edge*(1 + 1e-9), lambda_lower_bound=1e-3))[0]
    assert not usable(lib, LR.params(lambda_factor=f_edge*(1 - 1e-9), lambda_lower_bound=1e-3))[0]
    for bad in (dict(lambda_initial=0.0), dict(lambda_initial=NAN), dict(lambda_factor=1.0), dict(lambda_factor=INF),
                dict(lambda_upper_bound=NAN)):
        assert not usable(lib, LR.params(**bad))[0], bad


TOLS = (-INF, -1.0, -0.0, 0.0, 1e-300, 1e-5, 1.0, INF, NAN)
ERRORS = (0.0, -0.0, 5e-324, 1e-300, 1.0, 1e300, -1.0)


def test_refusal_is_exactly_endless_giveups(lib):
    """lm_params_usable accepts a tolerance triple iff a decrease of exactly 0 converges at every finite error the outer
    loop can stand at (one it did not stop at by error_tol; at a non-finite error the loop ends on isfinite)"""
    for a in TOLS:
        for r in TOLS:
            for e in TOLS:
                P = LR.params(absolute_error_tol=a, relative_error_tol=r, error_tol=e)
                ends = all(LR.check_convergence(r, a, e, x, x)[0] for x in ERRORS if not (x <= e))
                host = all(lib.host_lm_converged(x, x, C.byref(_lm(P))) for x in ERRORS if not (x <= e))
                assert ends == host, (a, r, e)
                assert usable(lib, P)[0] == ends, (a, r, e)


ENDLESS = [
    # "always run max_iterations": relative 0, absolute negative; LM stalls at a minimum (no step can decrease the cost)
    (dict(relative_error_tol=0.0, absolute_error_tol=-1.0), 1.0, [(1, 1.0, 0.0, 1.0)]),
    (dict(relative_error_tol=NAN, absolute_error_tol=NAN), 1.0, [(0, 0, 0, 0)]),
    # a noise-free graph at its ground truth with a negative error_tol: error 0, relative test 0/0
    (dict(relative_error_tol=1e-5, absolute_error_tol=-1.0, error_tol=-1.0), 0.0, [(1, 0.0, 0.0, 0.0)]),
]


@pytest.mark.parametrize("k", range(len(ENDLESS)))
def test_endless_giveups_are_refused(lib, k):
    over, err0, script = ENDLESS[k]
    P = LR.effective(LR.params(**over))
    old_rule = (math.isfinite(P["lambda_initial"]) and P["lambda_initial"] > 0 and math.isfinite(P["lambda_factor"])
                and P["lambda_factor"] > 1 and not math.isnan(P["lambda_upper_bound"]))
    assert old_rule                                       # the climb rule alone let these through
    cap = 10000
    rows, st, rp = check_against_replay(lib, P, err0, script, cap=cap)
    assert not st["ended"] and rp.reason == "cap" and len(rows) == cap
    assert st["iterations"] == 0 and set(rp.exits) == {"giveup"}
    assert not usable(lib, P)[0]
