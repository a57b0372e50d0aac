"""The first stage of the solver on the CPU: the case list of tests/factor_cases.py reaches every boundary it names, the
50-digit reference (tests/lie_reference.py) is consistent with itself, `se3.cuh` compiled for the host equals GTSAM
4.2.0's formulas case by case, the CPU oracle equals the reference on every case, and five mutations of `se3.cuh` each
fail a named case by at least 100 times its tolerance."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from mpmath import mp, mpf

import factor_cases as FC
import lie_reference as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")
EPS = 2.0**-52
CASES = FC.cases()
PROBLEM_CASES = [n for n, c in CASES.items() if c.delta is None]


def test_cases_reach_every_boundary():
    seen = set()
    for c in CASES.values():
        b = FC.boundaries(c)
        assert set(c.hits) <= b, (c.name, set(c.hits) - b)
        assert all(h in FC.REQUIRED for h in c.hits), c.name
        seen |= set(c.hits)
    missing = set(FC.REQUIRED) - seen
    assert not missing, sorted(missing)


# ---------------------------------------------------------------------------------------------- the reference itself
def _xi(rng, th, vm):
    a = rng.normal(size=3); a /= np.linalg.norm(a)
    return [mpf(th)*mpf(float(x)) for x in a] + [mpf(vm)*mpf(float(x)) for x in rng.normal(size=3)]


def test_true_maps_invert_each_other():
    rng = np.random.default_rng(0)
    for th in ("1e-25", "1e-12", "1e-9", "1e-5", "0.3", "2.5", "3.14", "3.14159265"):
        for vm in ("0", "1e-3", "1e3"):
            xi = _xi(rng, th, vm)
            back = LR.log_se3(LR.exp_se3(xi))
            n = LR.norm(xi[:3])
            xi = [x/n*mpf(th) for x in xi[:3]] + xi[3:]          # (the axis was normalised in fp64)
            back = LR.log_se3(LR.exp_se3(xi))
            scale = 1 + max(abs(x) for x in xi)
            assert max(abs(a - b) for a, b in zip(xi, back)) <= mpf("1e-40")*scale/(mp.pi - mpf(th))**2, (th, vm)


def test_formula_maps_against_true_maps():
    """the error of GTSAM 4.2.0's formulas in exact arithmetic, branch by branch (table of lie_reference's docstring)"""
    rng = np.random.default_rng(1)
    for th, vm in (("1e-12", "1"), ("0.7e-8", "1e3"), ("1e-8", "1")):                 # Expmap, first order
        xi = _xi(rng, th, vm); t = LR.norm(xi[:3])
        (R, p), (Rg, pg) = LR.exp_se3(xi), LR.g_exp_se3(xi)
        assert max(abs(a - b) for a, b in zip(R, Rg)) <= t*t/2*(1 + mpf("1e-6"))
        assert max(abs(a - b) for a, b in zip(p, pg)) <= t*LR.norm(xi[3:])/2*(1 + mpf("1e-6"))
    for th in ("0.3", "2.5", "3.1"):                                                  # closed forms: equal
        xi = _xi(rng, th, "1")
        P, Pg = LR.exp_se3(xi), LR.g_exp_se3(xi)
        assert max(abs(a - b) for a, b in zip(LR.pose_flat(P), LR.pose_flat(Pg))) <= mpf("1e-45")
        assert max(abs(a - b) for a, b in zip(LR.log_se3(P), LR.g_log_se3(P))) <= mpf("1e-44")
    for th in ("1e-9", "1e-5", "2e-4", "3e-4"):                                       # Logmap, Taylor branch
        xi = _xi(rng, th, "1"); t = LR.norm(xi[:3]); P = LR.exp_se3(xi)
        LR.trace_start(); w = LR.g_log_se3(P); tr = LR.trace_stop()
        assert "log:taylor" in tr
        assert max(abs(a - b) for a, b in zip(w[:3], xi[:3])) <= t**5/30*(1 + mpf("1e-3")) + mpf("1e-44")
    for th in ("1e-12", "9e-11"):                                                     # Pose3 Logmap, small angle
        xi = _xi(rng, th, "1"); t = LR.norm(xi[:3]); P = LR.exp_se3(xi)
        w = LR.g_log_se3(P)
        assert max(abs(a - b) for a, b in zip(w[3:], xi[3:])) <= t*LR.norm(P[1])/2*(1 + mpf("1e-6"))
    for d in ("5e-6", "1e-8", "0"):                                                   # Logmap, pi branch
        for ax, k in (((0.6, 0.0, 0.8), 2), ((0.6, 0.8, 0.0), 1), ((1.0, 0.0, 0.0), 0)):
            t = mp.pi - mpf(d); a = LR.vec(ax); a = [x/LR.norm(a) for x in a]
            LR.trace_start(); w = LR.g_log_so3(LR.exp_so3([t*x for x in a])); tr = LR.trace_stop()
            assert "log:pi" in tr and "logpi:" + "xyz"[k] in tr
            assert abs(LR.norm(w) - mp.pi) <= mpf("1e-9")
            assert max(abs(x - t*y) for x, y in zip(w, a)) <= mpf(d)*mp.pi/(2*abs(a[k])) + mpf(d) + mpf("1e-45")
    # the other logarithm: an axis whose sub-branch component is negative comes back negated
    t = mp.pi - mpf("5e-6"); a = LR.vec((-0.6, 0.0, -0.8))
    w = LR.g_log_so3(LR.exp_so3([t*x for x in a]))
    assert max(abs(x + t*y) for x, y in zip(w, a)) <= mpf("2e-5")


def test_straddled_thresholds_branches_agree():
    """either side of each threshold the two neighbouring formulas agree to the bound of that threshold, so the side
    fp64 rounding picks cannot matter beyond it"""
    a = [mpf("0.6"), mpf("0.48"), mpf("0.64")]
    R = LR.exp_so3([mpf("3.1622776e-4")*x for x in a])                                 # tr - 3 = -1e-7
    d = max(abs(x - y) for x, y in zip(LR.g_log_so3(R, force="acos"), LR.g_log_so3(R, force="taylor")))
    assert d <= mpf("2e-19")                                                           # theta^5/30
    R = LR.exp_so3([(mp.pi - mpf("1e-5"))*x for x in a])                               # tr + 1 = 1e-10
    d = max(abs(x - y) for x, y in zip(LR.g_log_so3(R, force="acos"), LR.g_log_so3(R, force="pi")))
    assert d <= mpf("3e-5")
    for k, l in ((0, 1), (1, 2)):                                                      # |R_kk + 1| = 1e-5: sub-branches
        ax = [mpf("0.8"), mpf("0.6"), mpf("0.8")]; ax[2 - k] = mp.sqrt(mpf("0.5e-5")); ax[(3 - k) % 3 if k else 0] = mpf("0.6")
        n = LR.norm(ax); R = LR.exp_so3([(mp.pi - mpf("1e-9"))*x/n for x in ax])
        d = max(abs(x - y) for x, y in zip(LR.g_log_so3(R, force="pi", pi_sub=k), LR.g_log_so3(R, force="pi", pi_sub=l)))
        assert d <= mpf("2e-6")                                                        # (pi - theta) pi / (2 a_k), a_k = 2.2e-3
    w = [mpf("1.49e-8")*x for x in a]; v = [mpf(1), mpf(2), mpf(3)]                    # theta^2 = DBL_EPSILON
    Rg = LR.g_exp_se3(w + v); Rt = LR.exp_se3(w + v)
    assert max(abs(x - y) for x, y in zip(LR.pose_flat(Rg), LR.pose_flat(Rt))) <= mpf("1.49e-8")*4


def test_exact_jacobian_equals_the_closed_form_of_pose_to_point():
    """50-digit central differences through the retraction against d/dX = [[q]x -I], d/dp = R^T (gtsam::PoseToPointFactor)"""
    rng = np.random.default_rng(2)
    X = (LR.exp_so3(LR.vec(rng.normal(size=3))), LR.vec(rng.normal(size=3))); p = LR.vec(rng.normal(size=3)); z = LR.vec(rng.normal(size=3))
    J = LR.jacobian_exact(LR.POSE2POINT3, [X, p], z, None, None)
    q = LR.act_inv(X, p); Q = LR.skew(q); Rt = LR.tr3(X[0])
    want = [[Q[3*i+j] for j in range(3)] + [-mpf(int(i == j)) for j in range(3)] + [Rt[3*i+j] for j in range(3)] for i in range(3)]
    assert max(abs(a - b) for ra, rb in zip(J, want) for a, b in zip(ra, rb)) <= mpf("1e-25")


# ---------------------------------------------------------------------------------------------- se3.cuh on the host
def _build_shim(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = CSRC
    if patch is not None:                      # a mutated copy of se3.cuh, seen only by this build
        src = open(os.path.join(CSRC, "se3.cuh")).read()
        assert src.count(patch[0]) >= 1, patch
        inc = str(tmp_path / "mut"); os.makedirs(inc, exist_ok=True)
        a, b = src.split(patch[2], 1) if len(patch) > 2 else ("", src)          # patch[2]: only after this marker
        open(os.path.join(inc, "se3.cuh"), "w").write(a + (patch[2] if len(patch) > 2 else "") + b.replace(patch[0], patch[1], 1))
    so = str(tmp_path / ("se3_host%s.so" % ("" if patch is None else "_mut")))
    r = subprocess.run([nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets",
                        "-I", inc, os.path.join(ROOT, "tests", "capi", "se3_host.cu"), "-o", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    dp = C.POINTER(C.c_double)

    def call(name, *args, out):
        o = np.zeros(out)
        getattr(lib, name)(*[np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp) for a in args], o.ctypes.data_as(dp))
        return o
    return call


def _shim_cases():
    """(name, kind, inputs): every relative rotation of the rotation cases through Logmap / local / Adjoint, every step
    of the retract case through Expmap / retract"""
    out = []
    for th in FC.THETAS + ["pi-1e-5"]:
        for ax, a in FC.AXES.items():
            for tm in (0.0, 1.0, 1e3):
                out.append((f"log {th}@{ax} t={tm:g}", "log", FC.pose12(FC.rotation(th, a), tm*np.array([0.48, -0.6, 0.64]))))
    c = CASES["retract"]
    for i in range(c.problem.n_pose):
        out.append((f"retract step {i}", "retract", (c.problem.pose[i], c.delta[6*i:6*i + 6])))
    return out


def _shim_errors(call):
    """{name: error / tolerance} of the host build against the formula maps; the tolerance is the a-priori bound"""
    res = {}
    G = FC.random_pose(np.random.default_rng(3), 1.0, 2.0)
    for name, kind, x in _shim_cases():
        if kind == "log":
            P = LR.pose(x)
            straddle = name.startswith("log pi-1e-5")
            B = float(LR.log_rot_bound(P[0])); S = 1 + np.abs(x[9:]).max()
            unit = EPS*B*np.array([1, 1, 1, S, S, S])*4
            want = np.array(LR.to_float(LR.g_log_se3(P)))
            got = call("host_se3_logmap", x, out=6)
            err = np.abs(got - want)/unit
            if straddle:                       # tr + 1 = 1e-10 to rounding: either neighbour, to the bound where they meet
                alt = np.array(LR.to_float(LR.g_log_se3(P, force="acos")))
                err = np.minimum(err, np.abs(got - alt)/unit)
            res[name] = err.max() if np.isfinite(err).all() else np.inf
            wr = call("host_so3_logmap", x[:9], out=3)
            assert np.array_equal(wr, got[:3], equal_nan=True), name
            # Logmap(G^-1 (G x)) through se3_local: the product is rounded, the bound is the same
            Gx = FC.compose12(G, x)
            want = np.array(LR.to_float(LR.g_local(LR.pose(G), LR.pose(Gx))))
            got = call("host_se3_local", G, Gx, out=6)
            S2 = 3*(1 + np.abs(G[9:]).max() + np.abs(Gx[9:]).max())
            B2 = float(LR.log_rot_bound(LR.between(LR.pose(G), LR.pose(Gx))[0]))
            if not straddle and np.pi - np.linalg.norm(want[:3]) > 2e-5 or np.linalg.norm(want[:3]) < 3:
                res[name + " local"] = (np.abs(got - want)/(EPS*B2*np.array([1, 1, 1, S2, S2, S2])*8)).max()
            Ad = call("host_se3_adjoint", x, out=36).reshape(6, 6)
            want = np.array(LR.to_float(LR.adjoint(P)))
            assert np.abs(Ad - want).max() <= 4*EPS*S, name
        else:
            T, xi = x
            want = np.array(LR.to_float(LR.pose_flat(LR.g_retract(LR.pose(T), LR.vec(xi)))))
            got = call("host_se3_retract", T, xi, out=12)
            S = 1 + np.abs(T[9:]).max() + np.abs(xi[3:]).max()
            S += np.abs(xi[3:]).max()*float(FC.expmap_translation_bound(np.linalg.norm(xi[:3])))
            unit = EPS*np.array([1.0]*9 + [S]*3)*8
            res[name] = (np.abs(got - want)/unit).max()
            E = call("host_se3_expmap", xi, out=12); R = call("host_so3_expmap", xi[:3], out=9)
            assert np.array_equal(E[:9], R, equal_nan=True), name
            wantE = np.array(LR.to_float(LR.pose_flat(LR.g_exp_se3(LR.vec(xi)))))
            res[name + " expmap"] = (np.abs(E - wantE)/(EPS*np.array([1.0]*9 + [1 + np.abs(xi[3:]).max()*float(FC.expmap_translation_bound(np.linalg.norm(xi[:3])))]*3)*8)).max()
    return res


def test_host_build_of_se3_equals_the_formula_maps(tmp_path):
    res = _shim_errors(_build_shim(tmp_path))
    worst = max(res, key=res.get)
    print(f"FACTOR host-se3 worst {worst}: {res[worst]:.2g} of the a-priori bound")
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad


MUTATIONS = {
    "pi sub-branch threshold 1e-5 -> 1e-4": ("fabs(R[8] + 1.0) > 1e-5", "fabs(R[8] + 1.0) > 1e-4"),
    "second and third pi sub-branch swapped": ("fabs(R[4] + 1.0) > 1e-5", "!(fabs(R[0] + 1.0) > 1e-5)"),
    "Taylor term tr3/12 -> tr3/6": ("tr3/12.0", "tr3/6.0"),
    "so3_expmap near-zero threshold eps -> 1e-10": ("th2 <= DBL_EPSILON", "th2 <= 1e-10"),
    "se3_logmap 0.5*t -> 0.5": ("(0.5*t)*WT[i]", "(0.5)*WT[i]"),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_of_se3_fails_a_named_case(tmp_path, mutation):
    """each mutation, applied to a copy of se3.cuh that only this build sees, fails at least one case by >= 100 x its
    tolerance (the swap: the x sub-branch is preferred to the y one)"""
    try:
        res = _shim_errors(_build_shim(tmp_path, MUTATIONS[mutation]))
    except AssertionError as ex:               # so3_expmap and se3_expmap disagree bit for bit
        assert mutation.startswith("so3_expmap"), ex
        return
    worst = max(res, key=res.get)
    print(f"FACTOR mutation '{mutation}' caught by {worst}: {res[worst]:.2g} x tolerance")
    assert res[worst] >= 100, (mutation, worst, res[worst])


# ---------------------------------------------------------------------------------------------- the CPU oracle
@pytest.mark.parametrize("name", PROBLEM_CASES)
def test_oracle_equals_reference(name):
    from oracle import oracle as O
    c = CASES[name]
    o = O.OracleProblem(c.problem)
    FC.check_problem(c, o.linearize_block, o.error_block, o.error(), "oracle")


def test_oracle_retract_equals_reference():
    from oracle import oracle as O
    c = CASES["retract"]
    o = O.OracleProblem(c.problem)
    o.retract(c.delta)
    err = FC.retract_errors(c, o.pose, o.point, o.flow)
    print(f"FACTOR oracle retract: R {err[0]:.2g} t {err[1]:.2g} orthonormality {err[2]:.2g} (eps)")
    assert err[0] <= 8 and err[1] <= 8 and err[2] <= 8 and err[3] == 0
