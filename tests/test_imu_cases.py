"""The visual-inertial factor on the CPU: the case list of tests/imu_cases.py reaches every boundary it names, the 50-digit
reference (tests/imu_lie_reference.py) is consistent with itself, `imu.cuh` compiled for the host equals the reference
case by case, and mutations of `imu.cuh` -- the parent's cancelling 1 - cos(theta) among them -- each fail a named case
by the margin stated in MUTATIONS."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from mpmath import mp, mpf

import imu_cases as IC
import imu_lie_reference as IL
import lie_reference as LR
from dynosam_b200.problem import COMBINED_IMU15

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")
EPS = 2.0**-52
CASES = IC.cases()
HOST_CASES = [n for n, c in CASES.items() if not n.startswith("big_")]


def test_cases_reach_every_boundary():
    seen = set()
    for c in CASES.values():
        b = IC.boundaries(c)
        assert set(c.hits) <= b, (c.name, set(c.hits) - b)
        assert all(h in IC.REQUIRED for h in c.hits), (c.name, set(c.hits) - set(IC.REQUIRED))
        seen |= set(c.hits)
    missing = set(IC.REQUIRED) - seen
    assert not missing, sorted(missing)


# ---------------------------------------------------------------------------------------------- the reference itself
def _axis(rng):
    a = rng.normal(size=3)
    return [mpf(float(x)) for x in a/np.linalg.norm(a)]


def _dmax(A, B):
    return max(abs(a - b) for a, b in zip(A, B))


def test_jr_closed_forms_equal_50_digit_differences():
    """d/dd Log(Exp(x) Exp(d)) at d = 0 is Jr(x)^-1 and d/dd Log(Exp(x)^-1 Exp(x + d)) is Jr(x): both by central
    differences through the true maps, against the closed forms"""
    rng = np.random.default_rng(0)
    h = mpf("1e-20")
    for th in ("1e-12", "0.999e-5", "1.001e-5", "2e-5", "1e-3", "0.3", "2.5", "3.1"):
        x = [mpf(th)*a for a in _axis(rng)]
        E = LR.exp_so3(x); Et = LR.tr3(E)
        Ji = [[None]*3 for _ in range(3)]; Jr = [[None]*3 for _ in range(3)]
        for j in range(3):
            d = [mpf(0)]*3; d[j] = h
            m = [-v for v in d]
            ci = [(a - b)/(2*h) for a, b in zip(LR.log_so3(LR.mul3(E, LR.exp_so3(d))), LR.log_so3(LR.mul3(E, LR.exp_so3(m))))]
            cr = [(a - b)/(2*h) for a, b in zip(LR.log_so3(LR.mul3(Et, LR.exp_so3([u + v for u, v in zip(x, d)]))),
                                                LR.log_so3(LR.mul3(Et, LR.exp_so3([u + v for u, v in zip(x, m)]))))]
            for i in range(3):
                Ji[i][j] = ci[i]; Jr[i][j] = cr[i]
        assert _dmax(sum(Ji, []), IL.jr_inv(x)) <= mpf("1e-30"), th
        assert _dmax(sum(Jr, []), IL.jr(x)) <= mpf("1e-30"), th


def test_formula_jr_against_true_jr():
    """the table of imu_lie_reference's docstring, row by row"""
    rng = np.random.default_rng(1)
    for th in ("1e-12", "1e-9", "1.4e-8"):                                     # theta^2 <= DBL_EPSILON
        x = [mpf(th)*a for a in _axis(rng)]; t = LR.norm(x)
        assert LR.dot(x, x) <= LR.EXP_NEAR_ZERO
        assert _dmax(IL.g_jr(x), IL.jr(x)) <= t*t/6*(1 + mpf("1e-6"))
        assert _dmax(IL.g_jr_inv(x), IL.jr_inv(x)) <= t/2*(1 + mpf("1e-6"))
        assert _dmax(IL.g_jr_inv(x), IL.jr_inv(x)) >= t/2*mpf("0.1")         # (the bound is attained, up to the axis)
    for th in ("1.5e-8", "1e-5", "0.3", "2.5", "3.14159"):                     # closed forms: equal
        x = [mpf(th)*a for a in _axis(rng)]
        assert _dmax(IL.g_jr(x), IL.jr(x)) == 0 and _dmax(IL.g_jr_inv(x), IL.jr_inv(x)) == 0


def test_jr_series_meets_closed_form_at_the_switch():
    """either side of theta^2 = 1e-10 (so3_jr, so3_jr_inv) the series and the closed form agree far below eps"""
    for th in ("0.999e-5", "1.001e-5"):
        t = mpf(th)
        a_s, c_s = mpf(1)/2 - t*t/24, mpf(1)/12 + t*t/720
        a_c = 2*mp.sin(t/2)**2/(t*t); c_c = 1/(t*t) - (1 + mp.cos(t))/(2*t*mp.sin(t))
        assert abs(a_s - a_c) <= mpf("1e-22") and abs(c_s - c_c) <= mpf("1e-22")


def test_residual_forms_and_exact_jacobian():
    """the formula residual equals the true one where the maps agree, and the 50-digit difference Jacobian is a
    derivative: a step of 1e-12 along a random direction moves the true residual by J d to 1e-22"""
    c = CASES["dt_g"]; p = c.problem; blk = p.blocks[0]
    rng = np.random.default_rng(2)
    for f in (0, 5, 11):
        i0, v0, i1, v1, b0, b1 = blk.idx[f]
        a = [LR.pose(p.pose[i0]), LR.vec(p.vel[v0]), LR.pose(p.pose[i1]), LR.vec(p.vel[v1]), LR.vec(p.bias[b0]), LR.vec(p.bias[b1])]
        r_t = IL.residual(*a, blk.meas[f]); r_g = IL.residual(*a, blk.meas[f], maps="gtsam")
        # (dR and R_j are orthonormal to rounding only: atan2 and acos read such a matrix differently, far below eps)
        assert _dmax(r_t, r_g) <= mpf(EPS)/16
        J = IL.jacobian_exact(*a, blk.meas[f])
        d = [mpf(float(x))*mpf("1e-12") for x in rng.normal(size=30)]
        b = list(a); o = 0
        for s, n in enumerate(IL.SLOT_DIMS):
            step = d[o:o + n]; o += n
            b[s] = LR.retract(a[s], step) if s in (0, 2) else [x + y for x, y in zip(a[s], step)]
        r2 = IL.residual(*b, blk.meas[f])
        lin = [sum(J[i][j]*d[j] for j in range(30)) for i in range(15)]
        assert _dmax([x - y for x, y in zip(r2, r_t)], lin) <= mpf("1e-22")


# ---------------------------------------------------------------------------------------------- imu.cuh on the host
def _build_shim(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [CSRC]
    if patch is not None:                      # a mutated copy of imu.cuh, seen only by this build
        src = open(os.path.join(CSRC, "imu.cuh")).read()
        assert src.count(patch[0]) == 1, patch
        d = str(tmp_path / "mut"); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "imu.cuh"), "w").write(src.replace(patch[0], patch[1]))
        inc = [d, CSRC]
    so = str(tmp_path / ("imu_host%s.so" % ("" if patch is None else "_mut")))
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "imu_host.cu"), "-o", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    dp = C.POINTER(C.c_double)

    def call(name, *args, out):
        o = np.zeros(out)
        getattr(lib, name)(*[np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp) for a in args], o.ctypes.data_as(dp))
        return o
    return call


def _host_errors(call, names=HOST_CASES):
    """{case: worst of b, A, e in units of the tolerance} of the host build, whitened on the host in fp64"""
    res = {}
    for name in names:
        c = CASES[name]; p = c.problem
        lin = {}
        for bi, blk in enumerate(p.blocks):
            if blk.type != COMBINED_IMU15:
                D = blk.meas.shape[1]
                x = (p.vel if D == 3 else p.bias)[blk.idx[:, 0]]
                isg = np.broadcast_to(1.0/(blk.sigma if blk.sigma_bcast else blk.sigma), (blk.n, D))
                rw = (x - blk.meas)*isg
                lin[bi] = (np.einsum("ni,ij->nij", isg, np.eye(D)), -rw, 0.5*(rw*rw).sum(1))
                continue
            A = np.zeros((blk.n, 15, 30)); b = np.zeros((blk.n, 15)); e = np.zeros(blk.n)
            for f in range(blk.n):
                i0, v0, i1, v1, b0, b1 = blk.idx[f]
                out = call("host_imu_eval", p.pose[i0], p.vel[v0], p.pose[i1], p.vel[v1], p.bias[b0], p.bias[b1], blk.meas[f], out=15 + 450)
                r2 = call("host_imu_residual", p.pose[i0], p.vel[v0], p.pose[i1], p.vel[v1], p.bias[b0], p.bias[b1], blk.meas[f], out=15)
                assert np.array_equal(out[:15], r2), (name, f, "r with and without J")
                R = IC._R(blk, f)
                rw = R@out[:15]
                A[f] = R@out[15:].reshape(15, 30); b[f] = -rw; e[f] = 0.5*rw@rw
            lin[bi] = (A, b, e)
        chi2 = float(sum(v[2].sum() for v in lin.values()))
        try:
            w = IC.check_problem(c, lambda bi: lin[bi][:2], lambda bi: lin[bi][2], chi2, "host")
            res[name] = max(w["b"]/IC.TOL["b"], w["A"]/IC.TOL["A"], w["e"]/IC.TOL["e"])
        except AssertionError as ex:
            w = ex.args[0][1] if isinstance(ex.args[0], tuple) and len(ex.args[0]) > 1 and isinstance(ex.args[0][1], dict) else None
            res[name] = max(w["b"]/IC.TOL["b"], w["A"]/IC.TOL["A"], w["e"]/IC.TOL["e"]) if w else np.inf
    return res


def test_host_build_of_imu_equals_the_reference(tmp_path):
    res = _host_errors(_build_shim(tmp_path))
    worst = max(res, key=res.get)
    print(f"IMU host worst {worst}: {res[worst]:.2g} of the tolerance")
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad


def test_host_jr_equals_the_true_maps(tmp_path):
    """so3_jr / so3_jr_inv against the 50-digit true maps at every theta of the cases, in eps (entries of size <= 1 +
    theta^2; jr_inv_bound near pi)"""
    call = _build_shim(tmp_path)
    worst = 0.0
    for th in IC.THETAS[1:] + ["pi-1e-5", "1e-12"]:
        x = [IC.theta_of(th)*a for a in IC.unit(IC.JR_AXIS)]
        xf = np.array(LR.to_float(x)); xm = LR.vec(xf)
        t = float(LR.norm(xm))
        e1 = np.abs(call("host_so3_jr", xf, out=9) - np.array(LR.to_float(IL.jr(xm)))).max()/EPS
        e2 = np.abs(call("host_so3_jr_inv", xf, out=9) - np.array(LR.to_float(IL.jr_inv(xm)))).max()/(EPS*float(IL.jr_inv_bound(t))/8*(1 + t*t))
        worst = max(worst, e1, e2)
        assert e1 <= 4 and e2 <= 4, (th, e1, e2)
    print(f"IMU host Jr / Jr^-1 worst {worst:.2g} eps")


# the first entry is the parent's so3_jr: (1 - cos)/theta^2 cancels, 3.7e3 eps in a Jr entry at theta = 2e-5
MUTATIONS = {
    "1 - cos(theta) formed directly": ("const double th = sqrt(th2), s2 = sin(0.5*th); a = 2.0*s2*s2/th2;",
                                       "const double th = sqrt(th2); a = (1.0 - cos(th))/th2;", "theta", 10),
    "JJ = JRw (Jr(theta) dropped)": ("m3mul(Jrt, JRw, JJ);", "for (int i = 0; i < 9; i++) JJ[i] = JRw[i];", "theta", 10),
    "Jr^-1 replaced by I": ("so3_jr_inv(r, Jri);", "for (int i = 0; i < 9; i++) Jri[i] = (i % 4 == 0);", "res", 10),
    "sign of the -dt R_p^T velocity column": ("put3(J, 3, 6, RpT, -dt);", "put3(J, 3, 6, RpT, dt);", "dt_g", 10),
    "E in place of E^T in the rotation rows": ("m3mul(Jri, ET, A);", "m3mul(Jri, E, A);", "phi", 10),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_of_imu_fails_a_named_case(tmp_path, mutation):
    """each mutation, applied to a copy of imu.cuh that only this build sees, fails its named case by at least the
    stated multiple of the tolerance"""
    old, new, case, margin = MUTATIONS[mutation]
    res = _host_errors(_build_shim(tmp_path, (old, new)), [case])
    print(f"IMU mutation '{mutation}' caught by {case}: {res[case]:.3g} x tolerance")
    assert res[case] >= margin, (mutation, res[case])
