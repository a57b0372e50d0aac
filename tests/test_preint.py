"""Combined IMU preintegration on the CPU: the case list of tests/preint_cases.py reaches every boundary it names, the
50-digit reference (tests/preint_reference.py) is pinned by pieces that do not depend on it, `preint.cuh` compiled for
the host equals the reference case by case within the a-priori bound, and mutations of `preint.cuh` each fail a named
case by the stated factor."""
import ctypes as C
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest
from mpmath import mp, mpf

import imu_lie_reference as IL
import lie_reference as LR
import preint_cases as PC
import preint_reference as PR
from dynosam_b200 import synth_imu
from dynosam_b200.binding import ImuParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")
EPS = PC.EPS
CASES = PC.cases()


@functools.lru_cache(maxsize=None)
def reference(name):
    c = CASES[name]
    z, S, R = PR.preintegrate(PR.params(c.P), c.stamps, c.acc_gyr, c.bh)
    return z, S, R


def _f(M, n=15):
    return np.array([[float(M[i, j]) for j in range(n)] for i in range(n)])


# ------------------------------------------------------------------------------------------------ the case list
def test_cases_reach_every_boundary():
    seen = set()
    for name, c in CASES.items():
        _, _, R = reference(name)
        b = PC.boundaries(c, Sigma_pd=R is not None)
        assert set(c.hits) <= b, (name, set(c.hits) - b)
        seen |= b
    missing = set(PC.REQUIRED) - seen
    assert not missing, sorted(missing)


# ------------------------------------------------------------------------------------------------ the host build
def build_shim(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [CSRC]
    if patch is not None:                      # a mutated copy of preint.cuh, seen only by this build
        src = open(os.path.join(CSRC, "preint.cuh")).read()
        for old, new in patch:
            assert src.count(old) == 1, old
            src = src.replace(old, new)
        d = str(tmp_path / "mut"); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "preint.cuh"), "w").write(src.replace(
            '#include "../../include/dynoba.h"', '#include "%s"' % os.path.join(ROOT, "include", "dynoba.h")))
        inc = [d, CSRC]
    so = str(tmp_path / ("preint_host%s.so" % ("" if patch is None else "_mut")))
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "preint_host.cu"), "-o", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def host_batch(lib, P, items):
    """items: [(stamps, acc_gyr, bh)] -> dict(record, cov, sqrt_info, status) of host_preint_batch"""
    n = len(items)
    off = np.zeros(n + 1, np.int32); off[1:] = np.cumsum([len(s) for s, _, _ in items])
    st = np.ascontiguousarray(np.concatenate([s for s, _, _ in items]))
    ag = np.ascontiguousarray(np.concatenate([a for _, a, _ in items]))
    bh = np.ascontiguousarray(np.stack([np.zeros(6) if b is None else b for _, _, b in items]))
    rec = np.zeros((n, 70)); cov = np.zeros((n, 15, 15)); R = np.zeros((n, 15, 15)); status = np.zeros(n, np.int32)
    lib.host_preint_batch(C.byref(P), n, off.ctypes.data_as(C.POINTER(C.c_int32)), _dp(st), _dp(ag), _dp(bh), _dp(rec),
                          _dp(cov), _dp(R), status.ctypes.data_as(C.POINTER(C.c_int32)))
    return dict(record=rec, cov=cov, sqrt_info=R, status=status)


BLOCKS = [("dR", 0, 9), ("dp", 9, 12), ("dv", 12, 15), ("dt", 15, 16), ("bh", 16, 22), ("JRw", 22, 31), ("JPa", 31, 40),
          ("JPw", 40, 49), ("JVa", 49, 58), ("JVw", 58, 67), ("g", 67, 70)]


def errors(name, rec, cov, R, status):
    """{quantity: worst |device - reference| over its a-priori tolerance} of one case"""
    c = CASES[name]
    z, S, Rr = reference(name)
    n = len(c.stamps) - 1
    zf = np.array([float(x) for x in z]); Sf = _f(S)
    out = {}
    for b, lo, hi in BLOCKS:
        tol = 16*EPS*(n + 1)*max(1.0, np.abs(zf[lo:hi]).max())
        out["rec_" + b] = np.abs(rec[lo:hi] - zf[lo:hi]).max()/tol
    d = np.sqrt(np.abs(np.diag(Sf)))
    out["cov"] = (np.abs(cov - Sf)/(32*EPS*(n + 1)*np.maximum(np.outer(d, d), 1e-300))).max()
    out["status"] = 0.0 if int(status) == (1 if Rr is None else 0) else np.inf
    if Rr is None:
        out["R"] = 0.0 if not np.any(R) else np.inf
    else:
        Rf = _f(Rr)
        Sn = Sf/np.outer(d, d)
        kappa = np.linalg.cond(Sn)
        out["R"] = np.abs(R - Rf).max()/(32*EPS*(n + 15)*kappa*np.abs(Rf).max())
    return out


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(tmp_path_factory.mktemp("preint"))


def host_errors(lib, names):
    res = {}
    for name in names:
        c = CASES[name]
        o = host_batch(lib, c.P, [(c.stamps, c.acc_gyr, c.bh)])
        res[name] = errors(name, o["record"][0], o["cov"][0], o["sqrt_info"][0], o["status"][0])
    return res


def test_host_build_equals_the_reference(shim):
    res = host_errors(shim, list(CASES))
    worst = max(((n, q, v) for n, r in res.items() for q, v in r.items()), key=lambda t: t[2])
    print(f"preint host worst: {worst[0]} {worst[1]} {worst[2]:.3g} of the tolerance")
    bad = {(n, q): v for n, r in res.items() for q, v in r.items() if not v <= 1.0}
    assert not bad, bad


def test_host_batch_is_the_intervals_alone(shim):
    """a batch of every case returns each case's bits"""
    names = list(CASES)
    by = {}
    for P in {id(CASES[n].P): CASES[n].P for n in names}.values():
        group = [n for n in names if CASES[n].P is P]
        o = host_batch(shim, P, [(CASES[n].stamps, CASES[n].acc_gyr, CASES[n].bh) for n in group])
        for i, n in enumerate(group):
            by[n] = {k: v[i] for k, v in o.items()}
    for n in names:
        c = CASES[n]
        a = host_batch(shim, c.P, [(c.stamps, c.acc_gyr, c.bh)])
        for k in a:
            assert np.array_equal(a[k][0], by[n][k]), (n, k)


# ------------------------------------------------------------------------------------------------ pins of the reference
def _n_step_state(P, stamps, ag, bh):
    st = PR.start(bh)
    ts = PR._m(stamps)
    for i in range(len(ts) - 1):
        st, _ = PR.step(P, st, PR._m(ag[i, :3]), PR._m(ag[i, 3:]), ts[i + 1] - ts[i])
    return st


def _nav_only(P, stamps, ag, bh):
    R, p, v = list(LR.I3), [mpf(0)]*3, [mpf(0)]*3
    ts = PR._m(stamps)
    for i in range(len(ts) - 1):
        R, p, v = PR.nav(P, R, p, v, PR._m(ag[i, :3]), PR._m(ag[i, 3:]), bh, ts[i + 1] - ts[i])
    return R, p, v


@pytest.mark.parametrize("name", ["rot_03", "bias_hat", "dt_mixed", "frontend_identity"])
def test_bias_jacobians_are_derivatives_of_the_n_step_map(name):
    """(a): the recursion's five bias Jacobians equal 50-digit central differences of the n-step map w.r.t. biasHat
    (in the chart at the final state: R Exp(dR), p + dp, v + dv), for records without a rotated sensor frame, to 1e-25
    (the 50-digit rounding of a difference quotient with step 1e-20)"""
    c = CASES[name]; P = PR.params(c.P)
    bh = PR._m(np.zeros(6) if c.bh is None else c.bh)
    st = _n_step_state(P, c.stamps, c.acc_gyr, bh)
    R0, p0, v0 = st["R"], st["p"], st["v"]
    h = mpf("1e-20")
    for j in range(6):
        res = []
        for s in (h, -h):
            b = list(bh); b[j] += s
            R, p, v = _nav_only(P, c.stamps, c.acc_gyr, b)
            res.append((LR.log_so3(LR.mul3(LR.tr3(R0), R)), [x - y for x, y in zip(p, p0)], [x - y for x, y in zip(v, v0)]))
        dR = [(x - y)/(2*h) for x, y in zip(res[0][0], res[1][0])]
        dp = [(x - y)/(2*h) for x, y in zip(res[0][1], res[1][1])]
        dv = [(x - y)/(2*h) for x, y in zip(res[0][2], res[1][2])]
        k = j % 3
        if j < 3:
            assert max(abs(dp[i] - st["JPa"][3*i + k]) for i in range(3)) < mpf("1e-25")
            assert max(abs(dv[i] - st["JVa"][3*i + k]) for i in range(3)) < mpf("1e-25")
            assert max(abs(x) for x in dR) < mpf("1e-25")
        else:
            assert max(abs(dR[i] - st["JRw"][3*i + k]) for i in range(3)) < mpf("1e-25")
            assert max(abs(dp[i] - st["JPw"][3*i + k]) for i in range(3)) < mpf("1e-25")
            assert max(abs(dv[i] - st["JVw"][3*i + k]) for i in range(3)) < mpf("1e-25")


@pytest.mark.parametrize("name", ["rot_03", "lever_arm", "frontend_viode", "jr_below", "rot_near_pi"])
def test_host_step_jacobians_equal_differences(shim, name):
    """(b): A, B and C of one step of the host build equal the reference's 50-digit central differences of the step in
    NavState's chart, sensor-pose branch included, to 64 eps of the largest entry"""
    c = CASES[name]; P = PR.params(c.P)
    bh = np.zeros(6) if c.bh is None else c.bh
    rng = np.random.default_rng(3)
    z = synth_imu.preintegrate(rng.normal(0, 3, (2, 3)), rng.normal(0, 0.5, (2, 3)), 0.01, bias_hat=bh)
    dt = float(c.stamps[1] - c.stamps[0])
    zo = np.zeros(70); A = np.zeros(81); B = np.zeros(27); Cm = np.zeros(27); F9 = np.zeros(135); Q = np.zeros(225)
    acc = np.ascontiguousarray(c.acc_gyr[0, :3]); om = np.ascontiguousarray(c.acc_gyr[0, 3:])
    shim.host_preint_step(C.byref(c.P), _dp(z), _dp(acc), _dp(om), C.c_double(dt), _dp(zo), _dp(A), _dp(B), _dp(Cm), _dp(F9), _dp(Q))
    zm = PR._m(z)
    Ar, Br, Cr = PR.step_jacobians(P, zm[0:9], zm[9:12], zm[12:15], PR._m(acc), PR._m(om), PR._m(bh), mpf(dt))
    for M, Mr, w in ((A, Ar, 9), (B, Br, 3), (Cm, Cr, 3)):
        Mf = np.array([[float(x) for x in row] for row in Mr])
        assert np.abs(M.reshape(9, w) - Mf).max() <= 64*EPS*max(1.0, np.abs(Mf).max()), (name, w, np.abs(M.reshape(9, w) - Mf).max())
    # and the [GTSAM-ext] F rows and Q of the host equal the reference's statements at the same A, B, C
    Fr = PR.F_of(Ar, Br, Cr)
    assert np.abs(F9.reshape(9, 15) - np.array([[float(x) for x in Fr[i]] for i in range(9)])).max() <= 64*EPS*max(1.0, np.abs(F9).max())
    Qr = _f(PR.injected_noise(P, Br, Cr, mpf(dt)))
    assert np.abs(Q.reshape(15, 15) - Qr).max() <= 64*EPS*np.abs(Qr).max()


def test_sigma_is_the_sum_of_propagated_injections():
    """(c): after n steps Sigma = sum_k Phi_{n<-k} Q_k Phi_{n<-k}^T, each Phi the product of the steps' F after k, with F
    formed from A, B, C differentiated from the step map; this pins the F recursion apart from the injected Q_k"""
    c = CASES["lever_arm"]; P = PR.params(c.P)
    bh = PR._m(c.bh)
    st = PR.start(bh); Fs, Qs = [], []
    ts = PR._m(c.stamps)
    for i in range(len(ts) - 1):
        dt = ts[i + 1] - ts[i]
        n, (A, B, Cm) = PR.step(P, st, PR._m(c.acc_gyr[i, :3]), PR._m(c.acc_gyr[i, 3:]), dt)
        Fs.append(mp.matrix(PR.F_of(A, B, Cm))); Qs.append(PR.injected_noise(P, B, Cm, dt)); st = n
    S = mp.matrix(15, 15)
    for k in range(len(Qs)):
        Phi = mp.eye(15)
        for F in Fs[k + 1:]:
            Phi = F*Phi
        S += Phi*Qs[k]*Phi.T
    assert mp.mnorm(S - st["S"], 1) <= mpf("1e-35")*mp.mnorm(S, 1)


def test_predict_zeroes_imu_eval(shim, tmp_path):
    """(d): imu_eval (imu.cuh's host build) gives a zero residual, to rounding, at (X_j, V_j) = predict(X_i, V_i, b_i),
    and the host predict equals the reference's"""
    import test_imu_cases as TIC
    call = TIC._build_shim(tmp_path)
    rng = np.random.default_rng(4)
    for name in ("rot_03", "lever_arm", "frontend_viode", "bias_hat"):
        c = CASES[name]
        o = host_batch(shim, c.P, [(c.stamps, c.acc_gyr, c.bh)])
        z = o["record"][0]
        R0 = PC._rot(rng.normal(size=3), 1.1)
        Xi = np.concatenate([R0.reshape(9), rng.normal(0, 5, 3)]); vi = rng.normal(0, 2, 3)
        bi = (np.zeros(6) if c.bh is None else c.bh) + rng.normal(0, 1e-3, 6)
        Xj = np.zeros(12); vj = np.zeros(3)
        shim.host_preint_predict(_dp(z), _dp(Xi), _dp(vi), _dp(bi), _dp(Xj), _dp(vj))
        Xr, vr = PR.predict(z, PR._m(Xi), PR._m(vi), PR._m(bi))
        scale = 1.0 + np.abs(Xi).max() + np.abs(vi).max()*z[15] + 10*z[15]**2
        assert np.abs(Xj - np.array([float(x) for x in Xr])).max() <= 64*EPS*scale
        assert np.abs(vj - np.array([float(x) for x in vr])).max() <= 64*EPS*(scale + np.abs(vi).max())
        r = call("host_imu_residual", Xi, vi, Xj, vj, bi, bi, z, out=15)
        assert np.abs(r).max() <= 256*EPS*scale, (name, np.abs(r).max())


def test_residual_falls_with_dt():
    """(e): on noise-free synth_imu.imu_samples along a rotating trajectory the COMBINED_IMU15 residual at the true states
    falls in proportion to the sample interval (Euler integration): about half when dt halves -- gravity's sign and the
    frames checked end to end (reference record, tests/imu_lie_reference.py residual)"""
    from dynosam_b200 import synth
    xi = np.array([0.05, -0.08, 0.1, 0.3, 0.1, -0.2])
    R0 = PC._rot((1, 1, 0), 0.4)
    D = PC.gtsam_defaults(synth_imu.GRAVITY)
    P = PR.params(D)
    w, v = synth_imu.body_rates(xi)
    X0 = LR.pose(np.concatenate([R0.reshape(9), [1.0, 2.0, 3.0]]))
    X1 = LR.retract(X0, LR.vec(xi))                    # the true pose after one frame: X0 Exp(xi)
    errs = []
    for ns in (10, 20, 40):
        dt = synth_imu.FRAME_DT/ns
        acc, gyr = synth_imu.imu_samples(R0, xi, ns + 1, dt)
        z, _, _ = PR.preintegrate(P, np.arange(ns + 1)*dt, np.concatenate([acc, gyr], 1))
        vi = LR.mv3(LR.vec(R0.reshape(9)), LR.vec(v))
        vj = LR.mv3(X1[0], LR.vec(v))
        r = IL.residual(X0, vi, X1, vj, [mpf(0)]*6, [mpf(0)]*6, [float(x) for x in z])
        errs.append(float(max(abs(x) for x in r[:9])))
    assert errs[0] > 1e-9, errs
    for a, b in zip(errs, errs[1:]):
        assert 0.4 <= b/a <= 0.6, errs


def test_sqrt_info_is_numpy_cholesky(shim):
    """(f): R^T R Sigma = I and R equals numpy's cholesky(inv(Sigma)).T"""
    for name in ("rot_03", "frontend_viode", "long_2000", "lever_arm"):
        c = CASES[name]
        o = host_batch(shim, c.P, [(c.stamps, c.acc_gyr, c.bh)])
        S, R = o["cov"][0], o["sqrt_info"][0]
        d = np.sqrt(np.diag(S)); kappa = np.linalg.cond(S/np.outer(d, d))
        assert np.allclose(np.tril(R, -1), 0) and np.all(np.diag(R) > 0)
        M = R.T@R@S
        assert np.abs(M - np.eye(15)).max() <= 1e3*EPS*kappa, (name, np.abs(M - np.eye(15)).max(), kappa)
        Rn = np.linalg.cholesky(np.linalg.inv(S)).T
        assert np.abs(R - Rn).max() <= 1e3*EPS*kappa*np.abs(Rn).max(), name


def test_record_equals_synth_imu_preintegrate(shim):
    """(g): without a sensor pose the record equals synth_imu.preintegrate (uniform dt) within rounding"""
    rng = np.random.default_rng(5)
    D = PC.gtsam_defaults(synth_imu.GRAVITY)
    for n, dt in ((10, 0.01), (200, 0.005)):
        acc = rng.normal(0, 3, (n + 1, 3)); gyr = rng.normal(0, 0.5, (n + 1, 3)); bh = rng.normal(0, 0.01, 6)
        o = host_batch(shim, D, [(np.arange(n + 1)*dt, np.concatenate([acc, gyr], 1), bh)])
        z = synth_imu.preintegrate(acc[:n], gyr[:n], dt, bias_hat=bh)
        assert np.abs(o["record"][0] - z).max() <= 64*n*EPS*max(1.0, np.abs(z).max())


def test_default_params_are_gtsams():
    from dynosam_b200 import binding
    p = ImuParams(); binding.load().dynoba_imu_default_params(C.byref(p))
    q = PC.gtsam_defaults((0, 0, 0))
    for k, _ in ImuParams._fields_:
        a, b = getattr(p, k), getattr(q, k)
        assert (list(a) == list(b)) if k != "has_body_P_sensor" else a == b == 0, k


def test_frontend_params_swap_bias_covariances():
    """binding.imu_frontend_params reproduces ImuFrontend.cc:106-109 literally: biasAccCovariance from the gyroscope's
    random walk, biasOmegaCovariance from the accelerometer's"""
    from dynosam_b200 import binding
    p = binding.imu_frontend_params((0, 9.8, 0), 0.2, 0.05, 0.02, 4e-5, 1e-3)
    assert p.bias_acc_cov[0] == 4e-5**2 and p.bias_omega_cov[0] == 0.02**2
    assert p.accelerometer_cov[0] == 0.2**2 and p.gyroscope_cov[0] == 0.05**2 and p.integration_cov[0] == 1e-3**2
    assert p.has_body_P_sensor == 1 and list(p.body_P_sensor) == list(np.eye(3).reshape(9)) + [0.0]*3
    q = PC.frontend((0, 9.8, 0), 0.2, 0.05, 0.02, 4e-5, 1e-3, np.eye(4))
    for k, _ in ImuParams._fields_:
        a, b = getattr(p, k), getattr(q, k)
        assert (list(a) == list(b)) if k != "has_body_P_sensor" else a == b, k


def test_refusals():
    """dynoba_imu_preintegrate_batch refuses bad input before any device work (these run without a GPU)"""
    from dynosam_b200 import binding
    P = PC.gtsam_defaults((0, 0, -9.81))
    ag = np.zeros((3, 6))
    for stamps, agl in (([[0.0]], [ag[:1]]), ([[0.0, 0.0]], [ag[:2]]), ([[0.0, -0.1]], [ag[:2]]),
                        ([[0.0, np.nan]], [ag[:2]]), ([[0.0, 0.1]], [np.full((2, 6), np.inf)])):
        with pytest.raises(binding.DynobaError) as e:
            binding.imu_preintegrate_batch(P, stamps, agl)
        assert e.value.status == binding.ERR_BAD_ARG
    Q = PC.gtsam_defaults((0, 0, np.nan))
    with pytest.raises(binding.DynobaError) as e:
        binding.imu_preintegrate_batch(Q, [[0.0, 0.1]], [ag[:2]])
    assert e.value.status == binding.ERR_BAD_ARG
    Q = PC.gtsam_defaults((0, 0, -9.81)); Q.has_body_P_sensor = 1; Q.body_P_sensor[0] = 2.0     # not a rotation
    with pytest.raises(binding.DynobaError) as e:
        binding.imu_preintegrate_batch(Q, [[0.0, 0.1]], [ag[:2]])
    assert e.value.status == binding.ERR_BAD_ARG
    r = binding.imu_preintegrate_batch(P, [], [])
    assert r["record"].shape == (0, 70)


# each mutation of preint.cuh, applied to a copy only its build sees, fails the named case by at least the factor given
MUTATIONS = {
    "Jacobian updates after the rotation update": ([
        ("  // bias Jacobians first: they use the rotation before this step\n",
         "  double Rsave[9]; for (int i = 0; i < 9; i++) Rsave[i] = s.R[i];\n  m3mul(Rsave, incR, s.R);\n"),
        ("  // NavState::update\n", "  for (int i = 0; i < 9; i++) s.R[i] = Rsave[i];\n")], "rot_03", 100),
    "new rotation in D_acc_R": ([("skew3(a, Sa); m3mul(s.R, Sa, T9);",
                                  "skew3(a, Sa); { double Rn1[9]; m3mul(s.R, incR, Rn1); m3mul(Rn1, Sa, T9); }")], "rot_03", 100),
    "C *= D_correctedOmega_omega dropped": ([("m3mul(C, Dww, t); for (int i = 0; i < 9; i++) C[i] = t[i];", "")], "frontend_viode", 100),
    "dt scaling dropped from the integration covariance": ([("t[i] += u[i] + dt*P.integration_cov[i];",
                                                            "t[i] += u[i] + P.integration_cov[i];")], "rot_03", 100),
    "lever-arm term dropped": ([("for (int k = 0; k < 3; k++) a[k] -= WWa[k];", "")], "lever_arm", 100),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_of_preint_fails_a_named_case(tmp_path, mutation):
    patch, case, factor = MUTATIONS[mutation]
    lib = build_shim(tmp_path, patch)
    res = host_errors(lib, [case])[case]
    worst = max(res.values())
    print(f"preint mutation '{mutation}' caught by {case}: {worst:.3g} x tolerance")
    assert worst >= factor, (mutation, res)
