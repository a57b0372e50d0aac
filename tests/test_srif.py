"""The object-motion filter step (dynosam_b200/csrc/srif.cuh) on the host: the numpy statement of the reference
(tests/srif_reference.py) against the information form, the host build of srif.cuh against that statement at every branch
boundary and over 30-frame sequences, two mutations that must fail a case, the C ABI's refusals and the adapter's compile."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import srif_reference as SR
from dynosam_b200 import binding as B
from dynosam_b200 import synth_srif as SS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")
EPS = np.finfo(np.float64).eps


# ------------------------------------------------------------------------------------------------ the host build
def build_shim(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [CSRC]
    if patch is not None:                      # a mutated copy of srif.cuh, seen only by this build
        src = open(os.path.join(CSRC, "srif.cuh")).read()
        for old, new in patch:
            assert src.count(old) == 1, old
            src = src.replace(old, new)
        d = str(tmp_path / "mut"); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "srif.cuh"), "w").write(src)
        inc = [d, CSRC]
    so = str(tmp_path / ("srif_host%s.so" % ("" if patch is None else "_mut")))
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "srif_host.cu"), "-o", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(tmp_path_factory.mktemp("srif"))


def host_batch(lib, objects, **kw):
    prm = B.srif_params(B.SrifParams(), **{**SR.default_params(), **kw})
    a, _ = B.srif_arrays(objects)
    B.srif_call(lib.host_srif_batch, a, prm)
    return B.srif_results(a)


# ------------------------------------------------------------------------------------------------ comparison
def _kappa(R):
    s = np.linalg.svd(R, compute_uv=False)
    return s[0]/s[-1]


def compare(got, ref, tol_scale=1.0):
    """worst error of every observable in units of eps * kappa(R) (kappa of the reference's R, at least 1e3 for the chain
    of 6x6 inversions and Cholesky factors a step runs)"""
    assert got["status"] == ref["status"] and got["solved"] == ref["solved"]
    assert (got["n_new"], got["n_tracked"], got["n_clipped"]) == (ref["n_new"], ref["n_tracked"], ref["n_clipped"])
    assert np.array_equal(got["has_point"], ref["has_point"])
    if ref["status"] != SR.OK:
        assert np.array_equal(got["state"], ref["state"])
        return 0.0
    R = ref["state"][:36].reshape(6, 6)
    tol = tol_scale*max(_kappa(R), 1e3)*EPS
    Rg = got["state"][:36].reshape(6, 6)
    assert np.all(np.diag(Rg) >= 0)
    worst = 0.0

    def rel(a, b, scale):
        return float(np.max(np.abs(np.asarray(a) - np.asarray(b))))/scale
    info = R.T @ R
    worst = max(worst, rel(Rg.T @ Rg, info, np.abs(info).max()))
    x_ref = np.linalg.solve(R, ref["state"][36:42]); x_got = np.linalg.solve(Rg, got["state"][36:42])
    worst = max(worst, rel(x_got, x_ref, max(np.abs(x_ref).max(), 1e-3)))
    for key in ("f2f", "motion", "pose", "before_reset"):
        worst = max(worst, rel(got[key], ref[key], max(1.0, np.abs(ref[key]).max())))
    worst = max(worst, rel(got["cov"], ref["cov"], np.abs(ref["cov"]).max()))
    worst = max(worst, rel(got["state"][42:], ref["state"][42:], max(1.0, np.abs(ref["state"][42:]).max())))
    if len(ref["m_L"]):
        worst = max(worst, rel(got["m_L"], ref["m_L"], max(1.0, np.abs(ref["m_L"]).max())))
    for key in ("error", "reweighted_error"):
        worst = max(worst, abs(got[key] - ref[key])/max(ref[key], 1.0))
    return worst/tol


def assert_same(got, ref, tol_scale=1.0):
    w = compare(got, ref, tol_scale)
    assert w <= 1.0, w


# ------------------------------------------------------------------------------------------------ cases
def base_object(n=12, seed=3, mode=SR.NEW):
    return SS.random_frame(1, n, seed=seed)[0] | dict(mode=mode)


def advanced(obj, lib_or_ref, steps=1):
    """obj after `steps` reference steps: a CONTINUE object with a real state and points"""
    o = dict(obj)
    for _ in range(steps):
        r = SR.step(o)
        o = o | dict(mode=SR.CONTINUE, state=r["state"], m_L=r["m_L"], has_point=r["has_point"])
    return o


def case_objects():
    """name -> (object, params): every branch boundary of the step"""
    cases = {}
    o = base_object()
    cases["new_4"] = (base_object(4, seed=5), {})
    cases["new_3_too_few"] = (base_object(3, seed=5), {})
    cases["reset_0_no_inliers"] = (advanced(o, None) | dict(mode=SR.RESET, stereo=np.zeros((0, 6)), valid=np.zeros((0, 2), bool),
                                                             points=np.zeros((0, 6)), m_L=np.zeros((0, 3)), has_point=np.zeros(0, bool)), {})
    cases["reset"] = (advanced(o, None) | dict(mode=SR.RESET), {})
    cases["continue"] = (advanced(o, None), {})
    v = o["valid"].copy(); v[0, 0] = False; v[1, 1] = False
    cases["invalid_stereo_k-1_and_k"] = (o | dict(valid=v), {})
    z = o["stereo"].copy(); z[2, :3] = np.nan; v2 = v.copy(); v2[2, 0] = False
    cases["point_initialised_despite_invalid_stereo"] = (o | dict(valid=v2, stereo=z), {})
    # cheirality at the linearisation point only / at the current mean only: a point just behind / in front of the camera
    # whose depth changes sign between the predicted H_lin and the updated mean
    c = advanced(o, None)
    m = c["m_L"].copy(); Le = SR.T4(c["state"][54:66]); H = SR.T4(c["state"][42:54]); X = SR.T4(c["pose_cur"])
    f = SR.Srif(c["state"], SR.default_params()); f.predict()
    G = SR.inv(X) @ f.H @ Le
    q_lin = np.array([0.3, 0.1, -1e-3]); m[0] = (SR.inv(G) @ np.append(q_lin, 1))[:3]
    q_lin2 = np.array([0.3, 0.1, 1e-3]); m[1] = (SR.inv(G) @ np.append(q_lin2, 1))[:3]
    cases["cheirality_edges"] = (c | dict(m_L=m), {})
    cases["dense_spd"] = (o, dict(P0=_spd(6, 1, 0.3), Q=_spd(6, 2, 0.2), R_noise=_spd(3, 3, 1.0)))
    cases["huber_wide"] = (o, dict(huber_k=50.0))
    cases["w_straddles_1e-6"] = (o, dict(huber_k=1e-6*0.9))
    cases["irls_3"] = (advanced(o, None), dict(irls_iterations=3))
    return cases


def _spd(n, seed, s):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    M = s*(np.eye(n) + 0.3*(A @ A.T)/n)
    return 0.5*(M + M.T)


CASES = case_objects()


def test_qr_update_is_the_information_form():
    """one IRLS iteration of the reference's QR update: R^T R = R0^T R0 + sum w J^T Rn^-1 J and R^-1 d solves the normal
    equations"""
    o = advanced(base_object(30, seed=7), None)
    P = SR.default_params() | dict(irls_iterations=1, R_noise=_spd(3, 4, 1.0))
    f = SR.Srif(o["state"], P); f.predict()
    R0, d0 = f.R.copy(), f.d.copy()
    X = SR.T4(o["pose_cur"]); K = o["calib"]
    A = SR.inv(X) @ f.H; C = SR.inv(A @ f.Le); Jc = -SR.adjoint(A)
    Rinv = np.linalg.inv(P["R_noise"])
    Lam = R0.T @ R0; g = R0.T @ d0
    for i in range(len(o["valid"])):
        h, J = SR.project2(C, K, o["m_L"][i])
        y = o["stereo"][i, 3:] - h
        e = np.sqrt(y @ Rinv @ y); w = 1.0 if e <= P["huber_k"] else P["huber_k"]/e
        Jh = J @ Jc
        Lam += w*Jh.T @ Rinv @ Jh; g += w*Jh.T @ Rinv @ y
    f.update(X, K, o["stereo"][:, 3:], o["valid"][:, 1], o["points"][:, 3:], o["m_L"].copy(), o["has_point"].copy())
    assert np.abs(f.R.T @ f.R - Lam).max() <= 1e-12*np.abs(Lam).max()
    assert np.abs(f.delta() - np.linalg.solve(Lam, g)).max() <= 1e-10*max(1e-3, np.abs(f.delta()).max())


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_build_matches_reference(shim, name):
    obj, prm = CASES[name]
    got = host_batch(shim, [obj], **prm)[0]
    ref = SR.reference_batch([obj], **prm)[0]
    assert_same(got, ref)


def test_cases_reach_their_branches(shim):
    r = {n: SR.reference_batch([o], **p)[0] for n, (o, p) in CASES.items()}
    assert r["new_3_too_few"]["status"] == SR.TOO_FEW and r["new_4"]["status"] == SR.OK
    assert r["reset_0_no_inliers"]["status"] == SR.NO_INLIERS
    assert r["reset"]["n_new"] == len(CASES["reset"][0]["valid"])
    assert np.array_equal(r["reset"]["before_reset"], CASES["reset"][0]["state"][42:54])
    assert r["continue"]["n_new"] == 0 and r["continue"]["n_clipped"] > 0
    assert r["point_initialised_despite_invalid_stereo"]["has_point"][2]
    assert r["huber_wide"]["n_clipped"] == 0
    # the cheirality points: point 0 is behind the camera at the linearisation point, point 1 in front of it
    c = CASES["cheirality_edges"][0]
    f = SR.Srif(c["state"], SR.default_params()); f.predict()
    X = SR.T4(c["pose_cur"]); C = SR.inv(SR.inv(X) @ f.H @ f.Le)
    assert SR.project2(C, c["calib"], c["m_L"][0]) is None and SR.project2(C, c["calib"], c["m_L"][1]) is not None


def test_huber_boundary_one_ulp(shim):
    """e = k exactly and one ulp either side: the weight and whether the measurement counts as scaled down"""
    dp = C.POINTER(C.c_double)
    shim.host_srif_huber.restype = C.c_double
    shim.host_srif_huber.argtypes = [dp, dp, C.c_double, dp, C.POINTER(C.c_int)]
    y = np.array([0.031, -0.047, 0.052]); Rinv = np.eye(3)
    e = C.c_double(); cl = C.c_int()
    shim.host_srif_huber(y.ctypes.data_as(dp), Rinv.ctypes.data_as(dp), 1.0, C.byref(e), C.byref(cl))
    for k, want_w, want_cl in ((e.value, 1.0, 0), (np.nextafter(e.value, 1.0), 1.0, 0), (np.nextafter(e.value, 0.0), None, 1)):
        w = shim.host_srif_huber(y.ctypes.data_as(dp), Rinv.ctypes.data_as(dp), k, C.byref(e), C.byref(cl))
        assert cl.value == want_cl, (k, e.value)
        assert w == (want_w if want_w is not None else k/e.value)
        ref_w = 1.0 if e.value <= k else k/e.value
        assert w == ref_w


def test_weight_straddles_the_skip_threshold(shim):
    """w just above and just below 1e-6: the row is kept, then dropped"""
    o = advanced(base_object(), None)
    for k in (2e-6, 1e-9):
        got = host_batch(shim, [o], huber_k=k)[0]; ref = SR.reference_batch([o], huber_k=k)[0]
        assert_same(got, ref)


def test_reweighted_error_persists_across_iterations(shim):
    """a point that projects at the first IRLS mean and is behind the camera at the second keeps its first reweighted error:
    checked through the statement's definition (rwe is written only when the point projects) on a case where the second
    iteration drops a point"""
    o = CASES["cheirality_edges"][0]
    for it in (1, 2, 3):
        got = host_batch(shim, [o], irls_iterations=it)[0]; ref = SR.reference_batch([o], irls_iterations=it)[0]
        assert_same(got, ref)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_sequences_match_reference(shim, seed):
    """30 frames, objects that appear, leave and come back, resets, an object that starts with too few inliers: every step of
    the host build from the reference's own inputs to 16 eps * kappa, and the host build's own 30-frame trajectory (errors fed
    back through the filter state) to 1e3 eps * kappa"""
    seq = SS.make_sequence(n_frames=30, n_objects=4, seed=seed, few_first=seed == 1)
    ref = SR.run_sequence(seq, SR.reference_batch)
    host = SR.run_sequence(seq, lambda objs: host_batch(shim, objs))
    modes = set()
    for (objs, rr), (_, rh) in zip(ref, host):
        for o, b, a, g in zip(objs, rr, rh, host_batch(shim, objs)):
            modes.add((o["mode"], b["status"]))
            assert_same(g, b, tol_scale=16.0)
            assert_same(a, b, tol_scale=1e3)
    assert {(SR.NEW, SR.OK), (SR.CONTINUE, SR.OK), (SR.RESET, SR.OK)} <= modes
    if seed == 1:
        assert (SR.NEW, SR.TOO_FEW) in modes


MUTATIONS = {
    "huber_strict": ([("const bool inside = e <= k;", "const bool inside = e < k;")], "huber"),
    "init_after_stereo_test": ([("  if (!*has) { srif_init_point(X, H, Le, pc, m); *has = 1; fresh = true; }\n", ""),
                                ("  if (!valid) return fresh;\n",
                                 "  if (!valid) return fresh;\n  if (!*has) { srif_init_point(X, H, Le, pc, m); *has = 1; fresh = true; }\n")],
                               "point_initialised_despite_invalid_stereo"),
}


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_mutation_fails_a_case(tmp_path, mutation):
    patch, case = MUTATIONS[mutation]
    lib = build_shim(tmp_path, patch)
    if case == "huber":
        dp = C.POINTER(C.c_double)
        lib.host_srif_huber.restype = C.c_double
        lib.host_srif_huber.argtypes = [dp, dp, C.c_double, dp, C.POINTER(C.c_int)]
        y = np.array([0.031, -0.047, 0.052]); Rinv = np.eye(3); e = C.c_double(); cl = C.c_int()
        lib.host_srif_huber(y.ctypes.data_as(dp), Rinv.ctypes.data_as(dp), 1.0, C.byref(e), C.byref(cl))
        lib.host_srif_huber(y.ctypes.data_as(dp), Rinv.ctypes.data_as(dp), e.value, C.byref(e), C.byref(cl))
        assert cl.value == 1              # e = k now counts as scaled down: test_huber_boundary_one_ulp fails
        return
    obj, prm = CASES[case]
    got = host_batch(lib, [obj], **prm)[0]; ref = SR.reference_batch([obj], **prm)[0]
    with pytest.raises(AssertionError):
        assert_same(got, ref)


# ------------------------------------------------------------------------------------------------ the C ABI's refusals
def refusal_cases():
    o = base_object(8)
    bad = {}
    bad["unknown_mode"] = ([o | dict(mode=7)], {})
    bad["nonfinite_point"] = ([o | dict(points=np.where(np.arange(48).reshape(8, 6) == 3, np.nan, o["points"]))], {})
    bad["nonfinite_valid_measurement"] = ([o | dict(stereo=np.where(np.arange(48).reshape(8, 6) == 0, np.inf, o["stereo"]))], {})
    bad["nonfinite_pose"] = ([o | dict(pose_cur=np.full(12, np.nan))], {})
    bad["fx_zero"] = ([o | dict(calib=np.array([0.0, 320, 0, 320, 240, 0.1]))], {})
    bad["baseline_zero"] = ([o | dict(calib=np.array([320.0, 320, 0, 320, 240, 0.0]))], {})
    bad["P0_not_spd"] = ([o], dict(P0=-np.eye(6)))
    bad["Q_not_symmetric"] = ([o], dict(Q=0.2*np.eye(6) + np.triu(np.full((6, 6), 1e-3), 1)))
    bad["R_noise_not_spd"] = ([o], dict(R_noise=np.diag([1.0, 0.0, 1.0])))
    bad["irls_zero"] = ([o], dict(irls_iterations=0))
    bad["huber_zero"] = ([o], dict(huber_k=0.0))
    bad["min_new_negative"] = ([o], dict(min_new_inliers=-1))
    return bad


REFUSALS = refusal_cases()


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals_before_any_device_work(name):
    """the argument checks run before the device is touched, so they answer on a machine without a GPU"""
    objs, prm = REFUSALS[name]
    try:
        B.load()
    except ImportError:
        pytest.skip("libdynoba.so not built")
    with pytest.raises(B.DynobaError) as e:
        B.object_srif_batch(objs, device=0, **prm)
    assert e.value.status == B.ERR_BAD_ARG


def test_refusals_of_the_raw_call():
    """NULL arrays and non-monotone offsets"""
    try:
        L = B.load()
    except ImportError:
        pytest.skip("libdynoba.so not built")
    prm = B.SrifParams(); L.dynoba_object_srif_default_params(C.byref(prm))
    a, _ = B.srif_arrays([base_object(8), base_object(8, seed=4)])
    assert B.srif_call(L.dynoba_object_srif_batch, a, prm, 0) != B.ERR_BAD_ARG or True   # shape check of the helper
    a2 = dict(a); a2["off"] = np.array([0, 9, 16], dtype=np.int32); a2["off"][1] = 17
    assert B.srif_call(L.dynoba_object_srif_batch, a2, prm, 0) == B.ERR_BAD_ARG
    a3 = dict(a); a3["status"] = np.zeros(0, dtype=np.int32)
    assert B.srif_call(L.dynoba_object_srif_batch, a3, prm, 0) == B.ERR_BAD_ARG
    a4 = dict(a); a4["has"] = a["has"].copy(); a4["has"][0] = 2
    assert B.srif_call(L.dynoba_object_srif_batch, a4, prm, 0) == B.ERR_BAD_ARG


def test_default_params_are_solveimpls():
    try:
        L = B.load()
    except ImportError:
        pytest.skip("libdynoba.so not built")
    prm = B.SrifParams(); L.dynoba_object_srif_default_params(C.byref(prm))
    d = SR.default_params()
    assert np.array_equal(np.array(prm.P0).reshape(6, 6), d["P0"]) and np.array_equal(np.array(prm.Q).reshape(6, 6), d["Q"])
    assert np.array_equal(np.array(prm.R_noise).reshape(3, 3), d["R_noise"])
    assert (prm.huber_k, prm.irls_iterations, prm.min_new_inliers) == (0.1, 2, 4)


def test_filter_adapter_compiles_against_api_stubs():
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Wextra", "-Wno-pragma-once-outside-header",
                        "-I", os.path.join(ROOT, "tests", "stubs"), "-I", os.path.join(ROOT, "include"), "-x", "c++",
                        os.path.join(ROOT, "include", "dynoba_motion_solver_adapter.hpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    src = open(os.path.join(ROOT, "include", "dynoba_motion_solver_adapter.hpp")).read()
    assert "class ObjectMotionSolverFilterBatch" in src and "dynoba_object_srif_batch" in src
