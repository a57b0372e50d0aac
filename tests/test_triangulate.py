"""The triangulation of dynosam_b200/csrc/triangulate.cuh on the host: its host build against the 50-digit statement of
tests/triangulation_reference.py at every branch edge (two cameras, left-only cameras, the rank test around 1.0, points
going to infinity, depths of either sign next to zero, the reprojection norm around 3.0), against cv2.triangulatePoints on
two-camera problems, and two mutations that must fail a case."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import triangulation_reference as TR
from dynosam_b200 import binding as B
from dynosam_b200 import lie

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")
K6 = np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372])
K5 = K6[:5]


def build_shim(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [CSRC]
    if patch is not None:                      # a mutated copy of triangulate.cuh, seen only by this build
        src = open(os.path.join(CSRC, "triangulate.cuh")).read()
        for old, new in patch:
            assert src.count(old) == 1, old
            src = src.replace(old, new)
        d = str(tmp_path / ("mut%d" % abs(hash(str(patch))))); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "triangulate.cuh"), "w").write(src)
        inc = [d, CSRC]
    so = str(tmp_path / ("triangulate_host%s.so" % ("" if patch is None else "_mut%d" % abs(hash(str(patch))))))   # dlopen caches by path
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "triangulate_host.cu"), "-o", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(tmp_path_factory.mktemp("tri"))


def host(lib, problems, rank_tol=1.0, thr=3.0):
    a = B.triangulate_arrays(problems)
    B.triangulate_call(lib.host_triangulate_batch, a, rank_tol, thr)
    return a


# ------------------------------------------------------------------------------------------------ problem makers
def camera(yaw=0.0, t=(0.0, 0.0, 0.0), pitch=0.0):
    return lie.pack(lie.ypr(yaw, pitch, 0.0)[None], np.asarray(t, np.float64)[None])[0]


def project(X, p, K=K5):
    q = lie.transform_to(X[None], np.asarray(p, np.float64)[None])[0]
    x, y = q[0]/q[2], q[1]/q[2]
    return np.array([K[0]*x + K[2]*y + K[3], K[1]*y + K[4]])


def problem(cams, p, noise=0.0, seed=0, K=K5):
    rng = np.random.default_rng(seed)
    kp = np.array([project(X, p, K) for X in cams]) + rng.normal(0, 1, (len(cams), 2))*noise
    return dict(poses=np.array(cams), kp=kp, calib=np.asarray(K, np.float64))


def stereo_cams(n, step=1.0, seed=0):
    """n stereo frames of a forward-moving camera: left, right, left, right, ..."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        X = camera(rng.normal(0, 0.02), (rng.normal(0, 0.1), rng.normal(0, 0.05), step*i))
        out += [X, TR.right_pose(X, K6[5])]
    return out


def check(lib, probs, **kw):
    """host build == reference in status, point within the a-priori bound; returns the references"""
    a = host(lib, probs, **kw)
    refs = []
    for i, q in enumerate(probs):
        r = TR.triangulate(q["poses"], q["kp"], q["calib"], kw.get("rank_tol", 1.0), kw.get("thr", 3.0))
        refs.append(r)
        assert a["status"][i] == r["status"], (i, a["status"][i], r)
        if r["status"] in (TR.OK, TR.OUTLIER, TR.BEHIND_CAMERA):
            err = np.linalg.norm(a["point"][i] - r["point"])
            assert err <= TR.point_bound(r), (i, err, TR.point_bound(r))
        if r["status"] in (TR.OK, TR.OUTLIER) and r["depths"].min() > 1e-3:     # (next to a camera the norm amplifies the point's error)
            assert abs(a["reproj"][i] - r["reproj"]) <= 1e-6*max(r["reproj"], 1.0), (i, a["reproj"][i], r["reproj"])
        if np.isfinite(r["sv"]).all():
            assert np.abs(a["sv"][i] - r["sv"]).max() <= 64*np.finfo(float).eps*r["sv"][0]*np.sqrt(len(q["kp"]))
    return a, refs


# ------------------------------------------------------------------------------------------------ branch edges
def test_two_cameras_and_fewer(shim):
    p = np.array([0.7, -0.3, 12.0])
    probs = [problem(stereo_cams(1), p, 0.3, 1),                                          # one stereo frame: left + right
             problem([camera(), camera(0.05, (1.0, 0.0, 0.5))], p, 0.3, 2),                # two monocular cameras
             problem([camera()], p),                                                      # one camera: degenerate
             dict(poses=np.zeros((0, 12)), kp=np.zeros((0, 2)), calib=K5)]                # none
    a, refs = check(shim, probs)
    assert [r["status"] for r in refs] == [TR.OK, TR.OK, TR.DEGENERATE, TR.DEGENERATE]
    assert np.isnan(a["point"][2]).all() and np.isnan(a["sv"][3]).all() and np.isnan(a["reproj"][2])


def test_left_only_cameras(shim):
    p = np.array([-2.0, 0.5, 20.0])
    cams = stereo_cams(6)[::2]                                                            # every right key-point missing
    check(shim, [problem(cams, p, 0.5, s) for s in range(4)] + [problem(cams[:2], p, 0.5, 9)])


def test_rank_straddles_rank_tol(shim):
    """A scales with (fx, fy, s, u0, v0, kp): choose the scale that puts sigma_3 at 1 +- 1e-6"""
    base = problem([camera(), camera(0.0, (0.05, 0.0, 0.0))], np.array([0.0, 0.0, 10.0]), 0.3, 4)
    s3 = TR.triangulate(base["poses"], base["kp"], base["calib"])["sv"][2]
    probs = []
    for side in (1 - 1e-6, 1 + 1e-6):
        lam = side/s3
        probs.append(dict(poses=base["poses"], kp=base["kp"]*lam, calib=K5*lam))
    _, refs = check(shim, probs)
    assert refs[0]["status"] == TR.DEGENERATE and refs[1]["status"] != TR.DEGENERATE
    assert refs[0]["sv"][2] < 1.0 < refs[1]["sv"][2]
    # the rank test counts singular values > rank_tol: rank_tol = 0 accepts anything that is not exactly singular
    check(shim, probs, rank_tol=0.0)


def test_far_points(shim):
    """v[3] -> 0: points at 1e2 .. 1e7 m seen from a short baseline"""
    probs = [problem(stereo_cams(3, 0.5), np.array([3.0, -1.0, d]), 0.05, int(np.log10(d))) for d in (1e2, 1e4, 1e5, 1e6, 1e7)]
    _, refs = check(shim, probs)
    assert {r["status"] for r in refs} <= {TR.OK, TR.BEHIND_CAMERA}


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_depth_next_to_zero(shim, sign):
    """the exact point at depth +-1e-7 m in one camera: cheirality decides, whatever the camera's index"""
    p = np.array([0.4, 0.2, 10.0])
    for pos in range(4):
        cams = [camera(0.0, (0.0, 0.0, 0.0)), camera(0.02, (0.5, 0.0, 0.0)), camera(-0.03, (-0.4, 0.1, 1.0))]
        near = camera(0.0, p - np.array([1e-9, 2e-9, sign*1e-7]))                              # looks along +z from next to p
        cams.insert(min(pos, 3), near)
        _, refs = check(shim, [problem(cams, p)])
        assert refs[0]["status"] == (TR.OK if sign > 0 else TR.BEHIND_CAMERA)
        d = refs[0]["depths"][min(pos, 3)]
        assert 0 < sign*d < 2e-7


def test_reprojection_norm_straddles_threshold(shim):
    """noise scaled so that the reference's norm is 3 +- 1e-6"""
    p = np.array([1.0, 0.3, 15.0])
    cams = stereo_cams(4)
    clean = problem(cams, p)
    noise = np.random.default_rng(5).normal(0, 1, clean["kp"].shape)

    def norm(t):
        return TR.triangulate(cams, clean["kp"] + t*noise, K5)["reproj"]
    lo, hi = 0.0, 10.0
    for _ in range(60):
        mid = 0.5*(lo + hi)
        lo, hi = (mid, hi) if norm(mid) < 3.0 else (lo, mid)
    probs = []
    for target in (3.0 - 1e-6, 3.0 + 1e-6):
        t = lo*target/3.0
        for _ in range(8):                                                                # secant on the reference's norm
            t = t*target/norm(t)
        probs.append(dict(poses=np.array(cams), kp=clean["kp"] + t*noise, calib=K5))
    _, refs = check(shim, probs)
    assert [r["status"] for r in refs] == [TR.OK, TR.OUTLIER]
    assert refs[0]["reproj"] < 3.0 < refs[1]["reproj"]


def test_random_problems_and_sizes(shim):
    rng = np.random.default_rng(11)
    probs = []
    for m in (2, 3, 8, 15, 16, 17, 32, 33, 40):
        p = np.array([rng.uniform(-5, 5), rng.uniform(-2, 2), rng.uniform(5, 60)])
        cams = stereo_cams((m + 1)//2, 1.0, int(rng.integers(1 << 20)))[:m]
        probs.append(problem(cams, p, rng.uniform(0.05, 0.3), int(rng.integers(1 << 20))))
    probs.append(problem(stereo_cams(3), np.array([0.0, 0.0, 20.0]), 0.2, 1))
    probs[-1]["kp"][2] += (300.0, 40.0)                                                    # a gross outlier
    _, refs = check(shim, probs)
    assert refs[-1]["status"] == TR.OUTLIER and sum(r["status"] == TR.OK for r in refs) >= 6


def test_two_cameras_against_cv2(shim):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    probs = []
    for i in range(20):
        p = np.array([rng.uniform(-4, 4), rng.uniform(-2, 2), rng.uniform(4, 80)])
        cams = [camera(rng.normal(0, 0.05), rng.normal(0, 0.3, 3)), camera(rng.normal(0, 0.05), rng.normal(0, 0.3, 3) + [1.0, 0, 0])]
        probs.append(problem(cams, p, 0.5, i))
    a = host(shim, probs)
    Km = np.array([[K5[0], K5[2], K5[3]], [0, K5[1], K5[4]], [0, 0, 1]])
    for i, q in enumerate(probs):
        P = [Km @ np.hstack([X[:9].reshape(3, 3).T, -(X[:9].reshape(3, 3).T @ X[9:])[:, None]]) for X in q["poses"]]
        h = cv2.triangulatePoints(P[0], P[1], q["kp"][0].reshape(2, 1), q["kp"][1].reshape(2, 1)).ravel()
        pc = h[:3]/h[3]
        assert a["status"][i] in (TR.OK, TR.OUTLIER)
        assert np.linalg.norm(a["point"][i] - pc) <= 1e-6*np.linalg.norm(pc), (i, a["point"][i], pc)


# ------------------------------------------------------------------------------------------------ mutations
def test_mutations_fail_a_case(tmp_path):
    """a rank test that lets rank 2 through, and a cheirality test that skips odd cameras (a stereo set's right cameras),
    each fail one of the cases above"""
    p = np.array([0.4, 0.2, 10.0])
    base = problem([camera(), camera(0.0, (0.05, 0.0, 0.0))], np.array([0.0, 0.0, 10.0]), 0.3, 4)
    s3 = TR.triangulate(base["poses"], base["kp"], base["calib"])["sv"][2]
    lam = (1 - 1e-6)/s3
    rank_case = dict(poses=base["poses"], kp=base["kp"]*lam, calib=K5*lam)
    cams = [camera(), camera(0.0, p - np.array([1e-9, 2e-9, -1e-7])), camera(0.02, (0.5, 0.0, 0.0))]
    behind_case = problem(cams, p)
    for patch, case in (([("if (rank < 3) {", "if (rank < 2) {")], rank_case),
                        ([("for (int c = lane; c < m; c += TRI_LANES) {", "for (int c = 2*lane; c < m; c += 2*TRI_LANES) {")], behind_case)):
        ref = TR.triangulate(case["poses"], case["kp"], case["calib"])
        lib = build_shim(tmp_path, patch)
        assert host(lib, [case])["status"][0] != ref["status"], patch
