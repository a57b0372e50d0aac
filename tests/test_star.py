"""SURVEY.md 8f-2: batched star problems -- the front end's joint optical-flow + pose refinement
(OpticalFlowAndPoseOptimizer::optimize, MotionSolver-inl.hpp:88-278) and object-motion refinement
(MotionOnlyRefinementOptimizer::optimize, :291-470), all objects of a frame in one launch."""
import numpy as np
import pytest

from dynosam_b200 import binding, lie

from dynosam_b200.synth_star import (FLOW_SIGMA, HUBER_K, K5, PRIOR_SIGMA, flow_parity_set, flow_rounds_set, make_flow_pose_problem as make_problem,
                                     make_motion_problem, motion_set)


def test_star_oracle_is_a_minimiser():
    """Pins the restatement: at its fixed point the gradient of the full objective vanishes and the pose is the ground truth
    (noise-free flows), so the dense LM in oracle/star_oracle.py solves the problem the reference poses."""
    from oracle import star_oracle as SO
    rng = np.random.default_rng(3)
    q = make_problem(rng, 60, noise=0.0)
    r = SO.flow_pose_lm(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], FLOW_SIGMA, PRIOR_SIGMA, 0.0,
                        max_iterations=50, relative_error_tol=1e-14, absolute_error_tol=1e-14)
    assert r["error_final"] < 1e-12 and r["error_final"] < 1e-6*r["error_initial"]
    assert np.abs(r["pose"] - q["gt"]).max() < 1e-7
    assert np.abs(r["flow"] - q["flow"]).max() < 1e-6
    # Huber: outliers pull less -- the robust fit is closer to the ground truth than the Gaussian one
    q = make_problem(rng, 120, noise=0.2, outliers=0.2)
    g = SO.flow_pose_lm(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], 1.0, 0.5, 0.0, max_iterations=10)
    h = SO.flow_pose_lm(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], 1.0, 0.5, 1.0, max_iterations=10)
    assert h["iterations"] >= 1 and g["iterations"] >= 1
    assert np.abs(h["pose"][9:] - q["gt"][9:]).max() < np.abs(g["pose"][9:] - q["gt"][9:]).max()


def test_star_batch_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rng = np.random.default_rng(0)
    with pytest.raises(binding.DynobaError):
        binding.flow_pose_batch([make_problem(rng, 10)])
    with pytest.raises(binding.DynobaError):
        binding.motion_refine_batch([make_motion_problem(rng, 10)])


def _build_capi_star(tmp_path):
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "capi_star"); libdir = os.path.join(root, "dynosam_b200")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "capi", "capi_star.c"),
                        "-o", exe, "-L", libdir, "-ldynoba", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def test_plain_c_program_links_the_star_abi(tmp_path):
    """tests/capi/capi_star.c: a C99 program links libdynoba.so and calls dynoba_flow_pose_batch; without a GPU it must stop with
    DYNOBA_ERR_CUDA (exit code 3)"""
    import subprocess
    import torch
    r = subprocess.run([_build_capi_star(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == (0 if torch.cuda.is_available() else 3), r.stdout + r.stderr


def test_star_batch_bad_arguments():
    L = binding.load()
    N = None
    assert L.dynoba_flow_pose_batch(0, -1, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N) == -1
    assert L.dynoba_flow_pose_batch(0, 1, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N) == -1
    assert L.dynoba_flow_pose_batch(0, 0, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N) == 0          # nothing to do
    assert L.dynoba_motion_refine_batch(0, -1, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N) == -1
    assert L.dynoba_motion_refine_batch(0, 2, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N) == -1
    assert L.dynoba_motion_refine_batch(0, 0, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N, N) == 0


def test_projection_factor_restatement():
    """gtsam::GenericProjectionFactor restated in oracle/star_oracle.py: analytic Jacobians against central differences on the
    manifold (pose perturbed by retract, [omega, v]), skew included; behind the camera: (2 fx, 2 fx) and zero Jacobians."""
    from oracle import star_oracle as SO
    rng = np.random.default_rng(8)
    K = np.array([700.0, 650.0, 1.5, 600.0, 180.0])
    for _ in range(5):
        X = lie.se3_exp(rng.normal(0, 0.3, (1, 6)))[0]
        p = lie.transform_from(X[None], np.array([[rng.uniform(-3, 3), rng.uniform(-2, 2), rng.uniform(4, 20)]]))[0]
        z = rng.uniform(0, 500, 2)
        r, Jx, Jp = SO.projection_factor(X, p, K, z)
        h = 1e-6
        for c in range(6):
            e = np.zeros((1, 6)); e[0, c] = h
            rp = SO.projection_factor(lie.retract(X[None], e)[0], p, K, z)[0]; rm = SO.projection_factor(lie.retract(X[None], -e)[0], p, K, z)[0]
            assert np.abs((rp - rm)/(2*h) - Jx[:, c]).max() < 1e-5*max(1.0, np.abs(Jx).max())
        for c in range(3):
            e = np.zeros(3); e[c] = h
            assert np.abs((SO.projection_factor(X, p + e, K, z)[0] - SO.projection_factor(X, p - e, K, z)[0])/(2*h) - Jp[:, c]).max() < 1e-5*max(1.0, np.abs(Jp).max())
    X = lie.identity()[0]
    r, Jx, Jp = SO.projection_factor(X, np.array([0.0, 0.0, -1.0]), K, np.zeros(2))
    assert np.array_equal(r, [1400.0, 1400.0]) and not Jx.any() and not Jp.any()


def _flow_pose_objective(q, X, flows, sig):
    """the objective of OpticalFlowAndPoseOptimizer written independently of oracle/: numpy projection + scipy's Huber loss"""
    from scipy.special import huber
    n = len(q["depth"])
    pc = np.stack([(q["kp_prev"][:, 0] - K5[3])/K5[0]*q["depth"], (q["kp_prev"][:, 1] - K5[4])/K5[1]*q["depth"], q["depth"]], 1)
    pw = lie.transform_from(np.tile(q["pose_prev"], (n, 1)), pc)
    c = lie.transform_to(np.tile(X, (n, 1)), pw)
    with np.errstate(all="ignore"):
        r = q["kp_prev"] + flows - np.stack([K5[0]*c[:, 0]/c[:, 2] + K5[3], K5[1]*c[:, 1]/c[:, 2] + K5[4]], 1)
    r[c[:, 2] <= 0] = 2.0*K5[0]                                            # Pose3FlowProjectionFactor.h: behind the camera
    nrm = np.linalg.norm(r, axis=1)/sig[0]
    loss = huber(sig[2], nrm) if sig[2] > 0 else 0.5*nrm**2
    return float(loss.sum() + 0.5*(((flows - q["flow"])/sig[1])**2).sum())


def test_flow_pose_oracle_against_independent_objective():
    """External pin of oracle/star_oracle.py (the reference holds no test of this optimiser): its error equals an objective written
    from scratch with numpy + scipy.special.huber at arbitrary values, and its LM ends in a stationary point of that objective."""
    from oracle import star_oracle as SO
    rng = np.random.default_rng(14)
    for sig in ((1.0, 0.5, 1.0), (FLOW_SIGMA, PRIOR_SIGMA, 0.0), (2.0, 1.0, 0.3)):
        q = make_problem(rng, 40, noise=0.4, outliers=0.1, behind=1)
        m = SO._FlowPose(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], *sig)
        for _ in range(3):                                                   # (a) same function
            m.step(rng.normal(0, 0.05, 2*40 + 6))
            assert abs(m.error() - _flow_pose_objective(q, m.o.pose[0], m.o.flow, sig)) <= 1e-10*max(m.error(), 1.0)
        r = SO.flow_pose_lm(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], *sig, max_iterations=200,
                            relative_error_tol=1e-15, absolute_error_tol=1e-15)
        f0 = _flow_pose_objective(q, r["pose"], r["flow"], sig)
        assert abs(f0 - r["error_final"]) <= 1e-10*max(f0, 1.0)
        h = 1e-6; g = []                                                     # (b) stationary: central differences through the retraction
        for j in range(6):
            e = np.zeros((1, 6)); e[0, j] = h
            g.append((_flow_pose_objective(q, lie.retract(r["pose"][None], e)[0], r["flow"], sig) -
                      _flow_pose_objective(q, lie.retract(r["pose"][None], -e)[0], r["flow"], sig))/(2*h))
        for i in (0, 7, 23):
            for a in range(2):
                fp = r["flow"].copy(); fp[i, a] += h; fm = r["flow"].copy(); fm[i, a] -= h
                g.append((_flow_pose_objective(q, r["pose"], fp, sig) - _flow_pose_objective(q, r["pose"], fm, sig))/(2*h))
        assert np.abs(g).max() < 1e-4*max(1.0, f0), (sig, np.abs(g).max(), f0)


def _motion_objective(q, poses, H, pts, sig_motion, sig_proj, k, sig_prior):
    """the objective of MotionOnlyRefinementOptimizer written independently of oracle/: numpy pinhole projection, 4x4 algebra,
    scipy.linalg.logm for the pose priors, scipy's Huber loss"""
    from scipy.linalg import logm
    from scipy.special import huber

    def mat(P):
        M = np.eye(4); M[:3, :3] = np.asarray(P)[:9].reshape(3, 3); M[:3, 3] = np.asarray(P)[9:]; return M

    def proj_res(X, p, z):
        c = (np.linalg.inv(mat(X)) @ np.concatenate([p, np.ones((len(p), 1))], 1).T).T[:, :3]
        with np.errstate(all="ignore"):
            r = np.stack([K5[0]*c[:, 0]/c[:, 2] + K5[3], K5[1]*c[:, 1]/c[:, 2] + K5[4]], 1) - z
        r[c[:, 2] <= 0] = 2.0*K5[0]
        return r
    total = 0.0
    for X, p, z in ((poses[0], pts[:, :3], q["kp_prev"]), (poses[1], pts[:, 3:], q["kp_cur"])):
        total += huber(k, np.linalg.norm(proj_res(X, p, z), axis=1)/sig_proj).sum()
    back = (np.linalg.inv(mat(H)) @ np.concatenate([pts[:, 3:], np.ones((len(pts), 1))], 1).T).T[:, :3]      # H^-1 m_k
    total += huber(k, np.linalg.norm(pts[:, :3] - back, axis=1)/sig_motion).sum()
    for X, prior in ((poses[0], q["pose_prev"]), (poses[1], q["pose_cur"])):
        L = np.real(logm(np.linalg.inv(mat(X)) @ mat(prior)))
        xi = np.array([L[2, 1], L[0, 2], L[1, 0], L[0, 3], L[1, 3], L[2, 3]])
        total += 0.5*((xi/sig_prior)**2).sum()
    return float(total)


def test_motion_refine_oracle_against_independent_objective():
    from oracle import star_oracle as SO
    rng = np.random.default_rng(15)
    q = make_motion_problem(rng, 25, outliers=0.1)
    args = (0.05, 2.0, 1.0, 1e-3)
    m = SO._MotionRefine(q["pose_prev"], q["pose_cur"], q["motion_init"], K5, q["kp_prev"], q["kp_cur"], q["points_init"], *args)
    for _ in range(3):
        m.step(np.concatenate([rng.normal(0, 0.02, 6*25), rng.normal(0, 1e-4, 12), rng.normal(0, 0.02, 6)]))
        f = _motion_objective(q, m.o.pose[:2], m.o.pose[2], m.o.point.reshape(25, 6), *args)
        assert abs(m.error() - f) <= 1e-9*max(f, 1.0), (m.error(), f)


def test_motion_refine_oracle_reduces_error():
    from oracle import star_oracle as SO
    rng = np.random.default_rng(4)
    q = make_motion_problem(rng, 30, outliers=0.1)
    r = SO.motion_refine_lm(q["pose_prev"], q["pose_cur"], q["motion_init"], K5, q["kp_prev"], q["kp_cur"], q["points_init"])
    assert r["iterations"] >= 1 and r["error_final"] < 0.1*r["error_initial"]
    assert np.abs(r["poses"] - np.stack([q["pose_prev"], q["pose_cur"]])).max() < 1e-6            # the 1e-5 priors hold the cameras
    assert r["motion_factor_error"].shape == (30,)


def test_flow_pose_oracle_outlier_rounds():
    """the outlier rounds of the restatement: gross outliers leave the graph, the inlier fit gets close to the ground truth"""
    from oracle import star_oracle as SO
    rng = np.random.default_rng(6)
    q = make_problem(rng, 150, noise=0.3, outliers=0.15)
    a = SO.flow_pose_refine(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], 1.0, 0.5, 1.0, outlier_rounds=0, max_iterations=10)
    b = SO.flow_pose_refine(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], 1.0, 0.5, 1.0, outlier_rounds=4, max_iterations=10)
    assert a["rounds"] == 0 and a["inlier"].all()
    assert 1 <= b["rounds"] <= 4 and 5 <= (~b["inlier"]).sum() <= 60
    assert np.abs(b["pose"][9:] - q["gt"][9:]).max() <= np.abs(a["pose"][9:] - q["gt"][9:]).max() + 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("sig", [(FLOW_SIGMA, PRIOR_SIGMA, HUBER_K), (1.0, 0.5, 1.0), (2.0, 1.0, 0.0)])
def test_star_batch_matches_oracle(sig):
    """Every problem of the batch runs the same LM as the CPU restatement: same accepted / rejected steps, same error, same
    pose and flows (fp64; tolerance 1e-9 relative on chi^2, 1e-7 on the values)."""
    from oracle import star_oracle as SO
    probs = flow_parity_set()
    out = binding.flow_pose_batch(probs, flow_sigma=sig[0], flow_prior_sigma=sig[1], huber_k=sig[2], outlier_rounds=0)
    assert len(out) == len(probs)
    moved = 0
    for q, r in zip(probs, out):
        o = SO.flow_pose_lm(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], *sig, max_iterations=10)
        assert abs(r["error_initial"] - o["error_initial"]) <= 1e-11*max(o["error_initial"], 1.0)
        if o["error_final"] < 1e-12*o["error_initial"]:
            # exact fit (<= 3 features: 4N residuals, 6 + 2N unknowns): the last steps act on rounding noise; same minimum, no step-by-step claim
            assert r["error_final"] < 1e-10*o["error_initial"] and r["iterations"] >= 1
            moved += 1
            continue
        assert (r["iterations"], r["inner_iterations"]) == (o["iterations"], o["inner_iterations"]), (len(q["depth"]), r, o)
        assert abs(r["error_final"] - o["error_final"]) <= 1e-9*max(o["error_final"], 1e-12) + 1e-12
        assert np.abs(r["pose"] - o["pose"]).max() < 1e-7 and np.abs(r["flow"] - o["flow"]).max() < 1e-6
        moved += r["iterations"] > 0
    assert moved >= len(probs) - 2


@pytest.mark.gpu
def test_star_batch_empty_and_large():
    """Edge cases: no problems, a problem with no features (nothing to do: the pose stays), and a frame-sized batch (one CTA per
    problem, more problems than SMs) whose every problem lowers its error."""
    assert binding.flow_pose_batch([]) == [] and binding.motion_refine_batch([]) == []
    rng = np.random.default_rng(2)
    probs = [make_problem(rng, 0)] + [make_problem(rng, int(n)) for n in rng.integers(30, 300, 400)]
    out = binding.flow_pose_batch(probs, flow_sigma=1.0, flow_prior_sigma=0.5, huber_k=1.0, outlier_rounds=0)
    assert out[0]["iterations"] == 0 and np.array_equal(out[0]["pose"], np.asarray(probs[0]["pose_init"]))
    closer = 0
    for q, r in zip(probs[1:], out[1:]):
        assert r["error_final"] < r["error_initial"] and r["iterations"] >= 1
        closer += np.abs(r["pose"][9:] - q["gt"][9:]).max() < np.abs(np.asarray(q["pose_init"])[9:] - q["gt"][9:]).max()
    assert closer >= 0.9*(len(probs) - 1)


@pytest.mark.gpu
def test_flow_pose_outlier_rounds_match_oracle():
    """LM + the reference's outlier rounds (MotionSolver-inl.hpp:201-247) in one launch: same inlier sets, number of rounds,
    iteration totals, error and pose as the CPU restatement."""
    from oracle import star_oracle as SO
    probs = flow_rounds_set()
    for sig in ((1.0, 0.5, 1.0), (FLOW_SIGMA, PRIOR_SIGMA, HUBER_K)):
        out = binding.flow_pose_batch(probs, flow_sigma=sig[0], flow_prior_sigma=sig[1], huber_k=sig[2])      # defaults: 4 rounds, 10 iterations
        with_rounds = 0; same = 0
        for q, r in zip(probs, out):
            o = SO.flow_pose_refine(q["pose_init"], q["pose_prev"], K5, q["kp_prev"], q["depth"], q["flow"], *sig, outlier_rounds=4, max_iterations=10)
            assert r["rounds"] == o["rounds"] and np.array_equal(r["inlier"], o["inlier"]), (len(q["depth"]), r["rounds"], o["rounds"])
            assert abs(r["error_initial"] - o["error_initial"]) <= 1e-11*max(o["error_initial"], 1.0)
            with_rounds += r["rounds"] > 0
            if (r["iterations"], r["inner_iterations"]) == (o["iterations"], o["inner_iterations"]):
                same += 1
                assert abs(r["error_final"] - o["error_final"]) <= 1e-9*max(o["error_final"], 1e-12) + 1e-12
                assert np.abs(r["pose"] - o["pose"]).max() < 1e-7 and np.abs(r["flow"] - o["flow"]).max() < 1e-6
            else:
                # a stopping test (relative decrease against 1e-5) fell on the other side in the last digits: one LM iteration more or
                # less at the same minimum
                assert abs(r["iterations"] - o["iterations"]) <= 1
                assert abs(r["error_final"] - o["error_final"]) <= 1e-4*o["error_final"] and np.abs(r["pose"] - o["pose"]).max() < 1e-4
        assert same >= len(probs) - 2, same
        if sig[0] == 1.0:
            assert with_rounds >= 5


def _proven_path(r, o):
    """None if the device took the oracle's LM path (iterations, inner iterations); otherwise the oracle's decision that proves
    the difference a last-digit one (its margin within its step bound, star_oracle.near_decision), or raises"""
    if (r["iterations"], r["inner_iterations"]) == (o["iterations"], o["inner_iterations"]):
        return None
    from oracle import star_oracle as SO
    d = SO.near_decision(o["trace"])
    assert d is not None, ("LM paths differ without a decision within its step bound", r["iterations"], r["inner_iterations"], o["iterations"], o["inner_iterations"])
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("soft", [False, True])
def test_motion_refine_batch_matches_oracle(soft):
    """Object-motion refinement, one CTA per problem: the same LM run as the dense CPU restatement.  A differing LM path is
    accepted only where the oracle recorded a decision whose margin lies within its step bound (_proven_path); every problem
    on the same path is compared.  The values after five LM iterations are compared at 1e-3 relative on chi^2, 1e-4 on the
    motion and 1e-3 on the points: they are not bounded by the single-step bound (eps kappa of the equilibrated system, 2e-9
    with the 1e-5 camera priors), because a step's rounding moves the next linearisation point along the weakly determined
    point depths; measured on an H100: chi^2 8e-6 .. 1e-5 relative, points 4e-4.  Each single step is pinned to a 50-digit
    reference in tests/test_star_cases_gpu.py."""
    from oracle import star_oracle as SO
    probs = motion_set()
    kw = dict(landmark_motion_sigma=0.05, huber_k=1.0, max_iterations=8) if soft else {}
    out = binding.motion_refine_batch(probs, **kw)
    same = 0; worst = dict(chi2=0.0, motion=0.0, points=0.0, factor=0.0)
    for q, r in zip(probs, out):
        o = SO.motion_refine_lm(q["pose_prev"], q["pose_cur"], q["motion_init"], K5, q["kp_prev"], q["kp_cur"], q["points_init"], **kw)
        assert abs(r["error_initial"] - o["error_initial"]) <= 1e-10*o["error_initial"]
        assert r["error_final"] < r["error_initial"]
        if _proven_path(r, o) is not None:
            continue
        same += 1
        worst["chi2"] = max(worst["chi2"], abs(r["error_final"] - o["error_final"])/o["error_final"])
        worst["motion"] = max(worst["motion"], np.abs(r["motion"] - o["motion"]).max())
        worst["points"] = max(worst["points"], np.abs(r["points"] - o["points"]).max())
        worst["factor"] = max(worst["factor"], np.abs(r["motion_factor_error"] - o["motion_factor_error"]).max()/max(o["motion_factor_error"].max(), 1.0))
        assert np.abs(r["poses"] - o["poses"]).max() < 1e-6
    print("motion_refine parity", "soft" if soft else "reference-params", "same LM path:", same, "of", len(probs), worst)
    assert worst["chi2"] < 1e-3 and worst["motion"] < 1e-4 and worst["points"] < 1e-3 and worst["factor"] < 1e-3, worst


# ---- golden fixtures (tests/golden/star_*.npz, written by tests/golden/make_golden.py): outputs of oracle/star_oracle.py on the seeded sets
def _load_golden(name):
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name))


STAR_SIGMAS = dict(flow_sigma=1.0, flow_prior_sigma=0.5, huber_k=1.0)


def _check_star_flow(g, results, offset=0):
    """results[i] belongs to problem offset + i of the fixture; exact-fit problems (<= 3 features) are compared at the minimum"""
    starts = np.concatenate([[0], np.cumsum(g["n"])])
    same = 0
    for i, r in enumerate(results):
        j = offset + i
        assert len(r["flow"]) == int(g["n"][j])
        assert abs(r["error_initial"] - g["error_initial"][j]) <= 1e-11*max(g["error_initial"][j], 1.0)
        assert r["rounds"] == int(g["rounds"][j])
        assert np.array_equal(np.asarray(r["inlier"], dtype=np.uint8), g["inlier_bits"][starts[j]:starts[j + 1]])
        if g["error_final"][j] < 1e-12*g["error_initial"][j]:
            assert r["error_final"] < 1e-10*g["error_initial"][j]
            same += 1
            continue
        if (r["iterations"], r["inner_iterations"]) == (int(g["iterations"][j]), int(g["inner_iterations"][j])):
            same += 1
            assert abs(r["error_final"] - g["error_final"][j]) <= 1e-9*max(g["error_final"][j], 1e-12) + 1e-12
            assert np.abs(r["pose"] - g["pose"][j]).max() < 1e-7
            assert np.abs(r["flow"].sum(0) - g["flow_sum"][j]).max() < 1e-6*max(len(r["flow"]), 1)
        else:       # a stopping test fell on the other side in the last digits: same minimum, one iteration more or less
            assert abs(r["iterations"] - int(g["iterations"][j])) <= 1
            assert abs(r["error_final"] - g["error_final"][j]) <= 1e-4*g["error_final"][j] and np.abs(r["pose"] - g["pose"][j]).max() < 1e-4
    assert same >= len(results) - 2, same


def _check_star_motion(g, results, offset=0, problems=None):
    """results[i] against stored run offset + i; where the LM path differs, the oracle is re-run on problems[offset + i] and must
    hold a decision within its step bound (_proven_path); where it agrees, the values agree as in
    test_motion_refine_batch_matches_oracle"""
    from oracle import star_oracle as SO
    for i, r in enumerate(results):
        j = offset + i
        assert len(r["points"]) == int(g["n"][j])
        assert abs(r["error_initial"] - g["error_initial"][j]) <= 1e-10*g["error_initial"][j]
        q = problems[j]
        o = SO.motion_refine_lm(q["pose_prev"], q["pose_cur"], q["motion_init"], K5, q["kp_prev"], q["kp_cur"], q["points_init"])
        assert (o["iterations"], o["inner_iterations"]) == (int(g["iterations"][j]), int(g["inner_iterations"][j]))
        if _proven_path(r, o) is not None:
            continue
        assert abs(r["error_final"] - g["error_final"][j]) <= 1e-3*g["error_final"][j]
        assert np.abs(r["motion"] - g["motion"][j]).max() < 1e-4 and np.abs(r["poses"] - g["poses"][j]).max() < 1e-6
        assert abs(r["motion_factor_error"].sum() - g["factor_error_sum"][j]) <= 1e-3*max(g["factor_error_sum"][j], 1.0)


def test_oracle_reproduces_golden_star():
    """the dense restatements still give the stored runs (a slice of every set, to keep the CPU suite short)"""
    from dynosam_b200 import synth_star
    from oracle import star_oracle as SO
    sig = (STAR_SIGMAS["flow_sigma"], STAR_SIGMAS["flow_prior_sigma"], STAR_SIGMAS["huber_k"])
    for name, probs, rounds, lo, hi in (("star_flow_pose_lm.npz", synth_star.flow_parity_set(), 0, 2, 9), ("star_flow_pose_rounds.npz", synth_star.flow_rounds_set(), 4, 0, 4)):
        rs = [SO.flow_pose_refine(q["pose_init"], q["pose_prev"], synth_star.K5, q["kp_prev"], q["depth"], q["flow"], *sig, outlier_rounds=rounds, max_iterations=10)
              for q in probs[lo:hi]]
        _check_star_flow(_load_golden(name), rs, offset=lo)
    probs = synth_star.motion_set()
    rs = [SO.motion_refine_lm(q["pose_prev"], q["pose_cur"], q["motion_init"], synth_star.K5, q["kp_prev"], q["kp_cur"], q["points_init"]) for q in probs[:5]]
    _check_star_motion(_load_golden("star_motion_refine.npz"), rs, problems=probs)


@pytest.mark.gpu
def test_cuda_reproduces_golden_star():
    """dynoba_flow_pose_batch / dynoba_motion_refine_batch against the stored runs, no oracle at run time"""
    from dynosam_b200 import binding, synth_star
    _check_star_flow(_load_golden("star_flow_pose_lm.npz"), binding.flow_pose_batch(synth_star.flow_parity_set(), outlier_rounds=0, **STAR_SIGMAS))
    _check_star_flow(_load_golden("star_flow_pose_rounds.npz"), binding.flow_pose_batch(synth_star.flow_rounds_set(), **STAR_SIGMAS))
    probs = synth_star.motion_set()
    _check_star_motion(_load_golden("star_motion_refine.npz"), binding.motion_refine_batch(probs), problems=probs)
