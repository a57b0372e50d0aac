"""The case list of the batched flow + pose and object-motion refinements (csrc/kernels_star.cu): batches of small problems,
each case naming the boundaries it reaches (`hits`), the single-step observation both halves of the test use, and one
comparator in units of an a-priori bound.  tests/test_star_cases.py checks on the CPU that every name of `REQUIRED` is reached
and that every claim is true; tests/test_star_cases_gpu.py runs the cases on the device.

Observing one damped step through the batch binding: max_iterations 1, lambda_initial lam, min_model_fidelity -1e308,
relative_error_tol 0, no outlier rounds.  iterations == inner_iterations == 1 then proves that the outputs are the candidate
of exactly one solve at lam.  The pose part of the step is read back as Log(Retract(X0, d_ref)^-1 X_out), the flows /
points as output minus input.

Comparator.  step: |D_i (d_dev - d_ref)_i| / (eps (kappa |D d_ref|_2 + rhs_i) + eps D_i R_i) with D the square root of the
damped diagonal, kappa that of the equilibrated damped system, rhs the D-scaled error the rounding of the residuals alone may
cause, and R_i the magnitude of the value read back.  errors: |e_dev - e_ref| / (eps * the summed rounding scales of the
factors).  The Huber cases at |r_w| = k and one ulp either side show that the kernel is continuous at k: there the two
branches' errors differ by about 1e-31 and their weights by about one ulp, far below both bounds, so they cannot tell which
branch ran and do not pin the `<=` of the branch test.  The branches themselves are pinned by the cases well inside them
(k = 1e-3 with whitened norms ~1e-1 .. 4, k = 1 on both sides, k = 0).  Large-N problems tile a period of 257 distinct features: 257 is coprime to the 256 threads and 32 lanes of a CTA,
so a wrong index never reads an identical copy.
"""
import re
from dataclasses import dataclass, field

import numpy as np

from dynosam_b200 import lie

EPS = 2.0**-52
PERIOD = 257


def _kernel_constants():
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dynosam_b200", "csrc", "kernels_star.cu")).read()
    threads = int(re.search(r"constexpr int STAR_THREADS = (\d+);", src).group(1))
    scr = int(re.search(r"MR_SCR = (\d+);", src).group(1))
    return threads, threads//32, scr


STAR_THREADS, STAR_WARPS, MR_SCR = _kernel_constants()
FLOW_N = [0, 1, 2, 3, 4, 31, 32, 33, 224, 225, 255, 256, 257, 511, 512, 513, 4096]
MOTION_N = [0, 1, 2, 6, 7, 31, 32, 33, 255, 256, 257, 1024]
LAMBDAS = [1e-300, 1e-5, 1.0, 1e5]
FLOW_DEFAULT = (10.0, 3.33, 1e-3)                       # flow_sigma, flow_prior_sigma, huber_k
MOTION_DEFAULT = (1e-3, 2.0, 1e-4, 1e-5)                # landmark_motion_sigma, projection_sigma, huber_k, pose_prior_sigma
K_MAIN = np.array([718.5, 702.25, 3.7, 611.25, 180.5])
K_BATCH = [np.array([721.5, 690.0, 0.0, 600.5, 170.25]), np.array([650.0, 655.5, 3.7, 640.0, 200.0]),
           np.array([800.0, 780.0, -12.0, 590.0, 160.5])]
K_DYADIC = np.array([512.0, 512.0, 0.0, 640.0, 192.0])

REQUIRED = (
    [f"flow:N={n}" for n in FLOW_N] + [f"motion:N={n}" for n in MOTION_N]
    + ["flow:exact_fit", "flow:first_on_warp7", "flow:two_per_thread", "motion:mixed_N_batch",
       "flow:calib_per_problem", "motion:calib_per_problem", "skew:0", "skew:3.7", "skew:-12"]
    + [f"flow:cheirality:{z}" for z in ("z<0", "z=-0", "z=+0", "z=1e-12", "z=denormal")]
    + [f"motion:cheirality:{w}" for w in ("a_only", "b_only", "both", "z=+0", "z=-0")]
    + [f"huber:{f}:{w}" for f in ("flow", "projection", "motion") for w in ("n=k", "n=k+ulp", "n=k-ulp")]
    + ["huber:k=0", "huber:k=default", "huber:k=1", "sigma:1e-3", "sigma:1e3", "prior:1e-5", "prior:1e-2",
       "motion_sigma:1e-3", "motion_sigma:0.05"]
    + [f"lambda:{lam:g}" for lam in LAMBDAS] + ["pose:1e3_from_origin"]
    + ["exit:error_tol", "exit:max_iterations=0", "exit:all_rejected", "exit:stop_flag", "exit:failed_cholesky",
       "exit:relative_termination", "exit:absolute_termination", "exit:nan_keypoint"]
    + [f"outlier:rounds={k}" for k in (1, 2, 3, 4)] + ["outlier:no_outliers_before_cap", "outlier:cap", "outlier:custom_threshold",
                                                       "outlier:all_removed"])


@dataclass
class Case:
    name: str
    kind: str                       # "flow" | "motion"
    problems: list
    hits: tuple
    sig: tuple = None
    lam: float = 1e-5
    params: dict = field(default_factory=dict)     # extra binding parameters (exit cases)
    exit: dict = None               # exit cases: expected iterations / inner per problem, outputs bit-equal to the inputs
    note: str = ""


def _dyadic_flow_feature(K, kp_off, depth=1.0):
    """key-point at an offset from (u0, v0) that back-projects and projects exactly in fp64 at identity poses"""
    return np.array([K[3] + kp_off[0], K[4] + kp_off[1]]), depth


def single_step_params(kind, lam):
    p = dict(max_iterations=1, lambda_initial=lam, min_model_fidelity=-1e308, relative_error_tol=0.0)
    if kind == "flow":
        p["outlier_rounds"] = 0
    return p


def binding_params(case):
    if case.kind == "flow":
        p = dict(flow_sigma=case.sig[0], flow_prior_sigma=case.sig[1], huber_k=case.sig[2])
    else:
        p = dict(landmark_motion_sigma=case.sig[0], projection_sigma=case.sig[1], huber_k=case.sig[2], pose_prior_sigma=case.sig[3])
    p.update(single_step_params(case.kind, case.lam))
    p.update(case.params)
    return p


# ---------------------------------------------------------------------------------------------- geometries
def _tile(a, n, period):
    a = np.asarray(a)
    return a[np.arange(n) % period] if n else a[:0]


def flow_geometry(seed, K=K_MAIN, period=PERIOD, origin=0.0, identity=False):
    """`period` distinct features of a camera step: key-points, depths, measured flows (noise, 10 % gross outliers)"""
    rng = np.random.default_rng(seed)
    X_prev = lie.se3_exp(rng.normal(0, 0.05, (1, 6)))[0] if not identity else lie.identity()[0].copy()
    X_prev[9:] += origin
    step = lie.se3_exp(np.array([[0.01, -0.02, 0.005, 0.05, -0.02, 0.9]]) + rng.normal(0, 0.01, (1, 6)))[0]
    X_gt = lie.compose(X_prev[None], step[None])[0]
    kp = np.stack([rng.uniform(50, 1190, period), rng.uniform(30, 340, period)], 1); depth = rng.uniform(5, 40, period)
    yn = (kp[:, 1] - K[4])/K[1]; xn = (kp[:, 0] - K[3] - K[2]*yn)/K[0]
    pw = lie.transform_from(np.tile(X_prev, (period, 1)), np.stack([xn*depth, yn*depth, depth], 1))
    q = lie.transform_to(np.tile(X_gt, (period, 1)), pw)
    proj = np.stack([K[0]*q[:, 0]/q[:, 2] + K[2]*q[:, 1]/q[:, 2] + K[3], K[1]*q[:, 1]/q[:, 2] + K[4]], 1)
    flow = proj - kp + rng.normal(0, 0.5, (period, 2))
    bad = rng.random(period) < 0.1; flow[bad] += rng.normal(0, 40.0, (int(bad.sum()), 2))
    init = lie.compose(X_gt[None], lie.se3_exp(rng.normal(0, 0.02, (1, 6))))[0]
    return dict(pose_init=init, pose_prev=X_prev, calib=np.asarray(K, float), kp_prev=kp, depth=depth, flow=flow)


def flow_problem(geo, n):
    q = dict(pose_init=geo["pose_init"], pose_prev=geo["pose_prev"], calib=geo["calib"])
    P = len(geo["depth"])
    for k in ("kp_prev", "depth", "flow"):
        q[k] = _tile(geo[k], n, P)
    q["period"] = P
    return q


def motion_geometry(seed, K=K_MAIN, period=PERIOD, origin=0.0):
    rng = np.random.default_rng(seed)
    Xa = lie.se3_exp(rng.normal(0, 0.05, (1, 6)))[0]; Xa[9:] += origin
    Xb = lie.compose(Xa[None], lie.se3_exp(np.array([[0.002, -0.01, 0.001, 0.02, -0.01, 0.6]])))[0]
    H = lie.se3_exp(np.array([[0.01, 0.03, -0.01, 0.3, 0.02, 0.5]]) + rng.normal(0, 0.01, (1, 6)))[0]
    if origin:
        H = lie.compose(lie.compose(np.array([np.r_[np.eye(3).ravel(), Xa[9:]]]), H[None]), np.array([np.r_[np.eye(3).ravel(), -Xa[9:]]]))[0]
    kp0 = np.stack([rng.uniform(400, 800, period), rng.uniform(100, 300, period)], 1); d0 = rng.uniform(8, 20, period)

    def back(X, kp, d):
        yn = (kp[:, 1] - K[4])/K[1]; xn = (kp[:, 0] - K[3] - K[2]*yn)/K[0]
        return lie.transform_from(np.tile(X, (len(kp), 1)), np.stack([xn*d, yn*d, d], 1))

    def proj(X, p):
        q = lie.transform_to(np.tile(X, (len(p), 1)), p)
        return np.stack([K[0]*q[:, 0]/q[:, 2] + K[2]*q[:, 1]/q[:, 2] + K[3], K[1]*q[:, 1]/q[:, 2] + K[4]], 1), q[:, 2]
    ma = back(Xa, kp0, d0)
    mb = lie.transform_from(np.tile(H, (period, 1)), ma)
    bad = rng.random(period) < 0.1; mb[bad] += rng.normal(0, 0.5, (int(bad.sum()), 3))
    (kpa, da), (kpb, db) = proj(Xa, ma), proj(Xb, mb)
    kpa = kpa + rng.normal(0, 0.3, (period, 2)); kpb = kpb + rng.normal(0, 0.3, (period, 2))
    ma0 = back(Xa, kpa, da*(1 + rng.normal(0, 0.05, period))); mb0 = back(Xb, kpb, db*(1 + rng.normal(0, 0.05, period)))
    H0 = lie.compose(H[None], lie.se3_exp(rng.normal(0, 0.02, (1, 6))))[0]
    return dict(pose_prev=Xa, pose_cur=Xb, motion_init=H0, calib=np.asarray(K, float), kp_prev=kpa, kp_cur=kpb,
                points_init=np.concatenate([ma0, mb0], 1))


def motion_problem(geo, n):
    q = dict(pose_prev=geo["pose_prev"], pose_cur=geo["pose_cur"], motion_init=geo["motion_init"], calib=geo["calib"])
    P = len(geo["kp_prev"])
    for k in ("kp_prev", "kp_cur", "points_init"):
        q[k] = _tile(geo[k], n, P)
    q["period"] = P
    return q


def _identity():
    return lie.identity()[0].copy()


# ---------------------------------------------------------------------------------------------- cases
def flow_cases():
    g = flow_geometry(1)
    sub = flow_geometry(1, period=64)
    cases = []
    hits = [f"flow:N={n}" for n in FLOW_N] + ["flow:exact_fit", "flow:first_on_warp7", "flow:two_per_thread", "skew:3.7",
                                              "huber:k=default", "lambda:1e-05"]
    cases.append(Case("flow:sizes", "flow", [flow_problem(g, n) for n in FLOW_N], tuple(hits), FLOW_DEFAULT))
    q257 = flow_problem(g, 257)
    for sig, h in (((1e-3, 1e-3, 0.0), ("sigma:1e-3", "huber:k=0")), ((1e3, 1e3, 0.0), ("sigma:1e3",)), ((1.0, 0.5, 1.0), ("huber:k=1",))):
        cases.append(Case(f"flow:sigma={sig}", "flow", [q257], h, sig))
    for lam in LAMBDAS:
        cases.append(Case(f"flow:lambda={lam:g}", "flow", [flow_problem(sub, 64)], (f"lambda:{lam:g}",), FLOW_DEFAULT, lam))
    geos = [flow_geometry(10 + i, K=K, period=40) for i, K in enumerate(K_BATCH)]
    cases.append(Case("flow:calib_batch", "flow", [flow_problem(gg, 40) for gg in geos], ("flow:calib_per_problem", "skew:0", "skew:3.7", "skew:-12"),
                      (1.0, 0.5, 1.0)))
    far = flow_geometry(5, period=64, origin=1e3)
    cases.append(Case("flow:far", "flow", [flow_problem(far, 64)], ("pose:1e3_from_origin",), (1.0, 0.5, 1.0)))
    # cheirality: identity poses, camera depth = the key-point's depth
    gi = flow_geometry(7, period=12, identity=True)
    gi["pose_init"] = _identity()
    for j, z in enumerate((-1.0, -0.0, 0.0, 1e-12)):
        gi["depth"][j] = z
    cases.append(Case("flow:cheirality", "flow", [flow_problem(gi, 12)], ("flow:cheirality:z<0", "flow:cheirality:z=-0",
                                                                          "flow:cheirality:z=+0", "flow:cheirality:z=1e-12"), (1.0, 0.5, 1.0)))
    # Huber at k on the flow factor: dyadic key-point and flow at identity poses, whitened residual (3, 4): |r_w| = 5 exactly
    kp, d = _dyadic_flow_feature(K_DYADIC, (128.0, 64.0))
    hq = dict(pose_init=_identity(), pose_prev=_identity(), calib=K_DYADIC, kp_prev=kp[None], depth=np.array([d]), flow=np.array([[3.0, 4.0]]))
    for w, k in (("n=k", 5.0), ("n=k+ulp", np.nextafter(5.0, 0.0)), ("n=k-ulp", np.nextafter(5.0, 10.0))):
        cases.append(Case(f"flow:huber:{w}", "flow", [hq], (f"huber:flow:{w}",), (1.0, 1.0, float(k)),
                          note="n = k + ulp means the norm lies one ulp above k (k one ulp below 5)"))
    return cases


def motion_cases():
    g = motion_geometry(2)
    sub = motion_geometry(2, period=64)
    cases = []
    cases.append(Case("motion:sizes", "motion", [motion_problem(g, n) for n in MOTION_N],
                      tuple(f"motion:N={n}" for n in MOTION_N) + ("skew:3.7", "prior:1e-5", "motion_sigma:1e-3"), MOTION_DEFAULT))
    cases.append(Case("motion:mixed", "motion", [motion_problem(g, n) for n in (1024, 0, 257, 1, 0, 1024)], ("motion:mixed_N_batch",), MOTION_DEFAULT))
    cases.append(Case("motion:soft", "motion", [motion_problem(sub, 64)], ("prior:1e-2", "motion_sigma:0.05"), (0.05, 2.0, 1.0, 1e-2)))
    for lam in (1e-300, 1.0, 1e5):
        cases.append(Case(f"motion:lambda={lam:g}", "motion", [motion_problem(sub, 64)], (f"lambda:{lam:g}",), (0.05, 2.0, 1.0, 1e-2), lam))
    geos = [motion_geometry(20 + i, K=K, period=20) for i, K in enumerate(K_BATCH)]
    cases.append(Case("motion:calib_batch", "motion", [motion_problem(gg, 20) for gg in geos], ("motion:calib_per_problem", "skew:0", "skew:-12"),
                      (0.05, 2.0, 1.0, 1e-2)))
    far = motion_geometry(6, period=32, origin=1e3)
    cases.append(Case("motion:far", "motion", [motion_problem(far, 32)], ("pose:1e3_from_origin",), (0.05, 2.0, 1.0, 1e-2)))
    # cheirality: identity camera poses, small motion; tracklets 0-4 behind X_a only, X_b only, both, at q_z = +0 and -0
    gc = motion_geometry(8, period=11)
    gc["pose_prev"] = _identity(); gc["pose_cur"] = _identity()
    pts = gc["points_init"]
    pts[0, 2] = -2.0; pts[1, 5] = -3.0; pts[2, 2] = -1.0; pts[2, 5] = -1.5; pts[3, 2] = 0.0; pts[4, 2] = -0.0
    cases.append(Case("motion:cheirality", "motion", [motion_problem(gc, 11)], tuple(f"motion:cheirality:{w}" for w in ("a_only", "b_only", "both", "z=+0", "z=-0")),
                      (0.05, 2.0, 1.0, 1e-2)))
    # Huber at k: dyadic points seen from identity poses.  projection: kp_a off by (3, 4) px; motion: m_b - m_a = (3, 4, 0) sigma_m
    ma = np.array([0.5, 0.25, 2.0]); pix = lambda m: np.array([K_DYADIC[0]*m[0]/m[2] + K_DYADIC[3], K_DYADIC[1]*m[1]/m[2] + K_DYADIC[4]])
    base = dict(pose_prev=_identity(), pose_cur=_identity(), motion_init=_identity(), calib=K_DYADIC)
    proj_q = dict(base, kp_prev=(pix(ma) - [3.0, 4.0])[None], kp_cur=pix(ma)[None], points_init=np.r_[ma, ma][None])
    mb = ma + np.array([0.375, 0.5, 0.0])
    mot_q = dict(base, kp_prev=pix(ma)[None], kp_cur=pix(mb)[None], points_init=np.r_[ma, mb][None])
    for w, k in (("n=k", 5.0), ("n=k+ulp", np.nextafter(5.0, 0.0)), ("n=k-ulp", np.nextafter(5.0, 10.0))):
        cases.append(Case(f"projection:huber:{w}", "motion", [proj_q], (f"huber:projection:{w}",), (1.0, 1.0, float(k), 1e-2)))
        cases.append(Case(f"motion:huber:{w}", "motion", [mot_q], (f"huber:motion:{w}",), (0.125, 1.0, float(k), 1e-2)))
    return cases


def lambda_climb(lam0, factor, upper):
    """the inner iterations of a tryLambda in which every step fails: lambda *= factor until it reaches the upper bound"""
    n = 0
    while True:
        lam0 *= factor; n += 1
        if lam0 >= upper:
            return n


def exit_cases():
    g = flow_geometry(3, period=40); q = flow_problem(g, 40)
    gm = motion_geometry(4, period=30); qm = motion_problem(gm, 30)
    sig, sigm = (1.0, 0.5, 1.0), (0.05, 2.0, 1.0, 1e-2)
    climb = lambda_climb(1e-5, 10.0, 1e5)
    cases = []
    for kind, qq, s in (("flow", q, sig), ("motion", [qm][0], sigm)):
        cases.append(Case(f"{kind}:exit:error_tol", kind, [qq], ("exit:error_tol",), s, params=dict(error_tol=1e300, max_iterations=10),
                          exit=dict(iterations=0, inner=0)))
        cases.append(Case(f"{kind}:exit:max_iterations=0", kind, [qq], ("exit:max_iterations=0",), s, params=dict(max_iterations=0),
                          exit=dict(iterations=0, inner=0)))
        cases.append(Case(f"{kind}:exit:all_rejected", kind, [qq], ("exit:all_rejected",), s, params=dict(min_model_fidelity=1e300, max_iterations=10),
                          exit=dict(iterations=0, inner=climb)))
        cases.append(Case(f"{kind}:exit:stop_flag", kind, [qq], ("exit:stop_flag",), s,
                          params=dict(min_model_fidelity=1e300, relative_error_tol=1e300, max_iterations=10), exit=dict(iterations=0, inner=0)))
    # a camera depth of one denormal: 1/z overflows, the damped system is not positive definite at any lambda
    gd = flow_geometry(7, period=12, identity=True); gd["pose_init"] = _identity(); gd["depth"][5] = 5e-324
    cases.append(Case("flow:exit:failed_cholesky", "flow", [flow_problem(gd, 12)], ("exit:failed_cholesky", "flow:cheirality:z=denormal"), sig,
                      exit=dict(iterations=0, inner=climb), note="the error itself is NaN there (0 * inf); only the control flow is claimed"))
    return cases


def trace_cases():
    """full LM runs compared with star_oracle's trace: (iterations, inner) equal unless the oracle recorded a decision within
    its step bound.  exit["ended"] is what ends the LM (termination cases) or the outlier rounds (outlier cases) of at
    least one problem in the oracle's run; "cap" means outliers remain after the last allowed round, "no_outliers" that a round found
    none (for outlier_rounds 4 before the cap)."""
    g = flow_geometry(3, period=40); q = flow_problem(g, 40)
    gm = motion_geometry(4, period=30); qm = motion_problem(gm, 30)
    cases = [Case("flow:relative_termination", "flow", [q], ("exit:relative_termination",), (1.0, 0.5, 1.0),
                  params=dict(max_iterations=50, min_model_fidelity=1e-3, relative_error_tol=1e-6, absolute_error_tol=0.0), exit=dict(ended="relative")),
             Case("flow:absolute_termination", "flow", [q], ("exit:absolute_termination",), (1.0, 0.5, 1.0),
                  params=dict(max_iterations=50, min_model_fidelity=1e-3, relative_error_tol=0.0, absolute_error_tol=1e-3), exit=dict(ended="absolute")),
             Case("motion:relative_termination", "motion", [qm], ("exit:relative_termination",), (0.05, 2.0, 1.0, 1e-2),
                  params=dict(max_iterations=50, min_model_fidelity=1e-3, relative_error_tol=1e-6, absolute_error_tol=0.0), exit=dict(ended="relative")),
             Case("motion:absolute_termination", "motion", [qm], ("exit:absolute_termination",), (0.05, 2.0, 1.0, 1e-2),
                  params=dict(max_iterations=50, min_model_fidelity=1e-3, relative_error_tol=0.0, absolute_error_tol=1e-3), exit=dict(ended="absolute"))]
    probs = [flow_problem(flow_geometry(40 + i, period=n), n) for i, n in enumerate((30, 90, 257))]
    for rounds, thr, hits, ended in ((1, 0.1, ("outlier:rounds=1", "outlier:cap"), "cap"), (2, 0.1, ("outlier:rounds=2", "outlier:cap"), "cap"),
                                     (3, 0.1, ("outlier:rounds=3", "outlier:custom_threshold"), None),
                                     (4, 0.0, ("outlier:rounds=4", "outlier:no_outliers_before_cap"), "no_outliers"),
                                     (4, 1e-12, ("outlier:all_removed",), "no_outliers")):
        cases.append(Case(f"flow:outlier_rounds={rounds}:thr={thr:g}", "flow", probs, hits, (1.0, 0.5, 1.0),
                          params=dict(outlier_rounds=rounds, outlier_threshold=thr, max_iterations=10, min_model_fidelity=1e-3,
                                      relative_error_tol=1e-5), exit=dict(ended=ended)))
    return cases


def oracle_run(case, q):
    """star_oracle's full run of one problem of a trace case"""
    from oracle import star_oracle as SO
    p = binding_params(case)
    lm = {k: v for k, v in p.items() if k in SO.DEFAULTS}
    if case.kind == "flow":
        return SO.flow_pose_refine(q["pose_init"], q["pose_prev"], q["calib"], q["kp_prev"], q["depth"], q["flow"], *case.sig,
                                   outlier_rounds=p["outlier_rounds"], outlier_threshold=p.get("outlier_threshold"), **lm)
    return SO.motion_refine_lm(q["pose_prev"], q["pose_cur"], q["motion_init"], q["calib"], q["kp_prev"], q["kp_cur"], q["points_init"],
                               *case.sig, **lm)


def nan_batch():
    """three problems and the same batch with a NaN key-point in the middle one"""
    g = flow_geometry(9, period=80)
    probs = [flow_problem(g, n) for n in (80, 33, 57)]
    bad = dict(probs[1]); bad["kp_prev"] = probs[1]["kp_prev"].copy(); bad["kp_prev"][7, 0] = np.nan
    return probs, [probs[0], bad, probs[2]]


def all_cases():
    nan = Case("flow:exit:nan_keypoint", "flow", nan_batch()[1], ("exit:nan_keypoint",), (1.0, 0.5, 1.0))
    return flow_cases() + motion_cases() + exit_cases() + trace_cases() + [nan]


# ---------------------------------------------------------------------------------------------- comparator
def step_score(d_err, D, ref_norm, kappa, rhs_err, R):
    """worst |D_i d_err_i| / (eps (kappa |D d_ref|_2 + rhs_err) + eps D_i R_i) over the components"""
    d_err, D, R = (np.asarray(x, dtype=np.float64) for x in (d_err, D, R))
    bound = EPS*(kappa*ref_norm + rhs_err) + EPS*D*R
    return float(np.max(np.abs(D*d_err)/bound)) if len(d_err) else 0.0


def error_score(e_dev, e_ref, scale):
    return abs(float(e_dev) - float(e_ref))/(EPS*max(float(scale), 1e-300))


def _local_offsets(mult, ng, nl):
    off = [ng]
    for m in mult[:-1]:
        off.append(off[-1] + nl*m)
    return off


def evaluate(case, outs):
    """scores of one case's device results (one per problem) in units of the bounds: dict(step, error_initial, error_final)
    and a list of violated claims (wrong control flow, tiled copies that differ)"""
    import star_reference as SR
    from mpmath import mpf
    worst =dict(step=0.0, error_initial=0.0, error_final=0.0); bad = []
    for p, (q, r) in enumerate(zip(case.problems, outs)):
        flow = case.kind == "flow"
        n = len(q["depth"]) if flow else len(q["kp_prev"])
        P = min(q.get("period") or n, n)
        local = r["flow"] if flow else r["points"]
        if n and P < n and not all(np.array_equal(local[i], local[i % P]) for i in range(n)):
            bad.append((case.name, p, "tiled copies differ"))
        sig = case.sig
        if flow:
            e0, s0 = SR.flow_objective(q, q["pose_init"], q["flow"][:P], sig)
        else:
            e0, s0 = SR.motion_objective(q, [q["pose_prev"], q["pose_cur"], q["motion_init"]], q["points_init"][:P], sig)
        worst["error_initial"] = max(worst["error_initial"], error_score(r["error_initial"], e0, s0))
        if n == 0:
            if (r["iterations"], r["inner_iterations"]) != (0, 0):
                bad.append((case.name, p, "N = 0 moved"))
            continue
        if (r["iterations"], r["inner_iterations"]) != (1, 1):
            bad.append((case.name, p, f"not one step: {r['iterations']}, {r['inner_iterations']}"))
            continue
        if flow:
            ref = SR.flow_step(q, sig, case.lam)
            e1, s1 = SR.flow_objective(q, r["pose"], r["flow"][:P], sig)
            pose_err = [SR.pose_step_error(q["pose_init"], ref["dg"], r["pose"])]
            R_pose = [[1.0]*3 + [1.0 + np.abs(r["pose"][9:]).max()]*3]
            nl, x_in = 2, q["flow"]
        else:
            ref = SR.motion_step(q, sig, case.lam)
            outp = [r["poses"][0], r["poses"][1], r["motion"]]
            e1, s1 = SR.motion_objective(q, outp, r["points"][:P], sig)
            X0 = [q["pose_prev"], q["pose_cur"], q["motion_init"]]
            pose_err = [SR.pose_step_error(X0[v], ref["dg"][6*v:6*v + 6], outp[v]) for v in range(3)]
            R_pose = [[1.0]*3 + [1.0 + np.abs(outp[v][9:]).max()]*3 for v in range(3)]
            nl, x_in = 6, q["points_init"]
        worst["error_final"] = max(worst["error_final"], error_score(r["error_final"], e1, s1))
        _, mult = (SR._distinct(q) if flow else SR._distinct_motion(q))
        off = _local_offsets(mult, len(ref["dg"]), nl)
        D = ref["D"]
        d_err = [float(x) for e in pose_err for x in e]
        Ds = list(D[:len(ref["dg"])]); R = [x for rp in R_pose for x in rp]
        ref_norm2 = sum((float(D[i])*float(ref["dg"][i]))**2 for i in range(len(ref["dg"])))
        for j in range(P):
            for c in range(nl):
                d = (mpf(float(local[j][c])) - mpf(float(x_in[j][c]))) - ref["dl"][j][c]
                d_err.append(float(d)); Ds.append(D[off[j] + c]); R.append(abs(local[j][c]) + abs(x_in[j][c]))
                ref_norm2 += mult[j]*(D[off[j] + c]*float(ref["dl"][j][c]))**2
        s = step_score(d_err, Ds, np.sqrt(ref_norm2), ref["kappa"], ref["rhs_err"], R)
        worst["step"] = max(worst["step"], s)
    return worst, bad
