"""CPU restatement of the front end's small per-object refinements (TEST INFRASTRUCTURE, NOT PRODUCT).

(1) flow_pose_lm / flow_pose_refine follow OpticalFlowAndPoseOptimizer::optimize
    (dynosam/include/dynosam/frontend/vision/MotionSolver-inl.hpp:88-278): per feature a Pose3FlowProjectionFactor (Robust Huber
    over Isotropic flow_sigma) and a PriorFactor<Point2> on the flow (Isotropic flow_prior_sigma), one Pose3 unknown,
    gtsam::LevenbergMarquardtOptimizer with maxIterations 10, then up to four outlier rounds (:201-247) driven by
    factor_graph_tools::determineFactorOutliers (dynosam_opt/include/dynosam_opt/FactorGraphTools.hpp:74-111).
(2) motion_refine_lm follows MotionOnlyRefinementOptimizer::optimize (:291-470, ProjectionError solver): two camera poses with
    tight priors, the object motion, two world points per tracklet; GenericProjectionFactor x2 + LandmarkMotionTernaryFactor per
    tracklet, LM with maxIterations 5.

Residuals / Jacobians of the DynOSAM factors come from the C oracle (orc_linearize_block: Pose3FlowProjectionFactor.h:73-133,
LandmarkMotionTernaryFactor.cc:41-72, pinned by tests/test_oracle_kat.py); gtsam::GenericProjectionFactor is restated here in
numpy (GTSAM 4.2 PinholeCamera::project: CalibratedCamera Dpose / Dpoint, Cal3_S2::uncalibrate) and pinned by numerical
differentiation in tests/test_star.py.  The damped normal equations are formed DENSE and solved by Cholesky, and the outer loop
is LevenbergMarquardtOptimizer::iterate / tryLambda (SURVEY Appendix A.4) written out literally.
PARITY UNPINNED by the reference's own tests: the reference holds no test, golden vector or fixture for either optimiser (only
their call sites), so the LM runs restated here are anchored on the factor KATs above, on GTSAM 4.2's published control flow and
on the properties checked in tests/test_star.py (ground truth recovered on noise-free problems, numerical Jacobians).
Only tests/ may import this module.
"""
from __future__ import annotations

import numpy as np

from dynosam_b200.problem import FLOWPROJ2, PRIOR6, TERNARY3, FactorBlock, Problem

from . import oracle as orc

DEFAULTS = dict(lambda_initial=1e-5, lambda_factor=10.0, lambda_upper_bound=1e5, lambda_lower_bound=0.0,
                min_model_fidelity=1e-3, relative_error_tol=1e-5, absolute_error_tol=1e-5, error_tol=0.0,
                max_iterations=100)
CHI2_99 = {2: 9.210340371976184, 3: 11.344866730144373}      # chi_squared_quantile(dim, 0.99)


EPS = np.finfo(float).eps


def _margin(x, scale):
    return abs(x)/scale if scale > 0 else np.inf


def _equilibrated_kappa(H, lam):
    """kappa of D^-1 (H + lam I) D^-1, D the square root of its diagonal -- the condition that bounds a Cholesky solve's
    error whatever the scaling of the unknowns; taken at the first lambda of a linearisation (a larger lambda only improves it)"""
    Hd = H + lam*np.eye(H.shape[0])
    if not H.size or not np.isfinite(Hd).all() or not (np.diag(Hd) > 0).all():
        return np.inf
    d = 1.0/np.sqrt(np.diag(Hd))
    ev = np.linalg.eigvalsh(Hd*np.outer(d, d))
    return ev[-1]/ev[0] if ev[0] > 0 else np.inf


def near_decision(trace, factor=64.0):
    """the first decision of an LM trace whose margin lies within `factor` times its step bound (eps kappa of the damped
    system it was taken on), or None: an implementation whose steps differ from this one's by rounding may decide it the
    other way, so a different (iterations, inner) is a last-digit decision only when such a decision exists"""
    for i, t in enumerate(trace):
        for k in ("fidelity", "stop", "relative", "absolute"):
            if k in t and t[k] <= factor*t["bound"]:
                return i, k, t[k], t["bound"]
    return None


def dense_lm(error, linear_system, get_state, set_state, step, **kw):
    """LevenbergMarquardtOptimizer::optimize on callbacks: error() at the current values, linear_system() -> whitened (A, b) at
    the current values, step(delta) retracts the current values, get/set_state snapshot them.

    `trace` records every decision with its margin, relative to the magnitudes it compares: per inner iteration the model
    fidelity against min_model_fidelity and |cost| against relative_error_tol * err, per outer iteration the relative and
    absolute decrease against their tolerances; `bound` is eps * kappa of the equilibrated damped system, the relative size of
    a difference rounding may make in the step and so in the compared errors.
    `ended` names what ended the loop."""
    P = dict(DEFAULTS); P.update(kw)
    err = error(); err0 = err
    lam = P["lambda_initial"]; iterations = inner = 0
    trace = []; ended = "error_tol" if err <= P["error_tol"] else ("max_iterations" if P["max_iterations"] <= 0 else None)
    if not (err <= P["error_tol"]) and P["max_iterations"] > 0:
        new_error = err
        while True:
            current_error = new_error
            A, b = linear_system()
            H = A.T @ A; g = A.T @ b
            kappa = _equilibrated_kappa(H, lam)
            while True:      # tryLambda
                rec = dict(lam=lam, bound=EPS*kappa)
                solved = True
                try:
                    L = np.linalg.cholesky(H + lam*np.eye(H.shape[0]))
                    delta = np.linalg.solve(L.T, np.linalg.solve(L, g))
                except np.linalg.LinAlgError:
                    solved = False
                success = stop = False; nerr = np.inf
                if solved:
                    old_lin = 0.5*float(b @ b); rr = A @ delta - b; lin = old_lin - 0.5*float(rr @ rr)
                    if np.isfinite(lin) and lin >= 0:
                        keep = get_state()
                        step(delta)
                        nerr = error(); cost = err - nerr
                        scale = abs(err) + abs(nerr)
                        if lin > np.finfo(float).eps*old_lin:
                            success = cost/lin > P["min_model_fidelity"]
                            rec["fidelity"] = _margin(cost - P["min_model_fidelity"]*lin, scale + abs(P["min_model_fidelity"]*lin))
                        if abs(cost) < P["relative_error_tol"]*err:
                            stop = True
                        if P["relative_error_tol"] > 0:
                            rec["stop"] = _margin(abs(cost) - P["relative_error_tol"]*err, scale)
                        if not success:
                            set_state(keep)
                trace.append(rec)
                if success:
                    lam = max(P["lambda_lower_bound"], lam/P["lambda_factor"]); err = nerr; iterations += 1; inner += 1
                    break
                elif not stop:
                    lam *= P["lambda_factor"]; inner += 1
                    if lam >= P["lambda_upper_bound"]:
                        break
                else:
                    break
            new_error = err
            with np.errstate(all="ignore"):
                rel = np.float64(current_error - new_error)/np.float64(current_error)
            done = (new_error <= P["error_tol"]) or (P["relative_error_tol"] != 0.0 and rel <= P["relative_error_tol"]) \
                or ((current_error - new_error) <= P["absolute_error_tol"])
            scale = abs(current_error) + abs(new_error)
            rec = dict(bound=trace[-1]["bound"] if trace else EPS)
            if P["relative_error_tol"] != 0.0 and np.isfinite(rel):
                rec["relative"] = _margin((current_error - new_error) - P["relative_error_tol"]*current_error, scale)
            rec["absolute"] = _margin((current_error - new_error) - P["absolute_error_tol"], scale + abs(P["absolute_error_tol"]))
            trace.append(rec)
            if not (iterations < P["max_iterations"] and not done and np.isfinite(current_error)):
                ended = ("error_tol" if new_error <= P["error_tol"] else
                         "relative" if P["relative_error_tol"] != 0.0 and rel <= P["relative_error_tol"] else
                         "absolute" if (current_error - new_error) <= P["absolute_error_tol"] else
                         "nonfinite" if not np.isfinite(current_error) else "max_iterations")
                break
    return dict(error_initial=err0, error_final=err, iterations=iterations, inner_iterations=inner, trace=trace, ended=ended)


# ------------------------------------------------------------------------------------------------ (1) flow + pose
class _FlowPose:
    def __init__(self, pose_init, pose_prev, calib5, kp_prev, depth, flow, flow_sigma, flow_prior_sigma, huber_k):
        n = self.n = len(depth)
        kp_prev = np.asarray(kp_prev, dtype=np.float64).reshape(n, 2); self.flow0 = np.asarray(flow, dtype=np.float64).reshape(n, 2).copy()
        meas = np.concatenate([kp_prev, np.asarray(depth, dtype=np.float64).reshape(n, 1), np.tile(np.asarray(pose_prev).reshape(1, 12), (n, 1))], 1)
        blk = FactorBlock(FLOWPROJ2, np.stack([np.arange(n), np.zeros(n, dtype=int)], 1), meas, np.array([flow_sigma]), float(huber_k))
        gblk = FactorBlock(FLOWPROJ2, blk.idx, meas, np.array([flow_sigma]), 0.0)             # the same factors with the Gaussian noise model
        prob = Problem(np.asarray(pose_init, dtype=np.float64).reshape(1, 12), np.zeros((0, 3)), flow=self.flow0.copy(),
                       calib=np.concatenate([np.asarray(calib5, dtype=np.float64), [0.0]]), blocks=[blk, gblk])
        self.o = orc.OracleProblem(prob)
        self.isp = 1.0/flow_prior_sigma
        self.active = np.ones(n, dtype=bool)

    def error(self):
        o = self.o
        e = float(o.error_block(0)[self.active].sum()) if self.n else 0.0
        return e + 0.5*float((((o.flow - self.flow0)*self.isp)**2).sum())

    def linear_system(self):
        n, o, isp = self.n, self.o, self.isp
        A = np.zeros((4*n, 2*n + 6)); b = np.zeros(4*n)
        if n:
            Af, bf = o.linearize_block(0)          # whitened, Huber-weighted: [n,2,8] (flow 2 | pose 6), [n,2]
            for i in range(n):
                if self.active[i]:
                    A[2*i:2*i + 2, 2*i:2*i + 2] = Af[i, :, 0:2]; A[2*i:2*i + 2, 2*n:] = Af[i, :, 2:8]; b[2*i:2*i + 2] = bf[i]
                A[2*n + 2*i:2*n + 2*i + 2, 2*i:2*i + 2] = isp*np.eye(2); b[2*n + 2*i:2*n + 2*i + 2] = -(o.flow[i] - self.flow0[i])*isp
        return A, b

    def get_state(self): return self.o.pose.copy(), self.o.flow.copy()
    def set_state(self, s): self.o.pose[:] = s[0]; self.o.flow[:] = s[1]

    def step(self, delta):
        n, o = self.n, self.o
        o.pose[0] = orc.se3_retract(o.pose[0], delta[2*n:]); o.flow += delta[:2*n].reshape(n, 2)

    def gaussian_errors(self):
        return self.o.error_block(1) if self.n else np.zeros(0)


def flow_pose_lm(pose_init, pose_prev, calib5, kp_prev, depth, flow, flow_sigma, flow_prior_sigma, huber_k, **kw):
    """one LM, no outlier rounds"""
    return flow_pose_refine(pose_init, pose_prev, calib5, kp_prev, depth, flow, flow_sigma, flow_prior_sigma, huber_k, outlier_rounds=0, **kw)


def flow_pose_refine(pose_init, pose_prev, calib5, kp_prev, depth, flow, flow_sigma, flow_prior_sigma, huber_k, outlier_rounds=4,
                     outlier_threshold=None, **kw):
    q = _FlowPose(pose_init, pose_prev, calib5, kp_prev, depth, flow, flow_sigma, flow_prior_sigma, huber_k)
    thr = 0.5*CHI2_99[2] if not outlier_threshold or outlier_threshold <= 0 else outlier_threshold
    X0 = q.o.pose[0].copy()
    r = dense_lm(q.error, q.linear_system, q.get_state, q.set_state, q.step, **kw)
    err_before = r["error_initial"]; its, inner, rounds = r["iterations"], r["inner_iterations"], 0
    trace = list(r["trace"]); ended = "no_rounds"
    if outlier_rounds > 0:
        out = q.active & (q.gaussian_errors() > thr)
        ended = "no_outliers"
        if out.any():
            for _ in range(outlier_rounds):
                q.active &= ~out
                q.o.pose[0] = X0                                  # optimised_values.update(pose_key, initial_pose)
                r = dense_lm(q.error, q.linear_system, q.get_state, q.set_state, q.step, **kw)
                its += r["iterations"]; inner += r["inner_iterations"]; rounds += 1; trace += r["trace"]
                out = q.active & (q.gaussian_errors() > thr)
                if not out.any():
                    break
            ended = "cap" if out.any() else "no_outliers"
    return dict(pose=q.o.pose[0].copy(), flow=q.o.flow.copy(), inlier=q.active.copy(), error_initial=err_before, error_final=r["error_final"],
                iterations=its, inner_iterations=inner, rounds=rounds, trace=trace, ended=ended, lm_ended=r["ended"])


# ------------------------------------------------------------------------------------------------ (2) object motion
def projection_factor(X, p, K5, z):
    """gtsam::GenericProjectionFactor<Pose3, Point3, Cal3_S2>::evaluateError with throwCheirality = false: unwhitened residual,
    d/dpose (2x6, [omega, v]), d/dpoint (2x3)"""
    X = np.asarray(X); R = X[:9].reshape(3, 3); t = X[9:]
    fx, fy, s, u0, v0 = K5
    q = R.T @ (np.asarray(p) - t)
    if q[2] <= 0:
        return np.full(2, 2.0*fx), np.zeros((2, 6)), np.zeros((2, 3))
    d = 1.0/q[2]; u = q[0]*d; v = q[1]*d
    Dpose = np.array([[u*v, -1 - u*u, v, -d, 0, d*u], [1 + v*v, -u*v, -u, 0, -d, d*v]])
    Rt = R.T
    Dpoint = d*np.array([Rt[0] - u*Rt[2], Rt[1] - v*Rt[2]])
    Dcal = np.array([[fx, s], [0, fy]])
    r = np.array([fx*u + s*v + u0 - z[0], fy*v + v0 - z[1]])
    return r, Dcal @ Dpose, Dcal @ Dpoint


def _robust(r, sigma, k):
    """noiseModel::Robust(Huber(k), Isotropic(sigma)): whitened residual, sqrt(weight), factor error"""
    rw = r/sigma; n = float(np.linalg.norm(rw))
    if k > 0 and n > k:
        return rw, np.sqrt(k/n), k*(n - 0.5*k)
    return rw, 1.0, 0.5*n*n


class _MotionRefine:
    def __init__(self, pose_prev, pose_cur, motion_init, calib5, kp_prev, kp_cur, points_init, sig_motion, sig_proj, huber_k, sig_prior):
        n = self.n = len(kp_prev)
        self.K5 = np.asarray(calib5, dtype=np.float64); self.kpa = np.asarray(kp_prev, dtype=np.float64).reshape(n, 2); self.kpb = np.asarray(kp_cur, dtype=np.float64).reshape(n, 2)
        self.sm, self.sp, self.k, self.spr = sig_motion, sig_proj, huber_k, sig_prior
        pts = np.asarray(points_init, dtype=np.float64).reshape(n, 6)
        poses = np.stack([np.asarray(pose_prev, dtype=np.float64).reshape(12), np.asarray(pose_cur, dtype=np.float64).reshape(12), np.asarray(motion_init, dtype=np.float64).reshape(12)])
        # C-oracle part: points 2i (k-1), 2i+1 (k); ternary(prev pt, cur pt, motion = pose 2); priors on poses 0, 1
        tern = FactorBlock(TERNARY3, np.stack([2*np.arange(n), 2*np.arange(n) + 1, np.full(n, 2)], 1), None, np.array([sig_motion]), float(huber_k))
        gtern = FactorBlock(TERNARY3, tern.idx, None, np.array([sig_motion]), 0.0)
        pri = FactorBlock(PRIOR6, np.array([[0], [1]]), poses[:2].copy(), np.full(6, sig_prior))
        prob = Problem(poses.copy(), pts.reshape(2*n, 3).copy(), calib=np.concatenate([self.K5, [0.0]]), blocks=[tern, gtern, pri])
        self.o = orc.OracleProblem(prob)

    def _proj(self):
        o = self.o
        for i in range(self.n):
            yield i, 0, projection_factor(o.pose[0], o.point[2*i], self.K5, self.kpa[i])
            yield i, 1, projection_factor(o.pose[1], o.point[2*i + 1], self.K5, self.kpb[i])

    def error(self):
        o = self.o
        e = (float(o.error_block(0).sum()) if self.n else 0.0) + float(o.error_block(2).sum())
        for _, _, (r, _, _) in self._proj():
            e += _robust(r, self.sp, self.k)[2]
        return e

    def linear_system(self):
        # unknowns: points (6n: m_a_i, m_b_i interleaved as the C oracle's point array), then X_a, X_b, H (18)
        n, o = self.n, self.o
        npt = 6*n
        A = np.zeros((7*n + 12, npt + 18)); b = np.zeros(7*n + 12)
        if n:
            At, bt = o.linearize_block(0)          # [n,3,12]: prev pt (3) | cur pt (3) | motion (6)
            for i in range(n):
                r0 = 7*i
                A[r0 + 4:r0 + 7, 6*i:6*i + 6] = At[i, :, 0:6]; A[r0 + 4:r0 + 7, npt + 12:] = At[i, :, 6:12]; b[r0 + 4:r0 + 7] = bt[i]
            for i, which, (r, Jx, Jp) in self._proj():
                rw, sw, _ = _robust(r, self.sp, self.k)
                r0 = 7*i + 2*which
                A[r0:r0 + 2, npt + 6*which:npt + 6*which + 6] = sw*Jx/self.sp
                A[r0:r0 + 2, 6*i + 3*which:6*i + 3*which + 3] = sw*Jp/self.sp
                b[r0:r0 + 2] = -sw*rw
        Ap, bp = o.linearize_block(2)              # [2,6,6], [2,6]
        for v in range(2):
            A[7*n + 6*v:7*n + 6*v + 6, npt + 6*v:npt + 6*v + 6] = Ap[v]; b[7*n + 6*v:7*n + 6*v + 6] = bp[v]
        return A, b

    def get_state(self): return self.o.pose.copy(), self.o.point.copy()
    def set_state(self, s): self.o.pose[:] = s[0]; self.o.point[:] = s[1]

    def step(self, delta):
        n, o = self.n, self.o
        o.point += delta[:6*n].reshape(2*n, 3)
        for v in range(3):
            o.pose[v] = orc.se3_retract(o.pose[v], delta[6*n + 6*v:6*n + 6*v + 6])


def motion_refine_lm(pose_prev, pose_cur, motion_init, calib5, kp_prev, kp_cur, points_init, landmark_motion_sigma=0.001,
                     projection_sigma=2.0, huber_k=0.0001, pose_prior_sigma=0.00001, **kw):
    kw.setdefault("max_iterations", 5)
    q = _MotionRefine(pose_prev, pose_cur, motion_init, calib5, kp_prev, kp_cur, points_init, landmark_motion_sigma, projection_sigma, huber_k, pose_prior_sigma)
    r = dense_lm(q.error, q.linear_system, q.get_state, q.set_state, q.step, **kw)
    r.update(motion=q.o.pose[2].copy(), poses=q.o.pose[:2].copy(), points=q.o.point.reshape(q.n, 6).copy(),
             motion_factor_error=q.o.error_block(1) if q.n else np.zeros(0))
    return r
