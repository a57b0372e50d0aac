"""numpy / scipy statement of ObjectMotionSolverFilter's per-object step (dynosam/src/frontend/vision/MotionSolver.cc:1395-1725,
1734-2089), written from the reference's semantics and sharing no code with dynosam_b200/csrc: poses are 4x4 matrices, the
retraction is T expm(xi^) (scipy.linalg.expm), the stereo projection and its pose derivative are GTSAM's StereoCamera::project2
closed form, the update's triangle comes from numpy.linalg.qr of the reference's literal A_qr (zero rows included).

step(obj, params) takes and returns the dicts of dynosam_b200.binding.object_srif_batch.  FilterMap holds what the reference's
filters_ map holds per object (state, tracklet -> m_L, frame_id_e) and makes solveImpl's new / resampled / in-filter decision;
run_sequence drives a backend (this statement, the host build, the device) over a synth_srif sequence."""
from __future__ import annotations

import numpy as np
import scipy.linalg as sl

NEW, RESET, CONTINUE = 0, 1, 2
OK, TOO_FEW, NO_INLIERS = 0, 1, 2
VALID = 0


def default_params():
    return dict(P0=0.3*np.eye(6), Q=0.2*np.eye(6), R_noise=np.eye(3), huber_k=0.1, irls_iterations=2, min_new_inliers=4)


def T4(p):
    T = np.eye(4); T[:3, :3] = np.asarray(p[:9]).reshape(3, 3); T[:3, 3] = p[9:12]
    return T


def p12(T):
    return np.concatenate([T[:3, :3].reshape(9), T[:3, 3]])


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def retract(T, xi):
    M = np.zeros((4, 4)); M[:3, :3] = skew(xi[:3]); M[:3, 3] = xi[3:]
    return T @ sl.expm(M)


def inv(T):
    R, t = T[:3, :3], T[:3, 3]
    Ti = np.eye(4); Ti[:3, :3] = R.T; Ti[:3, 3] = -R.T @ t
    return Ti


def adjoint(T):
    R, t = T[:3, :3], T[:3, 3]
    A = np.zeros((6, 6)); A[:3, :3] = R; A[3:, 3:] = R; A[3:, :3] = skew(t) @ R
    return A


def chol_upper(M):
    return np.linalg.cholesky(M).T


def project2(C, K, m):
    """gtsam::StereoCamera(C, K).project2(m) with its derivative by the pose; None on cheirality (q_z <= 0)"""
    fx, fy, _, u0, v0, b = K
    q = C[:3, :3].T @ (m - C[:3, 3])
    if q[2] <= 0:
        return None
    d = 1.0/q[2]; x, y = q[0], q[1]
    dfx, dfy = d*fx, d*fy
    uL, uR, v = dfx*x, dfx*(x - b), dfy*y
    v1, v2, dx = v/fy, fx*v/fy, d*x
    H1 = np.array([[uL*v1, -fx - dx*uL, v2, -dfx, 0.0, d*uL],
                   [uR*v1, -fx - dx*uR, v2, -dfx, 0.0, d*uR],
                   [fy + v*v1, -dx*v, -x*dfy, 0.0, -dfy, d*v]])
    return np.array([u0 + uL, u0 + uR, v0 + v]), H1


class Srif:
    """HybridObjectMotionSRIF"""

    def __init__(self, state, P):
        s = np.asarray(state, dtype=np.float64)
        self.R = s[:36].reshape(6, 6).copy(); self.d = s[36:42].copy()
        self.H, self.Le, self.prev, self.XK = T4(s[42:54]), T4(s[54:66]), T4(s[66:78]), T4(s[78:90])
        self.P = P

    def record(self):
        return np.concatenate([self.R.reshape(36), self.d, p12(self.H), p12(self.Le), p12(self.prev), p12(self.XK)])

    def reset(self, Le):                                   # :1689-1725
        self.d = np.zeros(6); self.R = chol_upper(np.linalg.inv(self.P["P0"]))
        self.prev = np.eye(4); self.Le = Le; self.XK = np.eye(4); self.H = np.eye(4)

    def delta(self):
        return sl.solve_triangular(self.R, self.d, lower=False)

    def mean(self):
        return retract(self.H, self.delta())

    def cov(self):
        return np.linalg.inv(self.R.T @ self.R)

    def f2f(self):
        return self.mean() @ inv(self.prev)

    def predict(self):                                     # :1445-1482
        Hm, Pc, F = self.mean(), self.cov(), self.f2f()
        self.prev = Hm
        self.H = F @ Hm
        self.d = np.zeros(6)
        self.R = chol_upper(np.linalg.inv(Pc + self.P["Q"]))

    def update(self, X, K, z, valid, pc, m, has):          # :1484-1687
        P = self.P
        n = len(valid)
        self.XK = X
        Xi = inv(X)
        A = Xi @ self.H
        C = inv(A @ self.Le)
        Jc = -adjoint(A)
        Hs = np.zeros((3*n, 6)); ys = np.zeros(3*n)
        Rinv = np.linalg.inv(P["R_noise"])
        e0 = np.zeros(n); rwe = np.zeros(n)
        n_new = 0
        for i in range(n):
            if not has[i]:
                m[i] = (inv(self.Le) @ inv(self.H) @ X @ np.append(pc[i], 1.0))[:3]    # projectToObject3
                has[i] = True; n_new += 1
            if not valid[i]:
                continue
            r = project2(C, K, m[i])
            if r is None:
                continue
            h, J = r
            y = z[i] - h
            Hs[3*i:3*i + 3] = J @ Jc; ys[3*i:3*i + 3] = y
            e0[i] = np.sqrt(y @ Rinv @ y)
        R0, d0 = self.R.copy(), self.d.copy()
        clipped = 0
        for _ in range(P["irls_iterations"]):
            Cc = inv(Xi @ self.mean() @ self.Le)
            w = np.ones(n); clipped = 0
            for i in range(n):
                if not valid[i]:
                    w[i] = 0.0; continue
                r = project2(Cc, K, m[i])
                if r is None:
                    w[i] = 0.0; continue
                y = z[i] - r[0]
                e = np.sqrt(y @ Rinv @ y)
                rwe[i] = e
                w[i] = 1.0 if e <= P["huber_k"] else P["huber_k"]/e
                clipped += not (e <= P["huber_k"])
            Aq = np.zeros((3*n + 6, 7))
            for i in range(n):
                if w[i] < 1e-6:
                    continue
                Li = np.linalg.inv(np.linalg.cholesky(P["R_noise"]/w[i]))
                Aq[3*i:3*i + 3, :6] = Li @ Hs[3*i:3*i + 3]; Aq[3*i:3*i + 3, 6] = Li @ ys[3*i:3*i + 3]
            Aq[3*n:, :6] = R0; Aq[3*n:, 6] = d0
            Rf = np.linalg.qr(Aq, mode="r")
            sg = np.where(np.diag(Rf[:6, :6]) < 0, -1.0, 1.0)
            self.R = np.triu(sg[:, None]*Rf[:6, :6]); self.d = sg*Rf[:6, 6]
        return np.linalg.norm(e0), np.linalg.norm(rwe), n_new, clipped


def step(obj, P=None):
    """one object's step for the frame (solveImpl after its PnP), as binding.object_srif_batch returns it"""
    P = P or default_params()
    mode, K = obj["mode"], np.asarray(obj["calib"], dtype=np.float64)
    z = np.asarray(obj["stereo"], dtype=np.float64).reshape(-1, 6); valid = np.asarray(obj["valid"], dtype=bool).reshape(-1, 2)
    pc = np.asarray(obj["points"], dtype=np.float64).reshape(-1, 6)
    m = np.array(obj["m_L"], dtype=np.float64).reshape(-1, 3); has = np.array(obj["has_point"], dtype=bool).reshape(-1)
    n = len(valid)
    f = Srif(obj["state"], P)
    res = dict(status=OK, solved=False, f2f=p12(np.eye(4)), motion=p12(np.eye(4)), pose=p12(np.eye(4)), cov=np.zeros((6, 6)),
               error=0.0, reweighted_error=0.0, before_reset=p12(np.eye(4)), n_new=0, n_tracked=0, n_clipped=0)
    if mode == NEW and n < P["min_new_inliers"]:
        res["status"] = TOO_FEW
    elif mode != CONTINUE and n == 0:
        res["status"] = NO_INLIERS
    if res["status"] != OK:
        res.update(state=np.asarray(obj["state"], dtype=np.float64).copy(), m_L=m, has_point=has)
        return res
    Xp, Xc = T4(obj["pose_prev"]), T4(obj["pose_cur"])
    if mode != CONTINUE:
        c = pc[:, :3].sum(0)/n                                    # construct_initial_frame (:1768-1787)
        Le = np.eye(4); Le[:3, 3] = (Xp @ np.append(c, 1.0))[:3]
        if mode == RESET:
            res["before_reset"] = p12(f.H)
        f.reset(Le)
        has[:] = False
    n_new = 0
    frames = [(Xp, 0), (Xc, 1)] if mode != CONTINUE else [(Xc, 1)]
    for X, k in frames:
        f.predict()
        e, r, nn, cl = f.update(X, K, z[:, 3*k:3*k + 3], valid[:, k], pc[:, 3*k:3*k + 3], m, has)
        n_new += nn
    Hm = f.mean()
    res.update(solved=obj.get("pnp_status", VALID) == VALID, f2f=p12(f.f2f()), motion=p12(Hm), pose=p12(Hm @ f.Le), cov=f.cov(),
               error=e, reweighted_error=r, n_new=n_new, n_tracked=n - n_new, n_clipped=cl, state=f.record(), m_L=m, has_point=has)
    return res


def reference_batch(objects, **P):
    p = default_params(); p.update(P)
    return [step(o, p) for o in objects]


class FilterMap:
    """the reference's filters_ map: per object the filter record, its tracklet -> m_L map and frame_id_e"""

    def __init__(self):
        self.filters = {}

    def objects(self, seq, k):
        """the batch objects of frame k (k >= 1) of a synth_srif sequence, with solveImpl's mode decision (:1795-1912)"""
        out = []
        for rec in seq["frames"][k - 1]:
            oid = rec["object_id"]
            f = self.filters.get(oid)
            mode = NEW if f is None else (RESET if rec["resampled"] else CONTINUE)
            pts = f["points"] if f is not None else {}
            tr = rec["tracklets"]
            out.append(dict(object_id=oid, tracklets=tr, mode=mode, pnp_status=rec["pnp_status"], pose_prev=seq["poses"][k - 1],
                            pose_cur=seq["poses"][k], calib=seq["calib"],
                            state=f["state"] if f is not None else np.zeros(90), stereo=rec["stereo"], valid=rec["valid"],
                            points=rec["points"], m_L=np.array([pts.get(int(t), np.zeros(3)) for t in tr]).reshape(-1, 3),
                            has_point=np.array([int(t) in pts for t in tr], dtype=bool)))
        return out

    def absorb(self, objects, results, k):
        for o, r in zip(objects, results):
            if r["status"] != OK:
                continue
            oid = o["object_id"]
            f = self.filters.setdefault(oid, dict(points={}, frame_id_e=k))
            if o["mode"] != CONTINUE:
                f["points"] = {}; f["frame_id_e"] = k            # resetState clears m_linearized_; the fake key frame is k
            f["state"] = r["state"]
            for t, m, h in zip(o["tracklets"], r["m_L"], r["has_point"]):
                if h:
                    f["points"][int(t)] = m


def run_sequence(seq, backend):
    """[(objects, results)] of every frame, the backend called once per frame on all of its objects"""
    fm = FilterMap()
    out = []
    for k in range(1, len(seq["poses"])):
        objs = fm.objects(seq, k)
        res = backend(objs)
        fm.absorb(objs, res, k)
        out.append((objs, res))
    return out
