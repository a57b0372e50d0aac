"""A 50-digit reference of the two per-object LM problems of csrc/kernels_star.cu: the joint optical-flow + pose problem
(OpticalFlowAndPoseOptimizer) and the object-motion problem (MotionOnlyRefinementOptimizer).  Built on lie_reference.py
(FLOWPROJ2, TERNARY3, PRIOR6, `whiten`, the maps); it imports neither the CUDA library nor the CPU oracle.

What it adds is gtsam::GenericProjectionFactor<Pose3, Point3, Cal3_S2> (skew included; behind the camera, q_z <= 0: residual
(2 fx, 2 fx) and zero Jacobians; its Jacobian by 50-digit central differences through the true retraction) and, for one
problem at given values:

* `flow_objective` / `motion_objective`: the graph's error (Huber, the factors removed by outlier rounds left out) and its
  a-priori rounding scale;
* `flow_step` / `motion_step`: the whitened damped normal equations at lambda (lambda I, GTSAM's default), eliminated block by block --
  the flows / the two points of a tracklet are local to one block, so the cost is linear in N -- the step, oldLin, newLin,
  and kappa of the equilibrated damped system (fp64, from the reference's matrix).

A problem's features may tile a period of distinct features (`period`): every copy of a distinct feature has the same
linearisation, so the reference evaluates it once and weights it by its multiplicity.  Raw residuals and Jacobians are
cached per (values, feature), so cases that only change sigmas, Huber k or lambda reuse them.
"""
import numpy as np
import scipy.sparse as sp
from mpmath import mp, mpf
from scipy.sparse.linalg import eigsh

import lie_reference as LR
from lie_reference import FLOWPROJ2, PRIOR6, TERNARY3

EPS = 2.0**-52
_CACHE = {}


def _key(*arrays):
    return b"".join(np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes() for a in arrays)


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


# ---- gtsam::GenericProjectionFactor<Pose3, Point3, Cal3_S2> (throwCheirality = false)
def projection(T, p, K):
    """(pixel, camera-frame point) of the world point p seen from pose T; pixel None behind the camera"""
    q = LR.act_inv(T, p)
    if q[2] <= 0:
        return None, q
    u, v = q[0]/q[2], q[1]/q[2]
    return [K[0]*u + K[2]*v + K[3], K[1]*v + K[4]], q


def projection_residual(T, p, K, z):
    uv, _ = projection(T, p, K)
    return [2*K[0]]*2 if uv is None else [a - b for a, b in zip(uv, z)]


def projection_jacobian(T, p, K, z):
    """2 x 9: pose [omega, v] (6) | point (3), the exact derivative by central differences (step 1e-20) through the true
    retraction; zero behind the camera"""
    if projection(T, p, K)[0] is None:
        return [[mpf(0)]*9 for _ in range(2)]
    d = mpf("1e-20"); cols = []
    for j in range(9):
        if j < 6:
            xi = [mpf(0)]*6; xi[j] = d; a = projection_residual(LR.retract(T, xi), p, K, z)
            xi[j] = -d; b = projection_residual(LR.retract(T, xi), p, K, z)
        else:
            pp = list(p); pp[j - 6] += d; a = projection_residual(T, pp, K, z)
            pp[j - 6] -= 2*d; b = projection_residual(T, pp, K, z)
        cols.append([(x - y)/(2*d) for x, y in zip(a, b)])
    return [[c[i] for c in cols] for i in range(2)]


def _camera_scale(T, p, K, q):
    """magnitude of the terms of a projected pixel that cancel in its residual (rounding scale of the residual)"""
    f = abs(K[0]) + abs(K[1]) + abs(K[2])
    qz = max(abs(q[2]), mpf("1e-300"))
    uv = (abs(q[0]) + abs(q[1]))/qz
    mag = max(abs(x) for x in list(p) + list(T[1]))
    return abs(K[3]) + abs(K[4]) + f*(uv + (1 + uv)*3*mag/qz)


def _rho(n, k):
    """d(Huber loss)/dn"""
    return n if (k <= 0 or n <= k) else mpf(k)


# ---- one block of rows: the factors of one feature / tracklet
class Rows:
    """whitened rows of one block: A_g (global columns), A_l (the block's own columns), b, rounding scale S of each row,
    the block's error and its rounding scale"""
    def __init__(self, ng, nl):
        self.Ag, self.Al, self.b, self.S = [], [], [], []
        self.ng, self.nl = ng, nl
        self.err = mpf(0); self.err_scale = mpf(0)

    def add(self, r, J, gcols, lcols, sigma, k, scale):
        """r: unwhitened residual, J: its Jacobian (columns mapped by gcols / lcols: lists of (J column, target column))"""
        rw, sw, e = LR.whiten(r, [mpf(sigma)], mpf(k))
        n = mp.sqrt(LR.dot(rw, rw))
        self.err += e; self.err_scale += e + _rho(n, k)*scale/sigma
        for i in range(len(r)):
            g = [mpf(0)]*self.ng; l = [mpf(0)]*self.nl
            if J is not None:
                for jc, tc in gcols:
                    g[tc] = J[i][jc]*sw/sigma
                for jc, tc in lcols:
                    l[tc] = J[i][jc]*sw/sigma
            self.Ag.append(g); self.Al.append(l); self.b.append(-rw[i]*sw); self.S.append(sw*scale/sigma)


def _mat(rows, ncol):
    return mp.matrix(rows) if rows else mp.matrix(0, ncol)


def eliminate(blocks, mult, glob, ng, lam):
    """the damped normal equations (A^T A + lam I) d = A^T b of global columns (ng) + per-block local columns, the blocks
    eliminated one by one.  blocks[j]: Rows, mult[j]: its multiplicity, glob: Rows of global-only factors (priors).
    Returns dict(dg, dl[j], old_lin, new_lin, kappa, rhs_err (D-scaled 2-norm of the step error that the residuals'
    rounding alone may cause), D (sqrt of the damped diagonal, global | local per block))."""
    lam = mpf(lam)
    S = mp.zeros(ng, ng); gs = mp.zeros(ng, 1)
    old = mpf(0); pre = []
    for Bk, m in zip(blocks + [glob], list(mult) + [1]):
        Ag, b = _mat(Bk.Ag, ng), mp.matrix(Bk.b) if Bk.b else mp.zeros(0, 1)
        if not Bk.b:
            pre.append(None); continue
        old += m*sum(x*x for x in Bk.b)/2
        S += m*(Ag.T*Ag); gs += m*(Ag.T*b)
        if Bk.nl == 0:
            pre.append(None); continue
        Al = _mat(Bk.Al, Bk.nl)
        Hll = Al.T*Al + lam*mp.eye(Bk.nl); Hlp = Al.T*Ag; gl = Al.T*b
        Hinv = mp.inverse(Hll)
        S -= m*(Hlp.T*Hinv*Hlp); gs -= m*(Hlp.T*Hinv*gl)
        pre.append((Ag, Al, b, Hll, Hlp, gl, Hinv))
    S += lam*mp.eye(ng)
    dg = mp.lu_solve(S, gs)
    new = mpf(0); dl = []
    for Bk, m, P in zip(blocks + [glob], list(mult) + [1], pre):
        if P is None:
            if Bk.b:
                rr = _mat(Bk.Ag, ng)*dg - mp.matrix(Bk.b); new += m*sum(x*x for x in rr)/2
            dl.append(None); continue
        Ag, Al, b, Hll, Hlp, gl, Hinv = P
        d = Hinv*(gl - Hlp*dg)
        rr = Ag*dg + Al*d - b; new += m*sum(x*x for x in rr)/2
        dl.append(d)
    kappa, lmin, D, rhs = _conditioning(blocks, mult, glob, ng, float(lam))
    return dict(dg=[dg[i] for i in range(ng)], dl=[None if d is None else [d[i] for i in range(d.rows)] for d in dl[:-1]],
                old_lin=old, new_lin=new, kappa=kappa, lam_min=lmin, D=D, rhs_err=rhs)


def _conditioning(blocks, mult, glob, ng, lam):
    """kappa of D^-1 (A^T A + lam I) D^-1 (D = sqrt of its diagonal), its smallest eigenvalue, D, and the D-scaled 2-norm
    bound ||D^-1 |A|^T beta|| / lambda_min of the step error caused by rounding beta = eps S of the right-hand side"""
    rows, cols, vals = [], [], []
    r0 = 0; c0 = ng; beta = []
    copies = []
    for Bk, m in zip(blocks, mult):
        Ag = np.array(LR.to_float(Bk.Ag)).reshape(len(Bk.b), ng); Al = np.array(LR.to_float(Bk.Al)).reshape(len(Bk.b), Bk.nl)
        copies.append((Ag, Al, np.array(LR.to_float(Bk.S)), m))
    nrow = sum(len(a[0])*a[3] for a in copies) + len(glob.b)
    ncol = ng + sum(a[1].shape[1]*a[3] for a in copies)
    for Ag, Al, Sv, m in copies:
        for _ in range(m):
            nr, nl = Al.shape
            for i in range(nr):
                for j in range(ng):
                    if Ag[i, j]:
                        rows.append(r0 + i); cols.append(j); vals.append(Ag[i, j])
                for j in range(nl):
                    if Al[i, j]:
                        rows.append(r0 + i); cols.append(c0 + j); vals.append(Al[i, j])
            beta.append(Sv); r0 += nr; c0 += nl
    if glob.b:
        Ag = np.array(LR.to_float(glob.Ag)).reshape(len(glob.b), ng)
        for i in range(len(glob.b)):
            for j in range(ng):
                if Ag[i, j]:
                    rows.append(r0 + i); cols.append(j); vals.append(Ag[i, j])
        beta.append(np.array(LR.to_float(glob.S))); r0 += len(glob.b)
    A = sp.csr_matrix((vals, (rows, cols)), shape=(nrow, ncol))
    H = (A.T @ A + lam*sp.identity(ncol)).tocsc()
    D = np.sqrt(H.diagonal())
    Di = sp.diags(1.0/D)
    Hs = (Di @ H @ Di).tocsc()
    if ncol <= 1500:
        ev = np.linalg.eigvalsh(Hs.toarray()); lmin, lmax = ev[0], ev[-1]
    else:
        lmax = eigsh(Hs, k=1, which="LA", return_eigenvectors=False)[0]
        lmin = eigsh(Hs, k=1, sigma=0, which="LM", return_eigenvectors=False)[0]
    beta = np.concatenate(beta) if beta else np.zeros(0)
    rhs = np.linalg.norm((abs(A).T @ beta)/D)*EPS/max(lmin, 1e-300)
    return lmax/lmin, lmin, D, rhs


# ---- (1) joint optical flow + pose
def _flow_raw(X, Xprev, K5, kp, depth, flow, jac=True):
    """unwhitened (residual, 2 x 8 Jacobian [flow 2 | pose 6] or None, rounding scale) of one Pose3FlowProjectionFactor"""
    def f():
        K = LR.vec(K5) + [mpf(0)]
        z = LR.vec(kp) + LR.vec([depth]) + LR.vec(Xprev)
        v = [LR.vec(flow), LR.pose(X)]
        r = LR.residual(FLOWPROJ2, v, z, None, K)
        J = LR.jacobian_gtsam(FLOWPROJ2, v, z, None, K) if jac else None
        q = LR.camera_point(FLOWPROJ2, v, z, None, K)
        pw = LR.act(v[1], q)
        sc = abs(z[0]) + abs(z[1]) + abs(v[0][0]) + abs(v[0][1]) + _camera_scale(v[1], pw + list(z[12:15]), K, q)
        return r, J, sc
    return _cached(_key(X, Xprev, K5, kp, [depth], flow, [jac]), f)


def _flow_rows(q, X, flows, j, sig, active, jac=True):
    kp, d = q["kp_prev"][j], q["depth"][j]
    R = Rows(6, 2)
    if active[j]:
        r, J, sc = _flow_raw(X, q["pose_prev"], q["calib"], kp, d, flows[j], jac)
        R.add(r, J, [(2 + c, c) for c in range(6)], [(0, 0), (1, 1)], sig[0], sig[2], sc)
    f, f0 = LR.vec(flows[j]), LR.vec(q["flow"][j])
    R.add([a - b for a, b in zip(f, f0)], [[mpf(1), mpf(0)], [mpf(0), mpf(1)]], [], [(0, 0), (1, 1)], sig[1], 0.0,
          abs(f[0]) + abs(f[1]) + abs(f0[0]) + abs(f0[1]))
    return R


def _distinct(q):
    n = len(q["depth"]); P = q.get("period") or n
    P = min(P, n)
    mult = [len(range(j, n, P)) for j in range(P)]
    return P, mult


def flow_objective(q, X, flows, sig, active=None):
    """(error, rounding scale) of the flow + pose graph at pose X and the distinct features' flows [P, 2]"""
    P, mult = _distinct(q)
    active = np.ones(P, bool) if active is None else active
    e = s = mpf(0)
    for j in range(P):
        R = _flow_rows(q, X, flows, j, sig, active, jac=False)
        e += mult[j]*R.err; s += mult[j]*R.err_scale
    return e, s


def flow_step(q, sig, lam, active=None):
    """the damped step at the initial values: dict(dg = pose step (6), dl = flow steps [P][2], old_lin, new_lin, kappa, ...)"""
    P, mult = _distinct(q)
    active = np.ones(P, bool) if active is None else active
    blocks = [_flow_rows(q, q["pose_init"], q["flow"], j, sig, active) for j in range(P)]
    return eliminate(blocks, mult, Rows(6, 0), 6, lam)


# ---- (2) object motion
def _motion_raw(Xa, Xb, H, K5, kpa, kpb, m, jac=True):
    """unwhitened (residual, Jacobian, scale) of the two projection factors and the motion factor of one tracklet"""
    def f():
        K = LR.vec(K5); Ta, Tb, TH = LR.pose(Xa), LR.pose(Xb), LR.pose(H)
        ma, mb = LR.vec(m[:3]), LR.vec(m[3:])
        out = []
        for T, p, z in ((Ta, ma, LR.vec(kpa)), (Tb, mb, LR.vec(kpb))):
            r = projection_residual(T, p, K, z); J = projection_jacobian(T, p, K, z) if jac else None
            out.append((r, J, abs(z[0]) + abs(z[1]) + _camera_scale(T, p, K, LR.act_inv(T, p))))
        r = LR.residual(TERNARY3, [ma, mb, TH], None, None, K + [mpf(0)])
        J = LR.jacobian_gtsam(TERNARY3, [ma, mb, TH], None, None, K + [mpf(0)]) if jac else None
        out.append((r, J, 3*max(abs(x) for x in ma + mb + TH[1])))
        return out
    return _cached(_key(Xa, Xb, H, K5, kpa, kpb, m, [jac]), f)


def _motion_rows(q, poses, pts, j, sig, jac=True):
    """sig = (landmark_motion_sigma, projection_sigma, huber_k, pose_prior_sigma); global columns X_a | X_b | H"""
    (ra, Ja, sa), (rb, Jb, sb), (rt, Jt, st) = _motion_raw(poses[0], poses[1], poses[2], q["calib"], q["kp_prev"][j], q["kp_cur"][j], pts[j], jac)
    R = Rows(18, 6)
    R.add(ra, Ja, [(c, c) for c in range(6)], [(6 + c, c) for c in range(3)], sig[1], sig[2], sa)
    R.add(rb, Jb, [(c, 6 + c) for c in range(6)], [(6 + c, 3 + c) for c in range(3)], sig[1], sig[2], sb)
    R.add(rt, Jt, [(6 + c, 12 + c) for c in range(6)], [(c, c) for c in range(6)], sig[0], sig[2], st)
    return R


def _prior_rows(q, poses, sig):
    R = Rows(18, 0)
    for v, key in ((0, "pose_prev"), (1, "pose_cur")):
        z = LR.vec(q[key]); T = LR.pose(poses[v])
        r = LR.residual(PRIOR6, [T], z, None, None)
        J = LR.jacobian_gtsam(PRIOR6, [T], z, None, None)
        R.add(r, J, [(c, 6*v + c) for c in range(6)], [], sig[3], 0.0, 1 + max(abs(x) for x in T[1] + z[9:]))
    return R


def motion_objective(q, poses, pts, sig):
    """(error, rounding scale) of the motion graph at poses [X_a, X_b, H] and the distinct tracklets' points [P, 6]"""
    P, mult = _distinct_motion(q)
    e = s = mpf(0)
    for j in range(P):
        R = _motion_rows(q, poses, pts, j, sig, jac=False)
        e += mult[j]*R.err; s += mult[j]*R.err_scale
    R = _prior_rows(q, poses, sig)
    return e + R.err, s + R.err_scale


def _distinct_motion(q):
    n = len(q["kp_prev"]); P = min(q.get("period") or n, n)
    return P, [len(range(j, n, P)) for j in range(P)]


def motion_step(q, sig, lam):
    P, mult = _distinct_motion(q)
    poses = [q["pose_prev"], q["pose_cur"], q["motion_init"]]
    blocks = [_motion_rows(q, poses, q["points_init"], j, sig) for j in range(P)]
    return eliminate(blocks, mult, _prior_rows(q, poses, sig), 18, lam)


# ---- reading a device step back
def pose_step_error(X0, dxi, Xout):
    """the tangent-space difference Log(Retract(X0, dxi)^-1 Xout) between the device's candidate and the reference's,
    the reference retraction evaluated with GTSAM's formula maps (what the device implements)"""
    ref = LR.g_retract(LR.pose(X0), dxi)
    return LR.log_se3(LR.between(ref, LR.pose(Xout)))
