"""A 50-digit reference of the visual-inertial factor COMBINED_IMU15 (GTSAM 4.2.0 CombinedImuFactor, ManifoldPreintegration,
no Coriolis term), of the SO(3) right Jacobian Jr and its inverse, and of the vector priors PRIOR_VEL3 / PRIOR_BIAS6.
Plain mpmath on Python lists, written from the mathematics; it imports neither the CUDA library, nor the CPU oracle, nor
the numpy statement tests/imu_reference.py.  The SO(3) maps come from tests/lie_reference.py (true maps and GTSAM's
formula maps, branch by branch).

Residual (the record z is the 70 doubles of include/dynoba.h: dR, dp, dv, dt, biasHat, the five bias Jacobians, g):

    dba = b_i.acc - biasHat.acc,  dbw = b_i.gyro - biasHat.gyro,  theta = delRdelBiasOmega dbw
    phi = Log(dR Exp(theta)),  dPc = dp + JPa dba + JPw dbw,  dVc = dv + JVa dba + JVw dbw       (bias correction)
    xP = dPc + dt R_i^T v_i + dt^2/2 R_i^T g,  xV = dVc + dt R_i^T g                            (correctPIM)
    R_p = R_i Exp(phi),  p_p = p_i + R_i xP,  v_p = v_i + R_i xV                                 (NavState retract)
    r = [Log(R_p^T R_j), R_p^T (p_j - p_p), R_p^T (v_j - v_p), b_i - b_j]                        (local coordinates)

in two forms: `residual(..., maps="true")` with the true Exp / Log, `maps="gtsam"` with GTSAM's formula maps
(`g_exp_so3` / `g_log_so3`, their branch constants).  The device's residual equals the formula form to rounding.

Jacobian: `jacobian_exact` differentiates the true-map residual by central differences in 50 digits (step 1e-20)
through the true retractions -- Pose3 T Exp(xi), addition for velocities and biases.  It shares nothing with the closed
form the kernel evaluates; the device's J is held to it within the a-priori bound of tests/imu_cases.py.

Jr and Jr^-1 in closed form, each as the true map (`jr`, `jr_inv`, a series below theta = 1e-10 in 50 digits) and as
GTSAM's formula (`g_jr`: DexpFunctor, first order I - W/2 at theta^2 <= DBL_EPSILON; `g_jr_inv`: LogmapDerivative, I at
theta^2 <= DBL_EPSILON).  Error of the formulas in exact arithmetic against the true maps (tests/test_imu_cases.py
asserts each row):

    map       branch                     condition                   |formula - true| (max entry)
    Jr        first order I - W/2        theta^2 <= DBL_EPSILON      theta^2/6 <= 3.7e-17
    Jr        closed form                otherwise                   0
    Jr^-1     I                          theta^2 <= DBL_EPSILON      theta/2 <= 7.5e-9
    Jr^-1     closed form                otherwise                   0

The device's so3_jr / so3_jr_inv switch to a second-order series at theta^2 < 1e-10 and so follow the true maps.

Whitening: noiseModel::Gaussian with the square-root information R used as given (dense, not necessarily triangular):
r_w = R r, A = R J, b = -r_w; the factor's error is 0.5 |R r|^2 and chi^2 the sum over factors.
"""
from mpmath import mp, mpf

import lie_reference as LR

mp.dps = 50

I3 = LR.I3


def unpack(z):
    """the record as 50-digit lists (z: 70 fp64 values)"""
    z = LR.vec(z)
    return dict(dR=z[0:9], dp=z[9:12], dv=z[12:15], dt=z[15], bh=z[16:22], JRw=z[22:31], JPa=z[31:40], JPw=z[40:49],
                JVa=z[49:58], JVw=z[58:67], g=z[67:70])


def _add(a, b):
    return [x + y for x, y in zip(a, b)]


def _sub(a, b):
    return [x - y for x, y in zip(a, b)]


def _scale(s, a):
    return [s*x for x in a]


def parts(Xi, vi, Xj, vj, bi, bj, z, maps="true", trace=None, phi_force=None):
    """the intermediate quantities of the residual: dict(theta, Rc, phi, Rp, E, dPc, dVc, r).  X = (R, t) 50-digit lists,
    the rest 50-digit lists.  `trace`, a dict, receives the branch names the formula Logmaps took, keyed 'phi' / 'res'.
    `phi_force` ('pi' / 'acos' / 'taylor', formula maps only) overrides the branch of phi's Logmap."""
    P = unpack(z) if not isinstance(z, dict) else z
    exp, log = (LR.exp_so3, LR.log_so3) if maps == "true" else (LR.g_exp_so3, LR.g_log_so3)
    dba = _sub(bi[:3], P["bh"][:3]); dbw = _sub(bi[3:], P["bh"][3:])
    th = LR.mv3(P["JRw"], dbw)
    Rc = LR.mul3(P["dR"], exp(th))
    if trace is not None: LR.trace_start()
    phi = log(Rc, force=phi_force) if phi_force else log(Rc)
    if trace is not None: trace["phi"] = LR.trace_stop()
    Ri, ti = Xi; Rj, tj = Xj
    Rp = LR.mul3(Ri, exp(phi))
    dPc = _add(_add(P["dp"], LR.mv3(P["JPa"], dba)), LR.mv3(P["JPw"], dbw))
    dVc = _add(_add(P["dv"], LR.mv3(P["JVa"], dba)), LR.mv3(P["JVw"], dbw))
    Rit = LR.tr3(Ri); dt = P["dt"]
    Rtg = LR.mv3(Rit, P["g"])
    xP = _add(_add(dPc, _scale(dt, LR.mv3(Rit, vi))), _scale(dt*dt/2, Rtg))
    xV = _add(dVc, _scale(dt, Rtg))
    pp = _add(ti, LR.mv3(Ri, xP)); vp = _add(vi, LR.mv3(Ri, xV))
    E = LR.mul3(LR.tr3(Rp), Rj)
    if trace is not None: LR.trace_start()
    rR = log(E)
    if trace is not None: trace["res"] = LR.trace_stop()
    Rpt = LR.tr3(Rp)
    r = rR + LR.mv3(Rpt, _sub(tj, pp)) + LR.mv3(Rpt, _sub(vj, vp)) + _sub(bi, bj)
    return dict(theta=th, Rc=Rc, phi=phi, Rp=Rp, E=E, dPc=dPc, dVc=dVc, pp=pp, vp=vp, r=r)


def residual(Xi, vi, Xj, vj, bi, bj, z, maps="true"):
    return parts(Xi, vi, Xj, vj, bi, bj, z, maps)["r"]


SLOT_DIMS = (6, 3, 6, 3, 6, 6)      # pose_i, vel_i, pose_j, vel_j, bias_i, bias_j


def jacobian_exact(Xi, vi, Xj, vj, bi, bj, z, d=mpf("1e-20")):
    """J[15][30] of the true-map residual by central differences through the true retractions"""
    P = unpack(z)
    args = [Xi, vi, Xj, vj, bi, bj]
    cols = []
    for s, n in enumerate(SLOT_DIMS):
        for c in range(n):
            hs = []
            for sg in (d, -d):
                a = list(args)
                if s in (0, 2):
                    xi = [mpf(0)]*6; xi[c] = sg
                    a[s] = LR.retract(args[s], xi)
                else:
                    x = list(args[s]); x[c] = x[c] + sg; a[s] = x
                hs.append(residual(*a, P))
            cols.append([(u - w)/(2*d) for u, w in zip(*hs)])
    return [[col[i] for col in cols] for i in range(15)]


# ---- Jr, Jr^-1
def jr(x):
    th = LR.norm(x); _, B, C = LR._abc(th); W = LR.skew(x)
    return LR.lin3(mpf(1), I3, -B, W, C, LR.mul3(W, W))


def _jr_inv_c(th):
    if th < mpf("1e-10"):
        return mpf(1)/12 + th*th/720
    return 1/(th*th) - (1 + mp.cos(th))/(2*th*mp.sin(th))


def jr_inv(x):
    th = LR.norm(x); W = LR.skew(x)
    return LR.lin3(mpf(1), I3, mpf(1)/2, W, _jr_inv_c(th), LR.mul3(W, W))


def g_jr(x):
    """GTSAM 4.2.0 so3::DexpFunctor::dexp()"""
    W = LR.skew(x)
    if LR.dot(x, x) <= LR.EXP_NEAR_ZERO:
        return LR.lin3(mpf(1), I3, -mpf(1)/2, W, mpf(0), W)
    return jr(x)


def g_jr_inv(x):
    """GTSAM 4.2.0 SO3::LogmapDerivative"""
    if LR.dot(x, x) <= LR.EXP_NEAR_ZERO:
        return list(I3)
    return jr_inv(x)


def jr_inv_bound(th):
    """a-priori bound, in units of eps, of the absolute error of a faithful fp64 Jr^-1 (entries of size 1 + theta^2):
    (1 + cos)/(2 theta sin) forms 1 + cos to an absolute eps, which is relative eps/(pi - theta)^2, and divides by
    sin ~ pi - theta: the coefficient carries eps/(2 pi (pi - theta)), the W^2 term pi^2 times that"""
    th = mpf(th)
    return 8 + (mp.pi/(2*(mp.pi - th)) if th > 1 else 0)


# ---- whitening
def whiten(r, R):
    """(r_w, error): R (15 x 15, rows of 50-digit numbers) times r, and 0.5 |r_w|^2"""
    rw = [LR.dot(row, r) for row in R]
    return rw, LR.dot(rw, rw)/2


def linearized(Xi, vi, Xj, vj, bi, bj, z, R, with_jacobian=True):
    """(A, b, error) of one factor: A = R J_exact, b = -R r (formula maps), error 0.5 |R r|^2"""
    r = residual(Xi, vi, Xj, vj, bi, bj, z, maps="gtsam")
    rw, e = whiten(r, R)
    b = [-x for x in rw]
    if not with_jacobian:
        return None, b, e
    J = jacobian_exact(Xi, vi, Xj, vj, bi, bj, z)
    A = [[LR.dot(row, [J[k][j] for k in range(15)]) for j in range(30)] for row in R]
    return A, b, e
