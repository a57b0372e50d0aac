"""A 50-digit reference of combined IMU preintegration (GTSAM 4.2.0 PreintegratedCombinedMeasurements::integrateMeasurement
with ManifoldPreintegration, no Coriolis), of noiseModel::Gaussian::Covariance and of PreintegrationBase::predict.  Plain
mpmath, written from the mathematics; it imports neither the CUDA library nor dynosam_b200/csrc/preint.cuh's host build.
SO(3) maps are the true ones of tests/lie_reference.py, Jr that of tests/imu_lie_reference.py.

One sample (measured acc, omega; dt) moves the NavState (R, p, v) of the interval:
    a = bRs (acc - bh_a) - [w]x [w]x arm,  w = bRs (omega - bh_w)          (no sensor pose: bRs = I, arm = 0)
    R' = R Exp(w dt),  p' = p + v dt + R a dt^2/2,  v' = v + R a dt
A, B, C are the derivatives of (R', p', v') in NavState's chart (R Exp(dR), p + R dp, v + R dv) w.r.t. the old state,
the measured acc and the measured omega, taken here by 50-digit central differences of that map (`step_jacobians`).
The bias Jacobians follow ManifoldPreintegration's recursion with the rotation before the step (`step`); for a record
without a sensor pose they are the derivatives of the n-step map w.r.t. biasHat (tests/test_preint.py checks that).

Covariance, the two [GTSAM-ext] statements of this module (`F_of`, `injected_noise`): Sigma' = F Sigma F^T + Q with
F = [[A, F_nb], [0, I]] (F_nb: -C's rotation rows by the gyro bias, -B's position and velocity rows by the acc bias) and
Q = G N G^T over the independent noises (acc white, gyro white, integration, acc / gyro bias walk, initial bias) with
N = blockdiag(aCov/dt, wCov/dt, dt iCov, dt baCov, dt bwCov, bInt/dt).
R = chol(Sigma^-1)^T: upper triangular, positive diagonal, R^T R = Sigma^-1 (None when Sigma is not positive definite).
"""
import numpy as np
from mpmath import mp, mpf

import imu_lie_reference as IL
import lie_reference as LR

mp.dps = 50
H = mpf("1e-20")                                # central-difference step: error O(H^2) = 1e-40


def _m(x):
    return [mpf(float(v)) for v in np.asarray(x, dtype=np.float64).reshape(-1)]


def params(P):
    """the ctypes ImuParams (or anything with the same attributes) as 50-digit lists"""
    d = {k: _m(list(getattr(P, k))) for k in ("n_gravity", "accelerometer_cov", "gyroscope_cov", "integration_cov",
                                               "bias_acc_cov", "bias_omega_cov", "bias_acc_omega_int", "body_P_sensor")}
    d["has_bps"] = bool(P.has_body_P_sensor)
    return d


def correct(P, acc, omega, bh):
    """(a, w) in the body frame from measured samples"""
    a = [x - b for x, b in zip(acc, bh[:3])]; w = [x - b for x, b in zip(omega, bh[3:])]
    if P["has_bps"]:
        bRs, arm = P["body_P_sensor"][:9], P["body_P_sensor"][9:]
        w = LR.mv3(bRs, w); a = LR.mv3(bRs, a)
        a = [x - y for x, y in zip(a, LR.cross(w, LR.cross(w, arm)))]
    return a, w


def nav(P, R, p, v, acc, omega, bh, dt):
    a, w = correct(P, acc, omega, bh)
    Ra = LR.mv3(R, a)
    return (LR.mul3(R, LR.exp_so3([x*dt for x in w])), [pi + vi*dt + ra*dt*dt/2 for pi, vi, ra in zip(p, v, Ra)],
            [vi + ra*dt for vi, ra in zip(v, Ra)])


def chart(R0, p0, v0, R1, p1, v1):
    """(dR, dp, dv) of (R1, p1, v1) in the chart at (R0, p0, v0)"""
    Rt = LR.tr3(R0)
    return LR.log_so3(LR.mul3(Rt, R1)) + LR.mv3(Rt, [a - b for a, b in zip(p1, p0)]) + LR.mv3(Rt, [a - b for a, b in zip(v1, v0)])


def step_jacobians(P, R, p, v, acc, omega, bh, dt):
    """A [9][9], B [9][3], C [9][3] of one step by central differences"""
    R1, p1, v1 = nav(P, R, p, v, acc, omega, bh, dt)
    cols = []
    for j in range(15):
        pair = []
        for s in (H, -H):
            d = [mpf(0)]*15; d[j] = s
            if j < 9:
                Rq = LR.mul3(R, LR.exp_so3(d[0:3])); pq = [x + y for x, y in zip(p, LR.mv3(R, d[3:6]))]
                vq = [x + y for x, y in zip(v, LR.mv3(R, d[6:9]))]
                out = nav(P, Rq, pq, vq, acc, omega, bh, dt)
            else:
                out = nav(P, R, p, v, [x + y for x, y in zip(acc, d[9:12])], [x + y for x, y in zip(omega, d[12:15])], bh, dt)
            pair.append(chart(R1, p1, v1, *out))
        cols.append([(x - y)/(2*H) for x, y in zip(*pair)])
    A = [[cols[j][i] for j in range(9)] for i in range(9)]
    B = [[cols[9 + j][i] for j in range(3)] for i in range(9)]
    C = [[cols[12 + j][i] for j in range(3)] for i in range(9)]
    return A, B, C


def F_of(A, B, C):
    """[GTSAM-ext CombinedImuFactor.cpp] F (15 x 15) of one step"""
    F = [[mpf(0)]*15 for _ in range(15)]
    for i in range(9):
        for j in range(9):
            F[i][j] = A[i][j]
    for i in range(3):
        for j in range(3):
            F[i][12 + j] = -C[i][j]; F[3 + i][9 + j] = -B[3 + i][j]; F[6 + i][9 + j] = -B[6 + i][j]
    for i in range(9, 15):
        F[i][i] = mpf(1)
    return F


def injected_noise(P, B, C, dt):
    """[GTSAM-ext CombinedImuFactor.cpp G_measCov_Gt] Q = G N G^T (15 x 15); noise order: acc white, gyro white,
    integration, acc bias walk, gyro bias walk, initial bias (acc, gyro)"""
    G = [[mpf(0)]*21 for _ in range(15)]
    for i in range(3):
        for j in range(3):
            G[i][3 + j] = -C[i][j]; G[i][18 + j] = C[i][j]                    # theta: gyro white, initial gyro bias
            G[3 + i][j] = -B[3 + i][j]; G[3 + i][15 + j] = B[3 + i][j]        # p: acc white, initial acc bias
            G[6 + i][j] = -B[6 + i][j]; G[6 + i][15 + j] = B[6 + i][j]        # v
        G[3 + i][6 + i] = mpf(1); G[9 + i][9 + i] = mpf(1); G[12 + i][12 + i] = mpf(1)
    N = [[mpf(0)]*21 for _ in range(21)]
    blocks = [(0, P["accelerometer_cov"], 1/dt), (3, P["gyroscope_cov"], 1/dt), (6, P["integration_cov"], dt),
              (9, P["bias_acc_cov"], dt), (12, P["bias_omega_cov"], dt)]
    for o, M, s in blocks:
        for i in range(3):
            for j in range(3):
                N[o + i][o + j] = M[3*i + j]*s
    for i in range(6):
        for j in range(6):
            N[15 + i][15 + j] = P["bias_acc_omega_int"][6*i + j]/dt
    Gm, Nm = mp.matrix(G), mp.matrix(N)
    return Gm*Nm*Gm.T


def step(P, st, acc, omega, dt):
    """one integrateMeasurement: the new state dict (R, p, v, T, bias Jacobians, Sigma) and (A, B, C)"""
    bh = st["bh"]
    R, p, v = st["R"], st["p"], st["v"]
    A, B, C = step_jacobians(P, R, p, v, acc, omega, bh, dt)
    a, w = correct(P, acc, omega, bh)
    th = [x*dt for x in w]
    inc = LR.exp_so3(th); Jr = IL.jr(th)
    D = [-x for x in LR.mul3(LR.mul3(R, LR.skew(a)), st["JRw"])]
    n = dict(st)
    n["JRw"] = [x - y*dt for x, y in zip(LR.mul3(LR.tr3(inc), st["JRw"]), Jr)]
    n["JPa"] = [x + y*dt - dt*dt/2*r for x, y, r in zip(st["JPa"], st["JVa"], R)]
    n["JPw"] = [x + dt*y + dt*dt/2*d for x, y, d in zip(st["JPw"], st["JVw"], D)]
    n["JVa"] = [x - r*dt for x, r in zip(st["JVa"], R)]
    n["JVw"] = [x + d*dt for x, d in zip(st["JVw"], D)]
    n["R"], n["p"], n["v"] = nav(P, R, p, v, acc, omega, bh, dt)
    n["T"] = st["T"] + dt
    F = mp.matrix(F_of(A, B, C))
    n["S"] = F*st["S"]*F.T + injected_noise(P, B, C, dt)
    return n, (A, B, C)


def start(bh):
    z = [mpf(0)]*9
    return dict(bh=list(bh), R=list(LR.I3), p=[mpf(0)]*3, v=[mpf(0)]*3, T=mpf(0), JRw=z, JPa=z, JPw=z, JVa=z, JVw=z,
                S=mp.matrix(15, 15))


def record(st, g):
    return (st["R"] + st["p"] + st["v"] + [st["T"]] + st["bh"] + st["JRw"] + st["JPa"] + st["JPw"] + st["JVa"] + st["JVw"]
            + list(g))


def sqrt_info(S):
    """R = chol(Sigma^-1)^T, or None when Sigma is not positive definite"""
    try:
        L = mp.cholesky(S)
    except ValueError:
        return None
    if min(L[i, i] for i in range(15)) <= 0:
        return None
    Li = mp.inverse(L)
    return mp.cholesky(Li.T*Li).T


def preintegrate(P, stamps, acc_gyr, bh=None):
    """(record [70], Sigma [15 x 15], R or None) of one interval; stamps, acc_gyr as float64 arrays"""
    st = start(_m(np.zeros(6) if bh is None else bh))
    ts = _m(stamps); ag = np.asarray(acc_gyr, dtype=np.float64).reshape(-1, 6)
    for i in range(len(ts) - 1):
        st, _ = step(P, st, _m(ag[i, :3]), _m(ag[i, 3:]), ts[i + 1] - ts[i])
    return record(st, P["n_gravity"]), st["S"], sqrt_info(st["S"])


def predict(z, Xi, vi, bi):
    """PreintegrationBase::predict with true maps: (Xj [12], vj [3])"""
    u = IL.unpack(z)
    dba = [x - y for x, y in zip(bi[:3], u["bh"][:3])]; dbw = [x - y for x, y in zip(bi[3:], u["bh"][3:])]
    phi = LR.log_so3(LR.mul3(u["dR"], LR.exp_so3(LR.mv3(u["JRw"], dbw))))
    dt = u["dt"]; Ri = Xi[:9]; ti = Xi[9:]
    Rtv = LR.mv3(LR.tr3(Ri), vi); Rtg = LR.mv3(LR.tr3(Ri), u["g"])
    xP = [a + b + c + dt*d + dt*dt/2*e for a, b, c, d, e in zip(u["dp"], LR.mv3(u["JPa"], dba), LR.mv3(u["JPw"], dbw), Rtv, Rtg)]
    xV = [a + b + c + dt*e for a, b, c, e in zip(u["dv"], LR.mv3(u["JVa"], dba), LR.mv3(u["JVw"], dbw), Rtg)]
    Rj = LR.mul3(Ri, LR.exp_so3(phi))
    return Rj + [a + b for a, b in zip(ti, LR.mv3(Ri, xP))], [a + b for a, b in zip(vi, LR.mv3(Ri, xV))]
