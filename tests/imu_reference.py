"""Independent numpy statement of the visual-inertial factors (no code shared with libdynoba or the package):
scipy's Rotation for Exp / Log, plain 3x3 algebra for the rest.

GTSAM 4.2.0 CombinedImuFactor with ManifoldPreintegration and no Coriolis term:
  biasCorrectedDelta:  dR Exp(delRdelBiasOmega dbw), dp / dv + del*delBias* db           (db = b_i - biasHat)
  correctPIM:          dP += dt R_i^T v_i + dt^2/2 R_i^T g,  dV += dt R_i^T g
  predict:             NavState(X_i, v_i).retract([Log(dRc), dP, dV])
  error:               predicted.localCoordinates(NavState(X_j, v_j)), then b_i - b_j   (Between(b_j, b_i))
Pose3 retract: T Exp([omega; v]) (GTSAM_POSE3_EXPMAP); velocities and biases retract by addition.
"""
import numpy as np
from scipy.spatial.transform import Rotation

IMU_D, IMU_JC = 15, 30
SLOT_DIMS = (6, 3, 6, 3, 6, 6)      # pose_i, vel_i, pose_j, vel_j, bias_i, bias_j


def exp3(w):
    return Rotation.from_rotvec(np.asarray(w, dtype=np.float64)).as_matrix()


def log3(R):
    return Rotation.from_matrix(R).as_rotvec()


def unpack(rec):
    rec = np.asarray(rec, dtype=np.float64)
    m = lambda o: rec[o:o + 9].reshape(3, 3)
    return dict(dR=m(0), dp=rec[9:12], dv=rec[12:15], dt=rec[15], bias_hat=rec[16:22], JRw=m(22), JPa=m(31), JPw=m(40),
                JVa=m(49), JVw=m(58), g=rec[67:70])


def imu_residual(Xi, vi, Xj, vj, bi, bj, rec):
    """15-vector residual; X = [R row-major (9) | t (3)]"""
    P = unpack(rec)
    Ri, ti = np.asarray(Xi[:9]).reshape(3, 3), np.asarray(Xi[9:12])
    Rj, tj = np.asarray(Xj[:9]).reshape(3, 3), np.asarray(Xj[9:12])
    db = np.asarray(bi) - P["bias_hat"]
    dba, dbw = db[:3], db[3:]
    phi = log3(P["dR"]@exp3(P["JRw"]@dbw))
    dP = P["dp"] + P["JPa"]@dba + P["JPw"]@dbw + P["dt"]*Ri.T@vi + 0.5*P["dt"]**2*Ri.T@P["g"]
    dV = P["dv"] + P["JVa"]@dba + P["JVw"]@dbw + P["dt"]*Ri.T@P["g"]
    Rp = Ri@exp3(phi)
    pp = ti + Ri@dP
    vp = np.asarray(vi) + Ri@dV
    return np.concatenate([log3(Rp.T@Rj), Rp.T@(tj - pp), Rp.T@(np.asarray(vj) - vp), np.asarray(bi) - np.asarray(bj)])


def retract_pose(X, xi):
    R, t = X[:9].reshape(3, 3), X[9:12]
    w, v = xi[:3], xi[3:]
    th = np.linalg.norm(w)
    if th < 1e-12:
        V = np.eye(3)
    else:
        W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        V = np.eye(3) + (1 - np.cos(th))/th**2*W + (th - np.sin(th))/th**3*W@W
    return np.concatenate([(R@exp3(w)).reshape(9), t + R@(V@v)])


def imu_numeric_jacobian(args, rec, h=1e-6):
    """central differences through each variable's retract: J[15][30], columns pose_i | vel_i | pose_j | vel_j | bias_i | bias_j"""
    J = np.zeros((IMU_D, IMU_JC)); col = 0
    for s, d in enumerate(SLOT_DIMS):
        for c in range(d):
            out = []
            for sg in (1.0, -1.0):
                a = [np.array(x, dtype=np.float64) for x in args]
                e = np.zeros(d); e[c] = sg*h
                a[s] = retract_pose(a[s], e) if d == 6 and s in (0, 2) else a[s] + e
                out.append(imu_residual(*a, rec))
            J[:, col] = (out[0] - out[1])/(2*h)
            col += 1
    return J


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def _jr(x):
    """SO(3) right Jacobian"""
    th = np.linalg.norm(x); W = _skew(x)
    if th < 1e-5:
        return np.eye(3) - 0.5*W + W@W/6.0
    return np.eye(3) - (1 - np.cos(th))/th**2*W + (th - np.sin(th))/th**3*W@W


def imu_jacobian(Xi, vi, Xj, vj, bi, bj, rec):
    """closed-form J[15][30] of imu_residual, composed the way GTSAM's H1..H6 are: predict through correctPIM and
    NavState::retract, then localCoordinates; velocity columns are the NavState ones times R^T"""
    P = unpack(rec)
    Ri, Rj = np.asarray(Xi[:9]).reshape(3, 3), np.asarray(Xj[:9]).reshape(3, 3)
    db = np.asarray(bi) - P["bias_hat"]
    th = P["JRw"]@db[3:]
    dRc = P["dR"]@exp3(th)
    phi = log3(dRc)
    Ephi = exp3(phi)
    dPc = P["dp"] + P["JPa"]@db[:3] + P["JPw"]@db[3:]
    dVc = P["dv"] + P["JVa"]@db[:3] + P["JVw"]@db[3:]
    Rp = Ri@Ephi
    r = imu_residual(Xi, vi, Xj, vj, bi, bj, rec)
    eR, ep, ev = r[:3], r[3:6], r[6:9]
    E = Rp.T@Rj
    Jinv = np.linalg.inv(_jr(eR))                    # LogmapDerivative
    dRp_dbw = _jr(th)@P["JRw"]                       # right tangent of the predicted rotation w.r.t. the gyro bias
    J = np.zeros((IMU_D, IMU_JC))
    # a right-tangent perturbation d of the predicted rotation moves eR by -Jinv E^T d, ep by [ep]x d, ev by [ev]x d;
    # the pose-i rotation moves it by Ephi^T d_i, the gyro bias by Jr(th) delRdelBiasOmega d_bw
    dRp = {"wi": Ephi.T, "bw": dRp_dbw}
    J[0:3, 0:3] = -Jinv@E.T@dRp["wi"]
    J[0:3, 9:12] = Jinv
    J[0:3, 21:24] = -Jinv@E.T@dRp["bw"]
    J[3:6, 0:3] = _skew(ep)@dRp["wi"] + Ephi.T@_skew(dPc)
    J[3:6, 3:6] = -Ephi.T
    J[3:6, 6:9] = -P["dt"]*Rp.T
    J[3:6, 12:15] = E
    J[3:6, 18:21] = -Ephi.T@P["JPa"]
    J[3:6, 21:24] = _skew(ep)@dRp["bw"] - Ephi.T@P["JPw"]
    J[6:9, 0:3] = _skew(ev)@dRp["wi"] + Ephi.T@_skew(dVc)
    J[6:9, 6:9] = -Rp.T
    J[6:9, 15:18] = Rp.T
    J[6:9, 18:21] = -Ephi.T@P["JVa"]
    J[6:9, 21:24] = _skew(ev)@dRp["bw"] - Ephi.T@P["JVw"]
    J[9:15, 18:24] = np.eye(6)
    J[9:15, 24:30] = -np.eye(6)
    return J
