"""Cases of the combined IMU preintegration (dynosam_b200/csrc/preint.cuh), each naming the boundaries it reaches, the
50-digit classifier that finds the boundaries a case actually reaches, and the a-priori tolerances the host build and the
device are held to against tests/preint_reference.py.

Tolerances, stated before any measurement (n = number of steps, eps = 2^-52):
    record block (dR, dp, dv, dt, each bias Jacobian):  16 eps (n + 1) max(1, |block|_max)
    Sigma_ij:                                           32 eps (n + 1) sqrt(Sigma_ii Sigma_jj)
    R:                                                  32 eps (n + 15) kappa_s |R|_max,  kappa_s the condition number of
                                                        Sigma scaled to a unit diagonal
    status:                                             equal
"""
from types import SimpleNamespace

import numpy as np
from mpmath import mp, mpf

from dynosam_b200.binding import ImuParams

EPS = 2.0**-52
REQUIRED = ["omega_zero", "exp_below", "exp_above", "jr_below", "jr_above", "rot_0.3", "rot_near_pi",
            "dt_1e-4", "dt_1", "dt_mixed", "m2", "m3", "m2000", "bias_zero", "bias_nonzero",
            "bps_identity", "bps_viode", "bps_lever", "int_zero", "int_default", "bint_zero", "bint_default",
            "g_y98", "g_z981", "not_pd"]
R_BODY_CAMERA = np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], dtype=np.float64)    # ViodeDataProvider.cc:415-418


def gtsam_defaults(g):
    """PreintegrationCombinedParams(g) of GTSAM 4.2.0 [GTSAM-ext]: every covariance I, no sensor pose"""
    p = ImuParams()
    p.n_gravity[:] = list(map(float, g))
    I3 = list(np.eye(3).reshape(9)); I6 = list(np.eye(6).reshape(36))
    for k in ("accelerometer_cov", "gyroscope_cov", "integration_cov", "bias_acc_cov", "bias_omega_cov"):
        getattr(p, k)[:] = I3
    p.bias_acc_omega_int[:] = I6
    p.body_P_sensor[:] = list(np.eye(3).reshape(9)) + [0.0]*3
    return p


def frontend(g, acc_nd, gyro_nd, acc_rw, gyro_rw, int_sigma, T):
    """ImuFrontend's parameters (binding.imu_frontend_params, restated without the library)"""
    p = gtsam_defaults(g)
    p.accelerometer_cov[:] = list((acc_nd**2*np.eye(3)).reshape(9)); p.gyroscope_cov[:] = list((gyro_nd**2*np.eye(3)).reshape(9))
    p.integration_cov[:] = list((int_sigma**2*np.eye(3)).reshape(9))
    p.bias_acc_cov[:] = list((gyro_rw**2*np.eye(3)).reshape(9)); p.bias_omega_cov[:] = list((acc_rw**2*np.eye(3)).reshape(9))
    p.body_P_sensor[:] = list(T[:3, :3].reshape(9)) + list(T[:3, 3]); p.has_body_P_sensor = 1
    return p


def _rot(axis, th):
    a = np.asarray(axis, dtype=np.float64); a = a/np.linalg.norm(a); W = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th)*W + (1 - np.cos(th))*W@W


def _samples(rng, m, theta, dt, axis=(0.3, -0.5, 0.8)):
    """m samples: random accelerometer values (|a| ~ 10), a constant gyro of per-step angle theta at the first dt"""
    a = np.asarray(axis, dtype=np.float64); a = a/np.linalg.norm(a)
    acc = rng.normal(0, 3, (m, 3)) + np.array([0.0, 0.0, 9.81])
    gyr = np.tile(a*theta/dt, (m, 1))
    return np.concatenate([acc, gyr], 1)


def _case(name, hits, P, stamps, acc_gyr, bh=None):
    return SimpleNamespace(name=name, hits=hits, P=P, stamps=np.asarray(stamps, dtype=np.float64),
                           acc_gyr=np.ascontiguousarray(acc_gyr, dtype=np.float64), bh=None if bh is None else np.asarray(bh, dtype=np.float64))


def cases(long=True):
    rng = np.random.default_rng(7)
    gz = (0.0, 0.0, -9.81); gy = (0.0, 9.8, 0.0)
    out = []
    dt = 0.005; m = 5; st = np.arange(m)*dt
    D = gtsam_defaults(gz)
    for name, th, hit in (("rot_zero", 0.0, "omega_zero"), ("exp_below", 1e-8, "exp_below"), ("exp_above", 1.6e-8, "exp_above"),
                          ("jr_below", 0.99e-5, "jr_below"), ("jr_above", 1.01e-5, "jr_above"), ("rot_03", 0.3, "rot_0.3"),
                          ("rot_near_pi", 3.1, "rot_near_pi")):
        out.append(_case(name, [hit, "bias_zero", "g_z981", "int_default", "bint_default"], D, st, _samples(rng, m, th, dt)))
    out.append(_case("dt_small", ["dt_1e-4", "rot_0.3"], D, np.arange(4)*1e-4, _samples(rng, 4, 0.3, 1e-4)))
    out.append(_case("dt_large", ["dt_1", "rot_0.3"], D, np.arange(3)*1.0, _samples(rng, 3, 0.3, 1.0)))
    out.append(_case("dt_mixed", ["dt_mixed", "dt_1e-4", "dt_1"], D, np.cumsum([0.0, 1e-4, 1.0, 0.01, 0.3, 2e-3]),
                     _samples(rng, 6, 0.02, 0.01)))
    out.append(_case("two_samples", ["m2"], D, [0.0, 0.01], _samples(rng, 2, 0.05, 0.01)))
    out.append(_case("three_samples", ["m3"], D, [0.0, 0.01, 0.02], _samples(rng, 3, 0.05, 0.01)))
    out.append(_case("bias_hat", ["bias_nonzero"], D, st, _samples(rng, m, 0.2, dt), bh=[0.1, -0.2, 0.05, 0.01, -0.02, 0.03]))
    T = np.eye(4)
    out.append(_case("frontend_identity", ["bps_identity", "g_z981"], frontend(gz, 0.2, 0.05, 0.02, 4e-5, 1e-3, T), st,
                     _samples(rng, m, 0.1, dt)))
    T = np.eye(4); T[:3, :3] = R_BODY_CAMERA.T
    out.append(_case("frontend_viode", ["bps_viode", "g_y98"], frontend(gy, 0.2, 0.05, 0.02, 4e-5, 1e-3, T), st,
                     _samples(rng, m, 0.1, dt)))
    T = np.eye(4); T[:3, :3] = _rot((1, 2, -1), 0.7); T[:3, 3] = [0.1, -0.05, 0.2]
    out.append(_case("lever_arm", ["bps_lever"], frontend(gz, 0.2, 0.05, 0.02, 4e-5, 1e-3, T), st, _samples(rng, m, 0.3, dt),
                     bh=[0.02, 0.01, -0.03, 0.001, 0.002, -0.001]))
    Z = gtsam_defaults(gz); Z.integration_cov[:] = [0.0]*9; Z.bias_acc_omega_int[:] = [0.0]*36
    out.append(_case("zero_int", ["int_zero", "bint_zero"], Z, st, _samples(rng, m, 0.2, dt)))
    # zero bias random walks and biasAccOmegaInt: the bias rows of Sigma are identically zero at every step (F's bias rows
    # are the identity and Q's bias block is dt times zero), whatever the rounding -- a structurally singular Sigma
    Z1 = gtsam_defaults(gz); Z1.bias_acc_omega_int[:] = [0.0]*36; Z1.bias_acc_cov[:] = [0.0]*9; Z1.bias_omega_cov[:] = [0.0]*9
    out.append(_case("not_pd", ["not_pd", "m3", "bint_zero"], Z1, [0.0, 0.01, 0.02], _samples(rng, 3, 0.2, 0.01)))
    if long:
        st2 = np.cumsum(np.concatenate([[0.0], rng.uniform(0.004, 0.006, 1999)]))
        out.append(_case("long_2000", ["m2000", "dt_mixed"], frontend(gy, 0.2, 0.05, 0.02, 4e-5, 1e-3, np.eye(4)), st2,
                         _samples(rng, 2000, 0.01, 0.005)))
    return {c.name: c for c in out}


def boundaries(c, Sigma_pd=None):
    """the boundaries case c reaches, classified in 50 digits from its inputs (Sigma_pd: the reference's verdict)"""
    b = set()
    st = [mpf(float(x)) for x in c.stamps]
    dts = [st[i + 1] - st[i] for i in range(len(st) - 1)]
    bh = [mpf(0)]*6 if c.bh is None else [mpf(float(x)) for x in c.bh]
    for i, dt in enumerate(dts):
        w = [mpf(float(c.acc_gyr[i, 3 + k])) - bh[3 + k] for k in range(3)]
        t2 = sum((x*dt)**2 for x in w)
        th = mp.sqrt(t2)
        if t2 == 0:
            b.add("omega_zero")
        elif t2 <= mpf(2)**-52:
            b.add("exp_below")
        elif t2 < mpf("1e-10"):
            b.add("jr_below")
            if t2 < 2*mpf(2)**-52:                      # within a factor 2 above so3_expmap's switch
                b.add("exp_above")
        else:
            b.add("jr_above")
        if abs(th - mpf("0.3")) < mpf("0.05"):
            b.add("rot_0.3")
        if th > 3:
            b.add("rot_near_pi")
        if abs(dt - mpf("1e-4")) < mpf("1e-9"):
            b.add("dt_1e-4")
        if abs(dt - 1) < mpf("1e-9"):
            b.add("dt_1")
    if len(set(float(d) for d in dts)) > 1:
        b.add("dt_mixed")
    m = len(st)
    b.add({2: "m2", 3: "m3", 2000: "m2000"}.get(m, "m_other"))
    b.add("bias_zero" if c.bh is None or not np.any(c.bh) else "bias_nonzero")
    P = c.P
    if P.has_body_P_sensor:
        R = np.array(P.body_P_sensor[:9]).reshape(3, 3); t = np.array(P.body_P_sensor[9:])
        if np.any(t != 0):
            b.add("bps_lever")
        elif np.array_equal(R, np.eye(3)):
            b.add("bps_identity")
        elif np.array_equal(R, R_BODY_CAMERA.T):
            b.add("bps_viode")
    b.add("int_zero" if not any(P.integration_cov) else ("int_default" if list(P.integration_cov) == list(np.eye(3).reshape(9)) else "int_other"))
    b.add("bint_zero" if not any(P.bias_acc_omega_int) else ("bint_default" if list(P.bias_acc_omega_int) == list(np.eye(6).reshape(36)) else "bint_other"))
    g = tuple(P.n_gravity)
    b.add({(0.0, 9.8, 0.0): "g_y98", (0.0, 0.0, -9.81): "g_z981"}.get(g, "g_other"))
    if Sigma_pd is False:
        b.add("not_pd")
    return b
