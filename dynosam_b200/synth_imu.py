"""Synthetic IMU data and preintegration for the visual-inertial graphs (host code for tests and benchmarks).

* ``imu_samples``: accelerometer / gyroscope samples in closed form along ``synth.make_problem``'s camera trajectory.
  That trajectory is a constant twist per frame, so the body-frame angular rate w_b and velocity v_b are constant and the
  specific force is f_b = w_b x v_b - R(t)^T g.  A seeded constant bias and white noise are added.
* ``preintegrate``: a numpy restatement of GTSAM 4.2.0's ``ManifoldPreintegration::update`` (no body_P_sensor, no
  Coriolis): deltaRij, deltaPij, deltaVij, deltaTij and the five bias Jacobians, packed as the 70-double record of
  ``DYNOBA_COMBINED_IMU15`` (include/dynoba.h).
* ``sqrt_info``: an SPD covariance and its square-root information R (R^T R = Sigma^-1).  The factor takes R as given,
  so this covariance is NOT GTSAM's preintegrated-covariance propagation: it is a seeded SPD matrix of the right scale
  whose off-diagonal terms couple the navigation rows with the bias rows.
* ``add_imu_chain``: velocities, biases, their priors and one COMBINED_IMU15 per frame pair, as
  VisionImuBackendModule::addInitialVisualInertialState / addVisualInertialStates build them.
"""
from __future__ import annotations

import numpy as np

from .problem import COMBINED_IMU15, PRIOR_BIAS6, PRIOR_VEL3, FactorBlock

GRAVITY = np.array([0.0, 0.0, -9.81])
FRAME_DT = 0.1                          # seconds between frames of synth.make_problem's trajectory
VEL_PRIOR_SIGMA = 1e-5                  # addInitialVisualInertialState: Isotropic velocity prior
BIAS_PRIOR_SIGMA = np.array([0.1]*3 + [0.01]*3)   # Diagonal bias prior: accelerometer, gyroscope


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def so3_exp(w):
    th = np.linalg.norm(w); W = skew(w)
    if th < 1e-12:
        return np.eye(3) + W
    return np.eye(3) + np.sin(th)/th*W + (1 - np.cos(th))/th**2*W@W


def so3_jr(w):
    th = np.linalg.norm(w); W = skew(w)
    if th < 1e-5:
        return np.eye(3) - 0.5*W + W@W/6.0
    return np.eye(3) - (1 - np.cos(th))/th**2*W + (th - np.sin(th))/th**3*W@W


def body_rates(xi_frame, frame_dt=FRAME_DT):
    """(w_b, v_b) of the constant twist xi_frame per frame ([omega; v], synth.make_problem's xi_cam)"""
    xi = np.asarray(xi_frame, dtype=np.float64)/frame_dt
    return xi[:3], xi[3:]


def imu_samples(R0, xi_frame, n_samples, dt, bias=None, acc_noise=0.0, gyro_noise=0.0, rng=None, g=GRAVITY):
    """accelerometer and gyroscope samples [n, 3] at t = k dt from the pose R0 of the interval's first frame"""
    w, v = body_rates(xi_frame)
    bias = np.zeros(6) if bias is None else np.asarray(bias)
    acc = np.empty((n_samples, 3)); gyro = np.empty((n_samples, 3))
    for k in range(n_samples):
        R = R0@so3_exp(w*k*dt)
        acc[k] = np.cross(w, v) - R.T@g + bias[:3]
        gyro[k] = w + bias[3:]
    if rng is not None:
        acc += rng.normal(0, acc_noise, acc.shape); gyro += rng.normal(0, gyro_noise, gyro.shape)
    return acc, gyro


def preintegrate(acc, gyro, dt, bias_hat=np.zeros(6), g=GRAVITY):
    """ManifoldPreintegration::update over the samples -> 70-double COMBINED_IMU15 record"""
    dR = np.eye(3); dp = np.zeros(3); dv = np.zeros(3); T = 0.0
    JRw = np.zeros((3, 3)); JPa = np.zeros((3, 3)); JPw = np.zeros((3, 3)); JVa = np.zeros((3, 3)); JVw = np.zeros((3, 3))
    for a_m, w_m in zip(acc, gyro):
        a = a_m - bias_hat[:3]; w = w_m - bias_hat[3:]
        dt22 = 0.5*dt*dt
        # Jacobians first, with the rotation before this step (ManifoldPreintegration::update)
        D_acc_bw = -dR@skew(a)@JRw
        incR = so3_exp(w*dt)
        JRw = incR.T@JRw - so3_jr(w*dt)*dt
        JPa = JPa + JVa*dt - dt22*dR
        JPw = JPw + dt*JVw + dt22*D_acc_bw
        JVa = JVa - dR*dt
        JVw = JVw + D_acc_bw*dt
        # NavState::update: integrate in the body frame, retract
        dp = dp + dv*dt + dt22*(dR@a)
        dv = dv + dR@a*dt
        dR = dR@incR
        T += dt
    return np.concatenate([dR.reshape(9), dp, dv, [T], bias_hat, JRw.reshape(9), JPa.reshape(9), JPw.reshape(9),
                           JVa.reshape(9), JVw.reshape(9), g])


def sqrt_info(rng, scale_nav=1e-3, scale_bias=1e-3, coupling=0.3):
    """(Sigma, R): seeded SPD 15x15 covariance and its upper-triangular square-root information R (R^T R = Sigma^-1)"""
    d = np.concatenate([np.full(9, scale_nav), np.full(6, scale_bias)])
    A = rng.normal(0, 1, (15, 15))
    C = np.eye(15) + coupling*(A + A.T)/np.sqrt(15)*0.5
    w, V = np.linalg.eigh(C)
    C = V@np.diag(np.maximum(w, 0.2))@V.T
    Sigma = np.diag(d)@C@np.diag(d)
    L = np.linalg.cholesky(np.linalg.inv(Sigma))       # Sigma^-1 = L L^T  ->  R = L^T
    return Sigma, np.ascontiguousarray(L.T)


def add_imu_chain(X_gt, xi_frame, seed, samples_per_frame=10, bias_true=None, noise=True, init_noise=True):
    """(vel_init [N,3], bias_init [N,6], blocks, meta) of the IMU chain over the N frames X_gt: V_k, b_k for every frame,
    the two priors on frame 0 and COMBINED_IMU15(X_k-1, V_k-1, X_k, V_k, b_k-1, b_k) for k >= 1"""
    rng = np.random.default_rng(seed)
    N = X_gt.shape[0]
    w, v = body_rates(xi_frame)
    R = X_gt[:, :9].reshape(N, 3, 3)
    vel_gt = np.einsum("nij,j->ni", R, v)
    bias_gt = np.concatenate([rng.normal(0, 0.05, 3), rng.normal(0, 0.005, 3)]) if bias_true is None else np.asarray(bias_true)
    dt = FRAME_DT/samples_per_frame
    recs, Rs = [], []
    for k in range(N - 1):
        acc, gyro = imu_samples(R[k], xi_frame, samples_per_frame, dt, bias_gt, 1e-3 if noise else 0.0,
                                1e-4 if noise else 0.0, rng)
        recs.append(preintegrate(acc, gyro, dt, np.zeros(6)))
        Rs.append(sqrt_info(rng)[1].reshape(225))
    vel_init = vel_gt + (rng.normal(0, 0.05, vel_gt.shape) if init_noise else 0.0)
    bias_init = np.zeros((N, 6))
    vel_init[0] = vel_gt[0]
    blocks = [FactorBlock(PRIOR_VEL3, np.array([[0]]), vel_gt[:1], np.array([VEL_PRIOR_SIGMA])),
              FactorBlock(PRIOR_BIAS6, np.array([[0]]), np.zeros((1, 6)), BIAS_PRIOR_SIGMA)]
    if N > 1:
        k = np.arange(1, N)
        blocks.append(FactorBlock(COMBINED_IMU15, np.stack([k - 1, k - 1, k, k, k - 1, k], 1), np.array(recs), np.array(Rs)))
    return vel_init, bias_init, blocks, dict(vel_gt=vel_gt, bias_gt=np.tile(bias_gt, (N, 1)))
