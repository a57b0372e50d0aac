"""Seeded synthetic inputs of the per-object refinements of the front end (SURVEY.md 8f-2): joint optical-flow + pose problems
(what OpticalFlowAndPoseOptimizer::optimize reads from two frames, MotionSolver-inl.hpp:117-160) and object-motion problems
(MotionOnlyRefinementOptimizer::optimize, :343-366).  Shared by tests/test_star.py, tests/golden/make_golden.py and
tools/star_bench.py, so that fixtures only store outputs."""
import numpy as np

from . import lie

K5 = np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854])
FLOW_SIGMA, PRIOR_SIGMA, HUBER_K = 10.0, 3.33, 0.001          # FrontendParams-like magnitudes (flow in pixels)


def _project(X, p):
    q = lie.transform_to(np.tile(X, (len(p), 1)), p)
    return np.stack([K5[0]*q[:, 0]/q[:, 2] + K5[3], K5[1]*q[:, 1]/q[:, 2] + K5[4]], 1), q[:, 2]


def _back_project(X, kp, depth):
    pc = np.stack([(kp[:, 0] - K5[3])/K5[0]*depth, (kp[:, 1] - K5[4])/K5[1]*depth, depth], 1)
    return lie.transform_from(np.tile(X, (len(kp), 1)), pc)


def make_motion_problem(rng, n, px_noise=0.3, depth_noise=0.05, outliers=0.0):
    """two camera poses, a moving rigid object: key-points in both frames, back-projected (noisy depth) world points, a
    perturbed initial motion"""
    Xa = lie.se3_exp(rng.normal(0, 0.05, (1, 6)))[0]
    Xb = lie.compose(Xa[None], lie.se3_exp(np.array([[0.002, -0.01, 0.001, 0.02, -0.01, 0.6]])))[0]
    H = lie.se3_exp(np.array([[0.01, 0.03, -0.01, 0.3, 0.02, 0.5]]) + rng.normal(0, 0.01, (1, 6)))[0]
    kp0 = np.stack([rng.uniform(400, 800, n), rng.uniform(100, 300, n)], 1); d0 = rng.uniform(8, 20, n)
    ma = _back_project(Xa, kp0, d0)
    mb = lie.transform_from(np.tile(H, (n, 1)), ma)
    if outliers > 0:
        bad = rng.random(n) < outliers; mb[bad] += rng.normal(0, 0.5, (int(bad.sum()), 3))
    kpa, da = _project(Xa, ma); kpb, db = _project(Xb, mb)
    kpa = kpa + rng.normal(0, px_noise, (n, 2)); kpb = kpb + rng.normal(0, px_noise, (n, 2))
    ma0 = _back_project(Xa, kpa, da*(1 + rng.normal(0, depth_noise, n))); mb0 = _back_project(Xb, kpb, db*(1 + rng.normal(0, depth_noise, n)))
    H0 = lie.compose(H[None], lie.se3_exp(rng.normal(0, 0.02, (1, 6))))[0]
    return dict(pose_prev=Xa, pose_cur=Xb, motion_init=H0, calib=K5, kp_prev=kpa, kp_cur=kpb, points_init=np.concatenate([ma0, mb0], 1), gt=H)


def make_flow_pose_problem(rng, n, noise=0.5, outliers=0.0, behind=0):
    """a camera step between two frames: key-points and depths in the previous frame, noisy measured flows (gross outliers /
    points that end up behind the camera on request), a perturbed initial pose"""
    X_prev = lie.se3_exp(rng.normal(0, 0.05, (1, 6)))[0]
    step = lie.se3_exp(np.array([[0.01, -0.02, 0.005, 0.05, -0.02, 0.9]]) + rng.normal(0, 0.01, (1, 6)))[0]
    X_gt = lie.compose(X_prev[None], step[None])[0]
    kp = np.stack([rng.uniform(50, 1190, n), rng.uniform(30, 340, n)], 1); depth = rng.uniform(5, 40, n)
    pc = np.stack([(kp[:, 0] - K5[3])/K5[0]*depth, (kp[:, 1] - K5[4])/K5[1]*depth, depth], 1)
    pw = lie.transform_from(np.tile(X_prev, (n, 1)), pc) if n else np.zeros((0, 3))
    q = lie.transform_to(np.tile(X_gt, (n, 1)), pw) if n else np.zeros((0, 3))
    proj = np.stack([K5[0]*q[:, 0]/q[:, 2] + K5[3], K5[1]*q[:, 1]/q[:, 2] + K5[4]], 1)
    flow = proj - kp + rng.normal(0, noise, (n, 2))
    if outliers > 0 and n:
        bad = rng.random(n) < outliers
        flow[bad] += rng.normal(0, 40.0, (int(bad.sum()), 2))
    if behind and n:
        depth[:behind] = 0.2                                     # points that end up behind the camera: cheirality branch
    init = lie.compose(X_gt[None], lie.se3_exp(rng.normal(0, 0.02, (1, 6))))[0]
    return dict(pose_init=init, pose_prev=X_prev, calib=K5, kp_prev=kp, depth=depth, flow=flow, gt=X_gt)


def flow_parity_set():
    """problems of 1 .. 700 features: exact fits, CTA-size boundaries, outliers, cheirality"""
    rng = np.random.default_rng(11)
    sizes = [1, 2, 3, 7, 33, 64, 100, 255, 256, 257, 300, 511, 700] + list(rng.integers(20, 400, 12))
    return [make_flow_pose_problem(rng, int(n), noise=0.5, outliers=0.1 if i % 3 == 0 else 0.0, behind=2 if i % 5 == 4 and n > 10 else 0) for i, n in enumerate(sizes)]


def flow_rounds_set():
    """problems whose gross outliers trigger the outlier rounds"""
    rng = np.random.default_rng(21)
    sizes = [40, 80, 150, 200, 260, 300] + list(rng.integers(30, 250, 10))
    return [make_flow_pose_problem(rng, int(n), noise=0.3, outliers=(0.0, 0.1, 0.2)[i % 3], behind=2 if i % 4 == 3 else 0) for i, n in enumerate(sizes)]


def motion_set():
    rng = np.random.default_rng(31)
    sizes = [6, 7, 20, 64, 100, 255, 256, 257] + list(rng.integers(10, 120, 6))
    return [make_motion_problem(rng, int(n), outliers=0.1 if i % 2 else 0.0) for i, n in enumerate(sizes)]


IMAGE_W, IMAGE_H = 1242, 375                                    # the image K5 belongs to


def make_pnp_problem(rng, n, noise_px=0.5, outliers=0.0, collinear=0, duplicate=0, calib=K5):
    """a 3D-2D absolute-pose problem (what geometricOutlierRejection3d2d reads, MotionSolver.cc:234-265): world points in front of
    a camera at the ground-truth pose, their key-points with Gaussian noise; round(outliers n) of them get a key-point drawn
    uniformly over the image instead (gross outliers), the first `collinear` points lie on one world line, and the last
    `duplicate` points repeat earlier ones exactly.  Returns calib, points [n,3], kp [n,2], gt (camera pose in the world, 12) and
    outlier [n] (bool)."""
    K = np.asarray(calib, dtype=np.float64)
    X = lie.se3_exp(np.concatenate([rng.normal(0, 0.2, 3), rng.normal(0, 2.0, 3)])[None])[0]
    u = rng.uniform(0, IMAGE_W, n); v = rng.uniform(0, IMAGE_H, n); z = rng.uniform(3.0, 40.0, n)
    y = (v - K[4])/K[1]
    pc = np.stack([((u - K[3]) - K[2]*y)/K[0]*z, y*z, z], 1)
    pw = lie.transform_from(np.tile(X, (n, 1)), pc) if n else np.zeros((0, 3))
    c = min(collinear, n)
    if c:          # exactly collinear in the world: equal y and z, so every cross product of differences is exactly zero
        pw[:c, 1] = pw[0, 1]; pw[:c, 2] = pw[0, 2]; pw[:c, 0] = pw[0, 0] + np.linspace(-1.0, 1.0, c)
    if duplicate and n > duplicate:
        pw[n - duplicate:] = pw[:duplicate]
    q = lie.transform_to(np.tile(X, (n, 1)), pw) if n else np.zeros((0, 3))
    kp = np.stack([K[0]*q[:, 0]/q[:, 2] + K[2]*q[:, 1]/q[:, 2] + K[3], K[1]*q[:, 1]/q[:, 2] + K[4]], 1) if n else np.zeros((0, 2))
    kp = kp + rng.normal(0, noise_px, (n, 2)) if noise_px > 0 else kp
    bad = np.zeros(n, bool)
    nb = int(round(outliers*n))
    if nb:
        bad[rng.permutation(n)[:nb]] = True
        kp[bad] = np.stack([rng.uniform(0, IMAGE_W, nb), rng.uniform(0, IMAGE_H, nb)], 1)
    if duplicate and n > duplicate:
        kp[n - duplicate:] = kp[:duplicate]; bad[n - duplicate:] = bad[:duplicate]
    return dict(calib=K.copy(), points=pw, kp=kp, gt=X, outlier=bad)


def pnp_parity_set():
    """problems of 0 .. 20 000 correspondences: below the five-match minimum, warp and tile boundaries, the camera's sizes,
    0 - 70 % gross outliers, collinear and duplicated subsets, an all-collinear problem"""
    rng = np.random.default_rng(41)
    sizes = [0, 4, 5, 6, 7, 31, 32, 33, 255, 256, 257, 800, 2700, 20000]
    fracs = [0.0, 0.1, 0.3, 0.5, 0.7]
    probs = [make_pnp_problem(rng, n, noise_px=0.5 if i % 4 else 0.0, outliers=fracs[i % 5] if n >= 5 else 0.0,
                              collinear=8 if i % 3 == 1 and n > 40 else 0, duplicate=5 if i % 3 == 2 and n > 40 else 0)
             for i, n in enumerate(sizes)]
    probs.append(make_pnp_problem(rng, 60, noise_px=0.0, collinear=60))                       # every triple collinear
    probs.append(make_pnp_problem(rng, 300, noise_px=0.5, outliers=0.7))
    probs.append(make_pnp_problem(rng, 1500, noise_px=0.5, outliers=0.1))
    return probs
