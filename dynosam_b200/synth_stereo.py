"""Seeded static stereo observations for the STEREO_PROJECTION static formulation (dynoba_builder_add_static_stereo) and
batched triangulation problems (dynoba_triangulate_batch).

Static tracklets follow synth.py's track rule (birth frame uniform in [0, N - 2], age uniform in [2, max_static_age],
clipped at the last frame).  Each landmark is placed in front of the camera at its birth frame, far enough that the
forward-moving camera of synth.py keeps it in front for its whole track, and observed as (uL, uR, v) = the fake stereo
projection of its true position (StereoCamera::project with Cal3_S2Stereo) plus Gaussian pixel noise.  Optional
fractions of the landmarks are far (disparity about 0.2 to 1 px, around the formulation's 0.5 px test), of the
measurements lose their right key-point (uR = NaN), and of the measurements are replaced by uniform outliers."""
from __future__ import annotations

import numpy as np

from . import lie
from .synth import IMG_H, IMG_W, KITTI_K, _expand, _tracks


def stereo_project(K, q):
    """(uL, uR, v) of camera-frame points q [n, 3] under calib6 K (fx fy s u0 v0 b; the skew is ignored, as GTSAM does)"""
    fx, fy, u0, v0, b = K[0], K[1], K[3], K[4], K[5]
    return np.stack([u0 + fx*q[:, 0]/q[:, 2], u0 + fx*(q[:, 0] - b)/q[:, 2], v0 + fy*q[:, 1]/q[:, 2]], 1)


def make_static_stereo(X_gt, n_static, seed=0, max_static_age=15, pixel_sigma=0.5, far_fraction=0.0, nan_right=0.0,
                       outlier_fraction=0.0, K=KITTI_K):
    """per-observation arrays in frame-major order: frame, tracklet, stereo [n, 3], and the true world points [n_static, 3]"""
    rng = np.random.default_rng(seed)
    N = X_gt.shape[0]
    birth, life = _tracks(rng, n_static, 0, N - 2, 2, max_static_age, N)
    d = rng.uniform(2.0, 50.0, n_static) + life                   # the camera advances about 1 m per frame
    far = rng.uniform(0, 1, n_static) < far_fraction
    d[far] = K[0]*K[5]/rng.uniform(0.2, 1.0, far.sum())           # disparity fx b / d in [0.2, 1] px
    u = rng.uniform(0, IMG_W, n_static); v = rng.uniform(0, IMG_H, n_static)
    pc = np.stack([(u - K[3])/K[0]*d, (v - K[4])/K[1]*d, d], 1)
    pw = lie.transform_from(X_gt[birth], pc)
    tid, off, _ = _expand(life)
    fr = birth[tid] + off
    z = stereo_project(K, lie.transform_to(X_gt[fr], pw[tid])) + rng.normal(0, pixel_sigma, (tid.size, 3))
    bad = rng.uniform(0, 1, tid.size) < outlier_fraction
    z[bad] = np.stack([rng.uniform(0, IMG_W, bad.sum()), rng.uniform(0, IMG_W, bad.sum()), rng.uniform(0, IMG_H, bad.sum())], 1)
    z[rng.uniform(0, 1, tid.size) < nan_right, 1] = np.nan
    order = np.argsort(fr, kind="stable")
    return dict(frame=fr[order], tracklet=tid[order].astype(np.int64), stereo=z[order], points=pw)


def make_scene(n_frames=20, n_static=300, seed=0, n_objects=0, n_dynamic=0, imu=False, init_noise_rot=2e-4,
               init_noise_trans=2e-3, **kw):
    """synth.make_problem's camera chain (and dynamic tracklets) with stereo static observations: (problem, static).  The
    initial camera poses are those of a front end that tracks well (the default noise keeps most reprojection norms under
    the formulation's 3 px)."""
    from . import synth
    p = synth.make_problem(n_frames=n_frames, n_objects=n_objects, n_static=0, n_dynamic=n_dynamic, seed=seed, imu=imu,
                           object_span=(n_frames, n_frames) if n_objects else None, init_noise_rot=init_noise_rot,
                           init_noise_trans=init_noise_trans)
    return p, make_static_stereo(p.meta["gt_camera"], n_static, seed=seed + 1, **kw)


def full_track_problems(X, static, K=KITTI_K):
    """one triangulation problem per landmark over its whole track -- the left camera of every observation and the right
    camera where uR is finite -- as the flat arrays of dynoba_triangulate_batch: (offsets, poses [c, 12], kp [c, 2], calib5)"""
    fr, tr, z = static["frame"], static["tracklet"], static["stereo"]
    order = np.lexsort((fr, tr)); fr, tr, z = fr[order], tr[order], z[order]
    right = np.isfinite(z[:, 1])
    XR = X.copy(); XR[:, 9:] = X[:, 9:] + K[5]*X[:, [0, 3, 6]]      # X * (I, (b, 0, 0))
    ncam = 1 + right.astype(np.int64)
    start = np.concatenate([[0], np.cumsum(ncam)])
    poses = np.zeros((start[-1], 12)); kp = np.zeros((start[-1], 2))
    poses[start[:-1]] = X[fr]; kp[start[:-1]] = z[:, [0, 2]]
    ri = start[:-1][right] + 1
    poses[ri] = XR[fr[right]]; kp[ri] = z[right][:, [1, 2]]
    first = np.flatnonzero(np.r_[True, tr[1:] != tr[:-1]])
    offsets = np.concatenate([start[first], [start[-1]]]).astype(np.int32)
    calib = np.tile(np.asarray(K, np.float64)[:5], (first.size, 1))
    return offsets, poses, kp, calib
