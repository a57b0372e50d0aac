"""Seeded synthetic DynOSAM batch graphs (SURVEY.md 8d / Appendix D).

Reproduces the *topology rules* of the reference's formulations (who is connected to whom, with
which factor type and noise), scaled to the BASELINE.json configs:

* camera chain: PriorFactor(X_0, sigma 1e-6) + BetweenFactor odometry
  (dynosam/include/dynosam/backend/VisionImuBackendModule.hpp:168-243, BackendDefinitions.cc:124-140)
* static points: PoseToPointFactor per observation, >= min_static_observations (2), track age <= 15
  (backend/Formulation-impl.hpp:145-212)
* HYBRID: one m_L per tracklet, HybridMotionFactor(X_k, H_k^j, m_L; z, L_e) per observation,
  PriorFactor(H_e = I, 1e-6) at the object key-frame, 3-motion HybridSmoothingFactor
  (src/backend/rgbd/HybridEstimator.cc:573-830)
* WCME: one point per (tracklet, frame), PoseToPoint + LandmarkMotionTernaryFactor chain, motion
  BetweenFactor smoothing (src/backend/rgbd/WorldMotionEstimator.cc:151-351)
* WCPE: one point per (tracklet, frame), PoseToPoint + LandmarkMotionPoseFactor(m_k-1, m_k, L_k-1, L_k) chain over
  object POSE variables L_k^j (one per frame the object is seen, no prior), 3-pose LandmarkPoseSmoothingFactor
  (src/backend/rgbd/WorldPoseEstimator.cc:89-315)

The trajectories follow test/internal/simulator.hpp's ConstantMotionBodyVisitor (constant twist).
All randomness comes from numpy's PCG64 seeded generator (the reference's simulator is not
reproducible, SURVEY.md section 4), so graphs are identical on every machine.
"""
from __future__ import annotations

import numpy as np

from . import lie
from .problem import (BETWEEN6, HYBRID3, MOTIONPOSE3, POSE2POINT3, PRIOR6, SMOOTH_HYBRID6, SMOOTH_POSE6, TERNARY3, FactorBlock, Problem,
                      camera_pose_key, dynamic_landmark_key, object_motion_key, object_pose_key, static_landmark_key)

KITTI_K = np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372])
IMG_W, IMG_H = 1242, 375

CONFIGS = {
    # name: (frames, objects, static landmarks, dynamic tracklets)
    "C1": dict(n_frames=20, n_objects=1, n_static=700, n_dynamic=300),
    "C2": dict(n_frames=2000, n_objects=0, n_static=500_000, n_dynamic=0),
    "C3": dict(n_frames=2000, n_objects=20, n_static=500_000, n_dynamic=500_000),
    "C5": dict(n_frames=10_000, n_objects=100, n_static=1_000_000, n_dynamic=1_000_000),
}


def _tracks(rng, n, first_lo, first_hi, life_lo, life_hi, end):
    """birth frame in [first_lo, first_hi], life in [life_lo, life_hi] clipped at `end` (exclusive)."""
    birth = rng.integers(first_lo, np.maximum(first_hi, first_lo) + 1, size=n)
    life = rng.integers(life_lo, life_hi + 1, size=n)
    life = np.minimum(life, end - birth)
    return birth.astype(np.int64), life.astype(np.int64)


def _expand(life):
    """for tracks with lengths `life` return (track index, offset within track) per observation."""
    start = np.concatenate([[0], np.cumsum(life)])
    tid = np.repeat(np.arange(life.shape[0]), life)
    off = np.arange(start[-1]) - start[tid]
    return tid, off, start


def make_problem(n_frames=20, n_objects=1, n_static=700, n_dynamic=300, formulation="hybrid", seed=42,
                 sigma_point=0.2, sigma_ternary=0.01, huber_k=1e-4, robust=True, meas_noise=None,
                 init_noise_rot=0.01, init_noise_trans=0.05, object_span=None, max_static_age=15,
                 max_dynamic_age=20, with_odometry=True, imu=False) -> Problem:
    """imu=True: the camera chain is visual-inertial (synth_imu.add_imu_chain): velocities, biases, their priors and one
    COMBINED_IMU15 per frame pair replace the odometry factors."""
    assert formulation in ("hybrid", "wcme", "wcpe")
    rng = np.random.default_rng(seed)
    N = int(n_frames)
    meas_noise = sigma_point if meas_noise is None else meas_noise
    kh = huber_k if robust else 0.0

    # ---------------- camera trajectory (constant twist)
    xi_cam = np.array([0.0, 0.004, 0.0, 0.02, 0.0, 1.0])
    X_gt = lie.se3_exp(np.arange(N)[:, None]*xi_cam[None])
    X_init = lie.retract(X_gt, np.concatenate([rng.normal(0, init_noise_rot, (N, 3)), rng.normal(0, init_noise_trans, (N, 3))], 1))
    X_init[0] = X_gt[0]

    blocks = []
    # ---------------- static landmarks
    ns = int(n_static)
    pts_init = [np.zeros((0, 3))]
    pt_keys = [np.zeros(0, dtype=np.uint64)]
    if ns:
        birth, life = _tracks(rng, ns, 0, N - 2, 2, max_static_age, N)
        order = np.argsort(birth, kind="stable"); birth, life = birth[order], life[order]
        d = rng.uniform(2.0, 50.0, ns); u = rng.uniform(0, IMG_W, ns); v = rng.uniform(0, IMG_H, ns)
        pc = np.stack([(u - KITTI_K[3])/KITTI_K[0]*d, (v - KITTI_K[4])/KITTI_K[1]*d, d], 1)
        pw = lie.transform_from(X_gt[birth], pc)
        tid, off, start = _expand(life)
        fr = birth[tid] + off
        z = lie.transform_to(X_gt[fr], pw[tid]) + rng.normal(0, meas_noise, (tid.shape[0], 3))
        p0 = lie.transform_from(X_init[birth], z[start[:-1]])      # initial = X_init * first measurement
        pts_init.append(p0); pt_keys.append(static_landmark_key(np.arange(ns)))
        blocks.append(FactorBlock(POSE2POINT3, np.stack([fr, tid], 1), z, np.array([sigma_point]), kh))

    # ---------------- objects
    J = int(n_objects); nd = int(n_dynamic) if J else 0
    pose_list = [X_init]; order_hint = [np.arange(N)]
    pose_keys = [camera_pose_key(np.arange(N))]
    aux = np.zeros((0, 12))
    gt_motion = None
    dyn_obs = None
    n_pt_static = ns
    if J:
        if object_span is None:
            object_span = (min(N, 400), min(N, 600)) if N > 40 else (N, N)
        D = rng.integers(object_span[0], object_span[1] + 1, J)
        slots = np.linspace(0, 1, J, endpoint=False) + rng.uniform(0, 1.0/J, J)
        s = np.floor(slots*(N - D + 1)).astype(np.int64); s = np.clip(s, 0, N - D)
        # object pose at its first frame: in front of the camera
        yaw = rng.uniform(-0.5, 0.5, J)
        off = np.stack([rng.uniform(-6, 6, J), rng.uniform(-0.5, 0.5, J), rng.uniform(8, 30, J)], 1)
        L_rel = lie.pack(np.stack([lie.ypr(0.0, y, 0.0) for y in yaw]), off)
        L_e = lie.compose(X_gt[s], L_rel)                          # object pose at key-frame e = s_j
        xi_obj = np.stack([rng.normal(0, 0.002, J), rng.uniform(-0.02, 0.02, J), rng.normal(0, 0.002, J),
                           rng.uniform(-0.3, 0.3, J), rng.normal(0, 0.02, J), rng.uniform(0.4, 1.2, J)], 1)
        aux = L_e
        # motion variable layout: object-major, frames s_j .. s_j+D_j-1 (WCME skips the first frame)
        skip = 1 if formulation == "wcme" else 0
        cnt = D - skip
        hstart = N + np.concatenate([[0], np.cumsum(cnt)])         # pose index of the first motion of object j
        oj, ok, _ = _expand(cnt)
        hframe = s[oj] + ok + skip                                 # frame of each motion variable
        if formulation == "hybrid":
            H_gt = lie.se3_exp((hframe - s[oj])[:, None]*xi_obj[oj])   # e_H_k = H^(k-e)
        elif formulation == "wcme":
            H_gt = lie.se3_exp(xi_obj[oj])                             # k-1 -> k motion (constant)
        else:
            H_gt = lie.compose(lie.se3_exp((hframe - s[oj])[:, None]*xi_obj[oj]), L_e[oj])   # object pose L_k = e_H_k L_e
        H_init = lie.retract(H_gt, np.concatenate([rng.normal(0, init_noise_rot, (H_gt.shape[0], 3)),
                                                   rng.normal(0, init_noise_trans, (H_gt.shape[0], 3))], 1))
        if formulation == "hybrid":
            H_init[hstart[:-1] - N] = lie.identity(J)               # key-frame motion starts at its prior
        pose_list.append(H_init); order_hint.append(hframe); gt_motion = H_gt
        pose_keys.append((object_pose_key if formulation == "wcpe" else object_motion_key)(oj + 1, hframe))

        # ---------------- dynamic tracklets
        per = np.full(J, nd//J); per[:nd - per.sum()] += 1
        tobj = np.repeat(np.arange(J), per)
        lo = s[tobj]; hi = s[tobj] + D[tobj] - 3
        birth = (lo + np.floor(rng.uniform(0, 1, nd)*(hi - lo + 1))).astype(np.int64)
        life = np.minimum(rng.integers(3, max_dynamic_age + 1, nd), s[tobj] + D[tobj] - birth)
        key = tobj*(N + 1) + birth
        order = np.argsort(key, kind="stable"); tobj, birth, life = tobj[order], birth[order], life[order]
        mL = rng.uniform(-1, 1, (nd, 3))*np.array([2.0, 1.0, 1.0])
        tid, off, start = _expand(life)
        fr = birth[tid] + off
        E_k = lie.se3_exp((fr - s[tobj[tid]])[:, None]*xi_obj[tobj[tid]])       # e_H_k (gt)
        mW = lie.transform_from(E_k, lie.transform_from(L_e[tobj[tid]], mL[tid]))
        z = lie.transform_to(X_gt[fr], mW) + rng.normal(0, meas_noise, (tid.shape[0], 3))
        hidx = hstart[tobj[tid]] + (fr - s[tobj[tid]]) - skip                    # motion var of (object, frame)
        dyn_obs = dict(frame=fr, tracklet=tid + ns, object=tobj[tid] + 1)        # per dynamic observation, in block order
        if formulation == "hybrid":
            # m_L init = L_e^-1 * E^-1 * X * z at the first observation (HybridObjectMotion::projectToObject3)
            f0 = start[:-1]
            E0 = pose_list[1][hidx[f0] - N]
            w0 = lie.transform_from(X_init[fr[f0]], z[f0])
            m0 = lie.transform_to(L_e[tobj], lie.transform_to(E0, w0))
            pts_init.append(m0)
            pt_keys.append(dynamic_landmark_key(np.zeros(nd, dtype=np.uint64), np.arange(nd) + ns))
            blocks.append(FactorBlock(HYBRID3, np.stack([fr, hidx, n_pt_static + tid], 1), z, np.array([sigma_point]), kh,
                                      aux_idx=tobj[tid]))
            # priors on the key-frame motions + 3-motion smoothing
            blocks.append(FactorBlock(PRIOR6, (hstart[:-1]).reshape(-1, 1), lie.identity(J), np.full(6, 1e-6)))
            tri_j, tri_o, _ = _expand(np.maximum(cnt - 2, 0))
            if tri_j.size:
                i0 = hstart[tri_j] + tri_o
                blocks.append(FactorBlock(SMOOTH_HYBRID6, np.stack([i0, i0 + 1, i0 + 2], 1), None,
                                          np.array([0.01, 0.01, 0.01, 0.1, 0.1, 0.1]), aux_idx=tri_j))
        else:
            npt = tid.shape[0]
            pidx = n_pt_static + np.arange(npt)
            pts_init.append(lie.transform_from(X_init[fr], z))
            pt_keys.append(dynamic_landmark_key(fr, tid + ns))
            blocks.append(FactorBlock(POSE2POINT3, np.stack([fr, pidx], 1), z, np.array([sigma_point]), kh))
            notfirst = off > 0
            cur = np.nonzero(notfirst)[0]
            if formulation == "wcme":
                blocks.append(FactorBlock(TERNARY3, np.stack([pidx[cur - 1], pidx[cur], hidx[cur]], 1), None,
                                          np.array([sigma_ternary]), kh))
                sm_j, sm_o, _ = _expand(np.maximum(cnt - 1, 0))
                if sm_j.size:
                    i0 = hstart[sm_j] + sm_o
                    blocks.append(FactorBlock(BETWEEN6, np.stack([i0, i0 + 1], 1), lie.identity(i0.shape[0]),
                                              np.array([0.01, 0.01, 0.01, 0.1, 0.1, 0.1])))
            else:
                # LandmarkMotionPoseFactor(m_k-1, m_k, L_k-1, L_k) (WorldPoseEstimator.cc:170-178) + 3-pose smoothing (:259-306)
                blocks.append(FactorBlock(MOTIONPOSE3, np.stack([pidx[cur - 1], pidx[cur], hidx[cur] - 1, hidx[cur]], 1), None,
                                          np.array([sigma_ternary]), kh))
                tri_j, tri_o, _ = _expand(np.maximum(cnt - 2, 0))
                if tri_j.size:
                    i0 = hstart[tri_j] + tri_o
                    blocks.append(FactorBlock(SMOOTH_POSE6, np.stack([i0, i0 + 1, i0 + 2], 1), None,
                                              np.array([0.01, 0.01, 0.01, 0.1, 0.1, 0.1])))

    # ---------------- camera chain
    blocks.append(FactorBlock(PRIOR6, np.array([[0]]), X_gt[:1], np.full(6, 1e-6)))
    nav = None
    if imu:
        from .synth_imu import add_imu_chain
        vel0, bias0, imu_blocks, imu_meta = add_imu_chain(X_gt, xi_cam, seed + 7919)
        blocks.extend(imu_blocks)
        nav = dict(vel=vel0, bias=bias0, vel_order=np.arange(N, dtype=np.int32), bias_order=np.arange(N, dtype=np.int32))
    elif with_odometry and N > 1:
        rel = lie.between(X_gt[:-1], X_gt[1:])
        rel = lie.retract(rel, np.concatenate([rng.normal(0, 0.02, (N - 1, 3)), rng.normal(0, 0.01, (N - 1, 3))], 1))
        blocks.append(FactorBlock(BETWEEN6, np.stack([np.arange(N - 1), np.arange(1, N)], 1), rel,
                                  np.array([0.02, 0.02, 0.02, 0.01, 0.01, 0.01])))

    prob = Problem(np.concatenate(pose_list), np.concatenate(pts_init), aux_pose=aux, calib=KITTI_K, blocks=blocks,
                   pose_order=np.concatenate(order_hint).astype(np.int32),
                   pose_keys=np.concatenate(pose_keys), point_keys=np.concatenate(pt_keys), **(nav or {}))
    prob.meta = dict(n_frames=N, n_objects=J, n_static=ns, n_dynamic=nd, formulation=formulation, seed=seed,
                     gt_camera=X_gt, gt_motion=gt_motion, dyn_obs=dyn_obs)
    if imu:
        prob.meta.update(imu_meta)
    return prob


def make_config(name: str, formulation="hybrid", seed=42, scale=1.0, **kw) -> Problem:
    cfg = dict(CONFIGS[name])
    if scale != 1.0:
        for k in ("n_frames", "n_objects", "n_static", "n_dynamic"):
            cfg[k] = max(int(round(cfg[k]*scale)), 1 if k == "n_frames" else 0)
    cfg.update(kw)
    p = make_problem(formulation=formulation, seed=seed, **cfg)
    p.meta["config"] = name
    return p


def make_all_types_problem(seed=3) -> Problem:
    from .problem import FLOWPROJ2, HYBRID_STEREO3, MOTIONPOSE3, SMOOTH_POSE6, STEREO3
    """A graph holding every factor type of SURVEY.md 8a (a3-a9, a15) on random but well-posed inputs."""
    rng = np.random.default_rng(seed)
    base = make_problem(n_frames=12, n_objects=2, n_static=150, n_dynamic=80, formulation="hybrid", seed=seed)
    N = base.meta["n_frames"]; npose = base.n_pose; npt = base.n_point
    K = np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372])
    blocks = list(base.blocks)
    # stereo observations of the first 100 static points from their first frames (positive depth by construction)
    ptp = base.blocks[0]
    sel = np.arange(0, min(300, ptp.n))
    cam = ptp.idx[sel, 0]; pid = ptp.idx[sel, 1]
    q = lie.transform_to(base.pose[cam], base.point[pid])
    q[:, 2] = np.abs(q[:, 2]) + 1.0
    zs = np.stack([K[3] + K[0]*q[:, 0]/q[:, 2], K[3] + K[0]*(q[:, 0] - K[5])/q[:, 2], K[4] + K[1]*q[:, 1]/q[:, 2]], 1)
    zs += rng.normal(0, 1.0, zs.shape)
    blocks.append(FactorBlock(STEREO3, np.stack([cam, pid], 1), zs, np.array([1.5, 1.5, 2.0]), 1.345))
    # a cheirality case: a point behind the camera
    hyb = [b for b in base.blocks if b.type == HYBRID3][0]
    hs = np.arange(0, min(200, hyb.n))
    blocks.append(FactorBlock(HYBRID_STEREO3, hyb.idx[hs], rng.uniform(0, 300, (hs.size, 3)), np.array([2.0]), 0.0,
                              aux_idx=hyb.aux_idx[hs]))
    # world-centric pieces on fresh point variables
    extra_pts = rng.normal(0, 3, (60, 3)) + [0, 0, 10]
    pts = np.concatenate([base.point, extra_pts]); e0 = npt
    mot = np.arange(N, npose)
    ch = np.array([i for i in range(39) if i % 10 != 9])                 # four chains of 10 points
    tri = np.stack([e0 + ch, e0 + ch + 1, rng.choice(mot, ch.size)], 1)
    blocks.append(FactorBlock(TERNARY3, tri, None, np.array([0.01]), 1e-4))
    mp = np.stack([e0 + np.arange(40, 58), e0 + np.arange(41, 59), rng.choice(mot, 18), rng.choice(mot, 18)], 1)
    blocks.append(FactorBlock(MOTIONPOSE3, mp, None, np.array([0.05]), 1e-3))
    sp = np.stack([mot[:-2][:20], mot[1:-1][:20], mot[2:][:20]], 1)
    blocks.append(FactorBlock(SMOOTH_POSE6, sp, None, np.array([0.01, 0.01, 0.01, 0.1, 0.1, 0.1])))
    # flow-projection star: 30 flows attached to camera 3
    flows = rng.normal(0, 1.0, (30, 2))
    kp = np.stack([rng.uniform(100, 1100, 30), rng.uniform(50, 320, 30)], 1); depth = rng.uniform(4, 30, 30)
    meas = np.concatenate([kp, depth[:, None], np.tile(base.pose[2], (30, 1))], 1)
    blocks.append(FactorBlock(FLOWPROJ2, np.stack([np.arange(30), np.full(30, 3)], 1), meas, np.array([0.5]), 0.0))
    return Problem(base.pose, pts, flow=flows, aux_pose=base.aux_pose, calib=K, blocks=blocks, pose_order=base.pose_order)
