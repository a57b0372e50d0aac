"""Seeded multi-frame sequences for the object-motion filter (dynoba_object_srif_batch): a moving RGB-D camera and several rigid
objects moving at near-constant velocity, with per-frame PnP inliers, back-projected camera-frame points (depth noise) and
fake-stereo key-points (uR = uL - fx b / depth, as RGBDCamera::rightKeypoint).  Objects appear and leave; an object is
resampled (fresh tracklets) every `resample_every` frames of its life and whenever it comes back."""
from __future__ import annotations

import numpy as np

from .lie import se3_exp

CALIB6 = np.array([320.0, 320.0, 0.0, 320.0, 240.0, 0.1])    # fx, fy, skew, u0, v0, baseline


def pose12(T):
    return np.concatenate([T[:3, :3].reshape(9), T[:3, 3]])


def _exp(xi):
    p = se3_exp(np.asarray(xi, dtype=np.float64))[0]
    T = np.eye(4); T[:3, :3] = p[:9].reshape(3, 3); T[:3, 3] = p[9:]
    return T


def make_sequence(n_frames=30, n_objects=4, n_points=60, seed=0, resample_every=9, invalid_rate=0.05, few_first=False,
                  calib=CALIB6):
    """dict(calib[6], poses[n_frames, 12], frames): frames[k - 1] (k = 1 .. n_frames - 1) is a list of objects seen at k, each
    dict(object_id, resampled, pnp_status, tracklets[n], stereo[n, 6], valid[n, 2], points[n, 6]) over its PnP inliers.
    few_first: the first frame of object 0 has 3 inliers (too few to start a filter)."""
    rng = np.random.default_rng(seed)
    fx, fy, _, u0, v0, b = calib
    X = [np.eye(4)]
    vc = np.array([0.0, 0.01, 0.0, 0.02, 0.0, 0.15])
    for k in range(1, n_frames):
        X.append(X[-1] @ _exp(vc + 0.002*rng.standard_normal(6)))
    objs = []
    for o in range(n_objects):
        L0 = np.eye(4); L0[:3, 3] = [rng.uniform(-2.5, 2.5), rng.uniform(-1.0, 1.0), rng.uniform(7.0, 12.0)]
        a = 0 if o < 2 else int(rng.integers(1, max(2, n_frames//3)))
        e = n_frames if o % 2 == 0 else int(rng.integers(2*n_frames//3, n_frames))
        gap = (a + 5, a + 7) if o == n_objects - 1 and n_frames > a + 12 else None     # leaves for two frames, comes back
        objs.append(dict(L=[L0], v=np.concatenate([0.03*rng.standard_normal(3), 0.1*rng.standard_normal(3)]),
                         pts=rng.uniform(-0.8, 0.8, (n_points, 3)), a=a, e=e, gap=gap, gen=0, seen=False, last=-2))
    frames = []
    for k in range(1, n_frames):
        fr = []
        for o, ob in enumerate(objs):
            ob["L"].append(ob["L"][-1] @ _exp(ob["v"] + 0.003*rng.standard_normal(6)))
            present = ob["a"] < k < ob["e"] and not (ob["gap"] and ob["gap"][0] <= k < ob["gap"][1])
            if not present:
                continue
            resampled = ob["last"] != k - 1 or (k - ob["a"]) % resample_every == 0
            if resampled:
                ob["gen"] += 1
            ob["last"] = k
            keep = rng.random(n_points) < 0.9
            if few_first and o == 0 and not ob["seen"]:
                keep[:] = False; keep[:3] = True
            ob["seen"] = True
            idx = np.nonzero(keep)[0]
            rec = dict(object_id=o, resampled=bool(resampled), pnp_status=0 if rng.random() > 0.1 else 2,
                       tracklets=(1000000*o + 1000*ob["gen"] + idx).astype(np.int64))
            stereo = np.zeros((len(idx), 6)); valid = np.ones((len(idx), 2), dtype=bool); pts = np.zeros((len(idx), 6))
            for f, kk in enumerate((k - 1, k)):
                Pw = (ob["L"][kk][:3, :3] @ ob["pts"][idx].T).T + ob["L"][kk][:3, 3]
                Xi = np.linalg.inv(X[kk])
                pc = (Xi[:3, :3] @ Pw.T).T + Xi[:3, 3]
                depth = pc[:, 2] + 0.01*rng.standard_normal(len(idx))
                uL = fx*pc[:, 0]/pc[:, 2] + u0 + 0.3*rng.standard_normal(len(idx))
                vv = fy*pc[:, 1]/pc[:, 2] + v0 + 0.3*rng.standard_normal(len(idx))
                # back-projection of the key-point at the measured depth
                yn = (vv - v0)/fy; xn = (uL - u0)/fx
                pts[:, 3*f:3*f + 3] = np.stack([xn*depth, yn*depth, depth], 1)
                stereo[:, 3*f:3*f + 3] = np.stack([uL, uL - fx*b/depth, vv], 1)
                valid[:, f] = rng.random(len(idx)) >= invalid_rate
            stereo[~np.repeat(valid, 3, axis=1)] = np.nan        # a missing right key-point has no value
            rec.update(stereo=stereo, valid=valid, points=pts)
            fr.append(rec)
        frames.append(fr)
    return dict(calib=np.asarray(calib, dtype=np.float64), poses=np.stack([pose12(T) for T in X]), frames=frames)


def random_frame(n_objects, n_inliers, seed=0, calib=CALIB6):
    """one frame of n_objects NEW objects of n_inliers PnP inliers each (the bench and the batch-size tests), as the objects
    of binding.object_srif_batch"""
    rng = np.random.default_rng(seed)
    fx, fy, _, u0, v0, b = calib
    X0, X1 = np.eye(4), _exp([0.0, 0.01, 0.0, 0.02, 0.0, 0.15])
    out = []
    for o in range(n_objects):
        L0 = np.eye(4); L0[:3, 3] = [rng.uniform(-2.5, 2.5), rng.uniform(-1.0, 1.0), rng.uniform(7.0, 12.0)]
        L1 = L0 @ _exp(np.concatenate([0.03*rng.standard_normal(3), 0.1*rng.standard_normal(3)]))
        m = rng.uniform(-0.8, 0.8, (n_inliers, 3))
        stereo = np.zeros((n_inliers, 6)); pts = np.zeros((n_inliers, 6))
        for f, (X, L) in enumerate(((X0, L0), (X1, L1))):
            Xi = np.linalg.inv(X)
            pc = (Xi[:3, :3] @ ((L[:3, :3] @ m.T).T + L[:3, 3]).T).T + Xi[:3, 3]
            depth = pc[:, 2] + 0.01*rng.standard_normal(n_inliers)
            uL = fx*pc[:, 0]/pc[:, 2] + u0 + 0.3*rng.standard_normal(n_inliers)
            vv = fy*pc[:, 1]/pc[:, 2] + v0 + 0.3*rng.standard_normal(n_inliers)
            pts[:, 3*f:3*f + 3] = np.stack([(uL - u0)/fx*depth, (vv - v0)/fy*depth, depth], 1)
            stereo[:, 3*f:3*f + 3] = np.stack([uL, uL - fx*b/depth, vv], 1)
        out.append(dict(mode=0, pnp_status=0, pose_prev=pose12(X0), pose_cur=pose12(X1), calib=np.asarray(calib, dtype=np.float64),
                        state=np.zeros(90), stereo=stereo, valid=np.ones((n_inliers, 2), dtype=bool), points=pts,
                        m_L=np.zeros((n_inliers, 3)), has_point=np.zeros(n_inliers, dtype=bool)))
    return out
