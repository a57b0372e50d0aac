"""CPU oracle for depth and back-projection (libdynofront dynofront_update_depths / back_project / dense_cloud).

Restates, in numpy, what the reference computes per frame:
  * Frame::updateDepthsFeatureContainer (Frame.cc:430-467): d = depth(int(v), int(u)); d > max || d <= 0 -> invalid, NaN depth;
  * Camera::backProject (Camera.cc:88-99): gtsam::PinholeCamera<Cal3_S2> at the identity pose, Cal3_S2::calibrate in GTSAM 4.2's
    operation order, BackprojectFromCamera (x d, y d, d), then X_world * p;
  * RGBDCamera::projectRight (RGBDCamera.cc:49,61-87): uR = uL - (fx b) / d, out of the image when uR < 0 || uR > W;
  * the per-feature loop of RGBDInstanceFrontendModule::fillOutputPacketWithTracks (:415-486);
  * Frame::projectToDenseCloud (Frame.cc:172-238) with Color::uniqueId / fromHSV (Colour.cc:73-100,178-185).
Every float64 / float32 operation is one IEEE operation in the stated order, so the device results are compared bit for bit.
calib5 = (fx, fy, s, u0, v0); poses are 12 doubles (row-major R, then t).
"""
from __future__ import annotations

import numpy as np

MAX_BACKGROUND_DEPTH, MAX_OBJECT_DEPTH = 200.0, 30.0     # params/FrontendParams.yaml


def calibrate(u, v, calib5):
    """Cal3_S2::calibrate: delta_u = u - u0, delta_v = v - v0, inv_fy_delta_v = (1/fy) delta_v,
    x = (1/fx) (delta_u - s inv_fy_delta_v), y = inv_fy_delta_v"""
    fx, fy, s, u0, v0 = (np.float64(c) for c in calib5)
    du = np.asarray(u, np.float64) - u0; dv = np.asarray(v, np.float64) - v0
    inv_fx = np.float64(1.0)/fx; inv_fy = np.float64(1.0)/fy
    ify_dv = inv_fy*dv
    return inv_fx*(du - s*ify_dv), ify_dv


def backproject_camera(u, v, d, calib5):
    """PinholeCamera::backproject at the identity pose (the identity transform itself not applied): [n][3]"""
    x, y = calibrate(u, v, calib5)
    d = np.asarray(d, np.float64)
    return np.stack(np.broadcast_arrays(x*d, y*d, d), -1)


def transform_from(X, p):
    """Pose3::transformFrom with the sum order q_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i"""
    X = np.asarray(X, np.float64).reshape(12); p = np.asarray(p, np.float64)
    out = np.empty_like(p)
    for r in range(3):
        out[..., r] = ((X[3*r]*p[..., 0] + X[3*r + 1]*p[..., 1]) + X[3*r + 2]*p[..., 2]) + X[9 + r]
    return out


def update_depths(kp, label, depth, max_background_depth=MAX_BACKGROUND_DEPTH, max_object_depth=MAX_OBJECT_DEPTH):
    """(depth_out, valid, n_invalid, n_outside), feature by feature as the reference loop"""
    kp = np.asarray(kp, np.float64).reshape(-1, 2); H, W = depth.shape
    n = len(kp); dout = np.full(n, np.nan); valid = np.zeros(n, np.uint8); n_inv = n_out = 0
    for i in range(n):
        u, v = kp[i]
        mx = max_background_depth if int(label[i]) == 0 else max_object_depth
        if not (-1.0 < u < W and -1.0 < v < H):             # truncated pixel outside the image (or NaN): defined as invalid
            n_inv += 1; n_out += 1
            continue
        d = depth[int(v), int(u)]                            # int() truncates toward zero, as static_cast<int>
        if d > mx or d <= 0:
            n_inv += 1                                       # markInvalid(), depth(Feature::invalid_depth)
        else:
            dout[i] = d; valid[i] = 1                        # NaN lands here: valid, no depth
    return dout, valid, n_inv, n_out


def right_u(u, d, fx, baseline):
    """RGBDCamera::rightKeypoint: fx_b_ = fx * baseline once, then uL - fx_b_ / depth"""
    fx_b = np.float64(fx)*np.float64(baseline)
    return np.float64(u) - fx_b/np.float64(d)


def back_project(kp, depth, usable, calib5, W, baseline=0.0, rgbd=False, right=None, X_world=None):
    """the per-feature loop of fillOutputPacketWithTracks: (index, point [m][3], stereo [m][3], outlier [n])"""
    kp = np.asarray(kp, np.float64).reshape(-1, 2); n = len(kp)
    index, points, stereo = [], [], []; outlier = np.zeros(n, np.uint8)
    for i in range(n):
        if not usable[i]:
            continue
        u, v = kp[i]; d = np.float64(depth[i])
        p = np.full(3, np.nan); s = np.full(3, np.nan)
        has_depth = not np.isnan(d)
        if has_depth:
            p = backproject_camera(u, v, d, calib5)
            if X_world is not None:
                p = transform_from(X_world, p)
        ur = np.nan if right is None else np.float64(right[i])
        if not np.isnan(ur):
            s = np.array([u, ur, v])
        elif rgbd and has_depth:
            ur = right_u(u, d, calib5[0], baseline)
            if ur < 0.0 or ur > W:                           # markOutlier(); continue
                outlier[i] = 1
                continue
            s = np.array([u, ur, v])
        index.append(i); points.append(p); stereo.append(s)
    return (np.array(index, np.int32), np.array(points).reshape(-1, 3), np.array(stereo).reshape(-1, 3), outlier)


def unique_id_rgb(ids):
    """Color::uniqueId(size_t(id), 0.5f, 0.95f) -> uint8 [n][3], in the reference's float / double mix"""
    f32 = np.float32
    ids = np.asarray(ids, np.int64)
    phi = f32((1.0 + np.sqrt(5.0))/2.0)
    fid = ids.astype(np.uint64).astype(np.float32)           # (float)(size_t)id
    t = fid*phi
    n = t - np.floor(t)                                      # float
    hue = (np.floor(n.astype(np.float64)*256.0)/255.0).astype(np.float32)
    hue = np.clip(hue, f32(0), f32(1))
    value = f32(0.95); chroma = value*f32(0.5)
    hp = hue*f32(6.0)
    # std::fmod(float, int) is the double overload; 1.0f - |...| and chroma * (...) stay double; x is rounded to float
    x = (np.float64(chroma)*(1.0 - np.abs(np.fmod(hp.astype(np.float64), 2.0) - 1.0))).astype(np.float32)
    z = np.zeros_like(x); c = np.full_like(x, chroma)
    conds = [hp < 1, hp < 2, hp < 3, hp < 4, hp < 5]
    r1 = np.select(conds, [c, x, z, z, x], c); g1 = np.select(conds, [x, c, c, x, z], z); b1 = np.select(conds, [z, z, x, c, c], x)
    m = value - chroma
    return np.stack([((ch + m)*f32(255)).astype(np.uint8) for ch in (r1, g1, b1)], -1)


def dense_cloud(depth, motion_mask, detection_mask, calib5, max_background_depth=MAX_BACKGROUND_DEPTH, max_object_depth=MAX_OBJECT_DEPTH):
    """projectToDenseCloud as planar arrays: (xyz f32[H][W][3], rgb u8[H][W][3], label u32[H][W], valid u8[H][W])"""
    H, W = depth.shape
    ok = np.ones((H, W), bool) if detection_mask is None else detection_mask != 0
    thresh = np.where(motion_mask == 0, max_background_depth, max_object_depth)
    with np.errstate(invalid="ignore"):
        ok &= ~((depth > thresh) | (depth <= 0) | ~np.isfinite(depth))
    ys, xs = np.nonzero(ok)
    xyz = np.zeros((H, W, 3), np.float32); rgb = np.zeros((H, W, 3), np.uint8); lab = np.zeros((H, W), np.uint32)
    xyz[ys, xs] = backproject_camera(xs.astype(np.float64), ys.astype(np.float64), depth[ys, xs], calib5).astype(np.float32)
    oid = motion_mask[ys, xs]
    obj = oid != 0
    rgb[ys[obj], xs[obj]] = unique_id_rgb(oid[obj])
    lab[ys, xs] = oid.astype(np.int64).astype(np.uint32)
    return xyz, rgb, lab, ok.astype(np.uint8)
