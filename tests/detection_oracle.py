"""CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT) for static feature detection on the device.

KltFeatureTracker::detectFeatures   dynosam/src/frontend/vision/StaticFeatureTracker.cc:330-418
SparseFeatureDetector::detect       dynosam/src/frontend/vision/FeatureDetector.cc:187-239
composed from the OpenCV routines the reference calls (cv2.createCLAHE, cv2.GFTTDetector, cv2.cornerSubPix) and the
range-tree ANMS of selection_oracle, plus a literal restatement of the mask build and of the filter / tracklet-id loop.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import selection_oracle as SO


@dataclass
class Params:
    use_clahe: bool = True
    use_anms: bool = True
    use_subpix: bool = True
    max_corners: int = 1000
    quality_level: float = 0.001
    min_distance: int = 15
    max_features: int = 800
    shrink_row: int = 0
    shrink_col: int = 0


def detection_mask(motion_mask, boundary_mask, cur_kp, radius):
    """detection_mask_impl: the boundary mask (255 without one) AND motion_mask == 0, then cv::circle(FILLED, 0) around every
    current feature at cv::Point(cv::Point2f(kp)): the double key-point becomes float, then cvRound (half to even, as np.rint)."""
    import cv2
    rows, cols = motion_mask.shape
    m = (boundary_mask.copy() if boundary_mask is not None else np.full((rows, cols), 255, np.uint8)).astype(np.uint8)
    m = cv2.bitwise_and(m, np.where(motion_mask == 0, 255, 0).astype(np.uint8))
    for x, y in np.asarray(cur_kp, np.float64).reshape(-1, 2):
        c = (int(np.rint(np.float32(x))), int(np.rint(np.float32(y))))
        cv2.circle(m, c, int(radius), 0, cv2.FILLED)
    return m


def stages(gray, mask, prm: Params):
    """the processed image, cv2.cornerMinEigenVal and the GFTT corners (integer (x, y), detector order) with their responses"""
    import cv2
    img = cv2.createCLAHE(2.0, (8, 8)).apply(gray) if prm.use_clahe else gray.copy()
    eig = cv2.cornerMinEigenVal(img, 3, 3)
    kps = cv2.GFTTDetector_create(prm.max_corners, prm.quality_level, prm.min_distance, 3, False).detect(img, mask)
    pts = np.array([k.pt for k in kps], np.float32).reshape(-1, 2)
    return img, eig, pts, np.array([k.response for k in kps], np.float32)


def opencv_float_orders_apply():
    """The device reproduces cv2's Sobel in the FMA order of OpenCV's AVX2 code path (DESIGN section 4); a cv2 that runs
    another path (no AVX2 / FMA3, optimisations off, another architecture) rounds differently and is no reference."""
    import cv2
    CV_CPU_AVX2, CV_CPU_FMA3 = 11, 12                           # opencv2/core/cvdef.h (not exported to Python)
    return bool(cv2.useOptimized() and cv2.checkHardwareSupport(CV_CPU_AVX2) and cv2.checkHardwareSupport(CV_CPU_FMA3)
                and "AVX2" in [t.lstrip("*") for t in cv2.getCPUFeaturesLine().split()])


def sobel_simd_end(W):
    """the first column of the Sobel y-derivative row pass that takes OpenCV's scalar tail: (W / 32) * 32"""
    return (W//32)*32


def min_eigen_image(img, simd_end=sobel_simd_end):
    """cv2.cornerMinEigenVal(img, 3, 3) in the float order DESIGN section 4 and the head of frontend.cu's detection section state,
    with numpy's correctly rounded float32 / float64 operations (fma(a, b, c) as one rounding of the exact a * b + c, which float64
    holds exactly for these operands).  simd_end(W) is the column where the y derivative's row pass leaves the FMA chain."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape
    f32, f64 = np.float32, np.float64
    s = 1.0/(4*3*255.0)
    f1, f0 = f32(s), f32(2*s)

    def r101(i, n):
        i = np.abs(i)
        return np.where(i >= n, 2*n - 2 - i, i)

    def fma(a, b, c):
        return (f64(a)*f64(b) + f64(c)).astype(f32)

    I = img.astype(f32)
    x = np.arange(W); xm, xp = r101(x - 1, W), r101(x + 1, W)
    y = np.arange(H); ym, yp = r101(y - 1, H), r101(y + 1, H)
    rd = I[:, xp] - I[:, xm]                                    # exact row differences
    dx = fma(rd[ym] + rd[yp], f1, rd*f0)
    L, M, R = I[:, xm], I, I[:, xp]
    simd = (x < simd_end(W))[None, :]
    rs = np.where(simd, fma(R, f1, fma(M, f0, L*f1)), (f1*L + f0*M) + f1*R)
    dy = rs[yp] - rs[ym]
    box = []
    for U, V in ((dx, dx), (dx, dy), (dy, dy)):
        P = (U*V).astype(f64)
        rows = (P[:, xm] + P) + P[:, xp]                        # (c[-1] + c[0]) + c[+1] in double
        rowat = lambda k: rows[r101(np.array(k), H)]
        out = np.empty((H, W), f32)
        rm, r0, rp = rowat(-1), rowat(0), rowat(1)
        S = (0.0 + rm) + r0
        for k in range(H):                                      # the running column sum: add the entering row, drop the leaving one
            s0 = S + rp
            out[k] = s0.astype(f32); S = s0 - rm
            rm, r0 = r0, rp
            rp = rowat(k + 2) if k + 2 <= H else np.zeros(W)
        box.append(out)
    a, b, c = box[0]*f32(0.5), box[1], box[2]*f32(0.5)
    return (a + c) - np.sqrt((a - c)*(a - c) + b*b)


def processed(gray, use_clahe=True):
    """the image detection works on: CLAHE(2.0, 8x8) or the plain frame"""
    import cv2
    return cv2.createCLAHE(2.0, (8, 8)).apply(gray) if use_clahe else gray


def assert_keypoints(got, ref, proc, starts):
    """Bit-exact, except for points whose cornerSubPix sampling window left the image during the iterations: there cv2's
    getRectSubPix takes its clamped-rectangle path, whose float sums the device reproduces up to the last bit of some patch
    entries, and a position may differ by at most 1e-4 px.  For every such point the iteration is replayed from its start
    corner with cv2's own patches (subpix_window_clamped), which must show that a window really was clamped.  Returns the
    number of such points."""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    diff = np.flatnonzero(np.any(got != ref, axis=1))
    for i in diff:
        assert np.abs(got[i] - ref[i]).max() <= 1e-4, (i, got[i], ref[i])
        clamped, end = subpix_window_clamped(proc, starts[i])
        assert clamped, (i, starts[i], ref[i])
        assert np.abs(np.array(end) - ref[i]).max() <= 1e-3, (i, end, ref[i])       # the replay follows cv2.cornerSubPix
    return len(diff)


def subpix_window_clamped(img, start, win=5, max_iter=40, eps=0.001, margin=1e-3):
    """Replays cv2.cornerSubPix from `start` with cv2.getRectSubPix patches and tells whether any visited (win+1)*2+1
    sampling window left the image, i.e. took getRectSubPix's clamped-rectangle path (within `margin` px of doing so counts,
    as the replay's sums are not in OpenCV's order).  Also returns the replayed end point."""
    import cv2
    rows, cols = img.shape
    P = 2*win + 3
    k = (np.arange(2*win + 1, dtype=np.float32) - win)/np.float32(win)
    g = np.exp(-k*k).astype(np.float32)
    mask = (g[:, None]*g[None, :]).astype(np.float64)
    px = np.arange(-win, win + 1, dtype=np.float64)[None, :]; py = px.T
    cx, cy = np.float32(start[0]), np.float32(start[1]); sx, sy = cx, cy
    clamped = False
    for _ in range(max_iter):
        ox, oy = float(cx) - (P - 1)*0.5, float(cy) - (P - 1)*0.5
        for dx in (-margin, 0.0, margin):
            for dy in (-margin, 0.0, margin):
                clamped = clamped or not (0 <= np.floor(ox + dx) < cols - P and 0 <= np.floor(oy + dy) < rows - P)
        sp = cv2.getRectSubPix(img, (P, P), (float(cx), float(cy)), patchType=cv2.CV_32F)
        gx = (sp[1:-1, 2:] - sp[1:-1, :-2]).astype(np.float64); gy = (sp[2:, 1:-1] - sp[:-2, 1:-1]).astype(np.float64)
        gxx, gxy, gyy = gx*gx*mask, gx*gy*mask, gy*gy*mask
        a, b, c = gxx.sum(), gxy.sum(), gyy.sum()
        bb1 = (gxx*px + gxy*py).sum(); bb2 = (gxy*px + gyy*py).sum()
        det = a*c - b*b
        if abs(det) <= np.finfo(np.float64).eps**2:
            break
        nx = np.float32(float(cx) + c/det*bb1 - b/det*bb2); ny = np.float32(float(cy) - b/det*bb1 + a/det*bb2)
        err = float((nx - cx)*(nx - cx) + (ny - cy)*(ny - cy)); cx, cy = nx, ny
        if cx < 0 or cx >= cols or cy < 0 or cy >= rows or err <= eps*eps:
            break
    if abs(cx - sx) > win or abs(cy - sy) > win:
        cx, cy = sx, sy
    return clamped, (float(cx), float(cy))


def detect(gray, motion_mask, boundary_mask, cur_kp, prm: Params, next_tracklet_id):
    """Returns (keypoints [n][2] float64, tracklet ids, next_tracklet_id, n_corners, starts [n][2]): starts are the integer
    corners the key-points were refined from."""
    import cv2
    rows, cols = motion_mask.shape
    mask = detection_mask(motion_mask, boundary_mask, cur_kp, prm.min_distance)
    img, _, pts, resp = stages(gray, mask, prm)
    n_cur = len(np.asarray(cur_kp).reshape(-1, 2))
    if prm.use_anms:
        assert (resp < 1.0).all()                               # suppressNonMax's int keys are all 0
        k = max(prm.max_features - n_cur, 0)
        sel = SO.anms_range_tree([(int(x), int(y)) for x, y in pts], k, np.float32(0.1), cols, rows) if len(pts) else []
        pts = pts[sel].reshape(-1, 2)
    starts = pts.copy()
    if prm.use_subpix and len(pts):
        pts = cv2.cornerSubPix(img, np.ascontiguousarray(pts.reshape(-1, 1, 2)), (5, 5), (-1, -1),
                               (cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_COUNT, 40, 0.001)).reshape(-1, 2)
    out, tid, st = [], [], []
    for (x, y), s0 in zip(pts, starts):
        kx, ky = float(x), float(y)
        u, v = int(kx), int(ky)
        if not (0.0 <= kx < cols and 0.0 <= ky < rows):                           # isKeypointContained
            continue
        if not (prm.shrink_row < v < rows - prm.shrink_row and prm.shrink_col < u < cols - prm.shrink_col):   # isWithinShrunkenImage
            continue
        if motion_mask[v, u] != 0:
            continue
        out.append((kx, ky)); tid.append(next_tracklet_id); next_tracklet_id += 1; st.append(s0)
    return np.array(out, np.float64).reshape(-1, 2), np.array(tid, np.int64), next_tracklet_id, len(resp), np.array(st, np.float64).reshape(-1, 2)
