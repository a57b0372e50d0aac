"""Static feature detection on the device against the CPU oracle (tests/detection_oracle.py).

Stage by stage through dynofront_detect_last_stages (CLAHE image, minimum-eigenvalue image, GFTT corners in order) on C4
frames and on a random texture whose size is not a multiple of 8; then the end-to-end key-points, tracklet ids,
next_tracklet_id and corner count for the first frame, ~300 and >= 800 current features, boundary mask, shrink margins,
each stage switched off once and both radii; streaming against call by call; the boundary mask after track_dynamic;
capacity; refusals.
"""
import ctypes as C

import numpy as np
import pytest

import detection_oracle as DO
from frame_cases import c4, cur_features, dev_params, texture

W, H = 1242, 375


needs_opencv_orders = pytest.mark.skipif(not DO.opencv_float_orders_apply(),
                                         reason="cv2 does not run OpenCV's AVX2 + FMA3 code path, whose float orders the device reproduces")


@pytest.mark.gpu
@needs_opencv_orders
@pytest.mark.parametrize("which", ["c4", "texture"])
def test_stages_bit_exact(which):
    import cv2
    from dynosam_b200.frontend import FeatureTrackerGPU
    if which == "c4":
        g, m, f = c4(3)
    else:
        g = texture(251, 333, 1); m = np.zeros(g.shape, np.int32); m[50:90, 100:160] = 2; f = np.zeros(g.shape + (2,), np.float32)
    rows, cols = g.shape
    rng = np.random.default_rng(1)
    kp = cur_features(rng, m, 150)
    t = FeatureTrackerGPU(cols, rows)
    t.set_frame(f, m, None)
    for p in (DO.Params(), DO.Params(min_distance=8, max_corners=3000)):
        t.detect_static(g, kp, dev_params(p), 0)
        cl, eig, corners = t.detect_stages()
        mask = DO.detection_mask(m, None, kp, p.min_distance)
        ref_cl, ref_eig, ref_pts, _ = DO.stages(g, mask, p)
        assert np.array_equal(cl, cv2.createCLAHE(2.0, (8, 8)).apply(g))
        assert np.array_equal(eig, ref_eig) and np.array_equal(eig, cv2.cornerMinEigenVal(ref_cl, 3, 3))
        assert corners.shape == ref_pts.shape and np.array_equal(corners, ref_pts.astype(np.int32))


@pytest.mark.gpu
@needs_opencv_orders
@pytest.mark.parametrize("case", ["first", "n300", "n800", "boundary_shrink", "no_clahe", "no_anms", "no_subpix", "r8"])
def test_detect_static_bit_exact(case):
    from dynosam_b200.frontend import FeatureTrackerGPU
    g, m, f = c4(4)
    rng = np.random.default_rng(7)
    n = {"first": 0, "n800": 820}.get(case, 300)
    kp = cur_features(rng, m, n)
    p = DO.Params()
    boundary = None
    if case == "boundary_shrink":
        boundary = np.full((H, W), 255, np.uint8); boundary[:, :200] = 0; boundary[300:, :] = 0
        p.shrink_row, p.shrink_col = 12, 20
    if case == "no_clahe": p.use_clahe = False
    if case == "no_anms": p.use_anms = False
    if case == "no_subpix": p.use_subpix = False
    if case == "r8": p.min_distance = 8
    t = FeatureTrackerGPU(W, H)
    t.set_frame(f, m, boundary)
    got, gid, gnext, gnc = t.detect_static(g, kp, dev_params(p), 5000)
    ref, rid, rnext, rnc, starts = DO.detect(g, m, boundary, kp, p, 5000)
    assert gnc == rnc
    off = DO.assert_keypoints(got, ref, DO.processed(g, p.use_clahe), starts) if p.use_subpix else DO.assert_keypoints(got, ref, None, None)
    assert np.array_equal(gid, rid) and gnext == rnext
    if case == "n800":
        assert len(got) == 0 and gnc > 0                           # K = 0: no new features
    elif case == "first":
        assert len(got) > 400
    assert t.last_ms > 0
    print(case, len(got), "features,", off, "within 1e-4 px at the border")


@pytest.mark.gpu
@needs_opencv_orders
def test_detect_streaming_equals_call_by_call():
    """gray=None after next_frame works on the resident current frame; the boundary mask is the uploaded one even after
    track_dynamic has drawn into its working copy."""
    from dynosam_b200.frontend import DetectParams, FeatureTrackerGPU, TrackParams
    rng = np.random.default_rng(11)
    frames = [c4(k, seed=9) for k in range(3)]
    boundary = np.full((H, W), 255, np.uint8); boundary[:40, :] = 0
    a = FeatureTrackerGPU(W, H); b = FeatureTrackerGPU(W, H)
    prm = DetectParams()
    a.next_frame(frames[0][0], frames[0][2], frames[0][1], boundary)
    for k in (1, 2):
        g, m, f = frames[k]
        kp = cur_features(rng, m, 250)
        a.next_frame(g, f, m, boundary)
        ys, xs = np.nonzero(m > 0); s = rng.choice(len(ys), 300, replace=False)
        dyn = np.stack([xs[s] + 0.5, ys[s] + 0.5], 1)
        a.track_dynamic(dyn, m[ys[s], xs[s]], np.zeros(300, np.int32), np.arange(300, dtype=np.int64), TrackParams(min_distance=15), 0, want_masks=False)
        ra = a.detect_static(None, kp, prm, 100)
        b.set_frame(f, m, boundary)
        rb = b.detect_static(g, kp, prm, 100)
        assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]) and ra[2:] == rb[2:]
        ref = DO.detect(g, m, boundary, kp, DO.Params(), 100)
        DO.assert_keypoints(ra[0], ref[0], DO.processed(g), ref[4])
        assert np.array_equal(ra[1], ref[1]) and ra[2] == ref[2]


def _corner_image(h, w, seed):
    """a low-contrast texture with bright squares whose corners sit 2-6 px from each image corner (and from mid-edges)"""
    import cv2
    rng = np.random.default_rng(seed)
    img = 60 + rng.integers(0, 40, (h, w)).astype(np.float32)
    for x0, y0 in ((3, 3), (w - 5, 2), (w - 6, 4), (2, h - 4), (w - 4, h - 5), (w//2, 3), (3, h//2), (w - 4, h//2), (w//3, h - 3)):
        xs = slice(x0, min(x0 + 14, w)) if x0 < w//2 or x0 == w//2 else slice(max(x0 - 14, 0), x0 + 1)
        ys = slice(y0, min(y0 + 14, h)) if y0 < h//2 or y0 == h//2 else slice(max(y0 - 14, 0), y0 + 1)
        img[ys, xs] = 230 - 20*rng.random()
    return np.ascontiguousarray(cv2.GaussianBlur(img, (0, 0), 0.8).clip(0, 255).astype(np.uint8))


@pytest.mark.gpu
@needs_opencv_orders
@pytest.mark.parametrize("use_anms", [False, True])
def test_detect_corners_at_image_corners(use_anms):
    """strong corners within 6 px of every image corner and edge reach cornerSubPix, whose window then leaves the image"""
    from dynosam_b200.frontend import FeatureTrackerGPU
    h, w = 251, 333
    g = _corner_image(h, w, 3); m = np.zeros((h, w), np.int32); f = np.zeros((h, w, 2), np.float32)
    p = DO.Params(use_anms=use_anms, min_distance=5, max_corners=3000, max_features=800)
    t = FeatureTrackerGPU(w, h); t.set_frame(f, m, None)
    got, gid, gnext, gnc = t.detect_static(g, np.zeros((0, 2)), dev_params(p), 0)
    ref, rid, rnext, rnc, starts = DO.detect(g, m, None, np.zeros((0, 2)), p, 0)
    assert gnc == rnc and np.array_equal(gid, rid) and gnext == rnext
    near = lambda q, dx, dy: ((np.abs(q[:, 0] - dx) <= 6) & (np.abs(q[:, 1] - dy) <= 6)).any()
    if not use_anms:                                             # every image corner has a refined point next to it
        for cx, cy in ((0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1)):
            assert near(starts, cx, cy), (cx, cy)
    off = DO.assert_keypoints(got, ref, DO.processed(g), starts)
    print("corners", use_anms, len(got), "features,", off, "within 1e-4 px with a clamped window")


@pytest.mark.gpu
def test_detect_capacity():
    from dynosam_b200.frontend import DetectParams, FeatureTrackerGPU, _p
    g, m, f = c4(5)
    t = FeatureTrackerGPU(W, H); t.set_frame(f, m, None)
    prm = DetectParams()
    full = t.detect_static(g, np.zeros((0, 2)), prm, 10)
    total = len(full[0]); assert total > 20
    small = t.detect_static(g, np.zeros((0, 2)), prm, 10, capacity=5)          # the wrapper's retry
    assert np.array_equal(small[0], full[0]) and np.array_equal(small[1], full[1]) and small[2] == full[2]
    cap = 7
    kp = np.full((cap + 1, 2), -7.0); tid = np.full(cap + 1, -7, np.int64)
    nid = C.c_int64(10); nf = C.c_int32(); nc = C.c_int32(); pc = prm.c(); gg = np.ascontiguousarray(g)
    t._ck(t.lib.dynofront_detect_static(t.h, _p(gg), 0, None, C.byref(pc), C.byref(nid), cap, _p(kp), _p(tid), C.byref(nf), C.byref(nc), None))
    assert nf.value == total and nid.value == 10 + total
    assert np.array_equal(kp[:cap], full[0][:cap]) and np.array_equal(tid[:cap], full[1][:cap])
    assert (kp[cap] == -7.0).all() and tid[cap] == -7                            # nothing written past capacity


@pytest.mark.gpu
def test_detect_refusals():
    from dynosam_b200.frontend import DetectParams, FeatureTrackerGPU, FrontendError
    g, m, f = c4(2)
    t = FeatureTrackerGPU(W, H); t.set_frame(f, m, None)
    for bad in (DetectParams(use_harris=True), DetectParams(block_size=5), DetectParams(min_distance=16)):
        with pytest.raises(FrontendError):
            t.detect_static(g, np.zeros((0, 2)), bad, 0)
    with pytest.raises(FrontendError):                                          # no resident frame yet
        FeatureTrackerGPU(W, H).detect_static(None, np.zeros((0, 2)), DetectParams(), 0)
