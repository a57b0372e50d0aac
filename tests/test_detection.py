"""Static feature detection on the device (KltFeatureTracker::detectFeatures), CPU side.

The oracle's pieces are pinned against independent code: its mask against a brute-force disc test built from the midpoint
rasteriser of make_disc (frontend.cu), its GFTT order against a numpy sort by (value desc, address desc) on an image with
tied eigenvalues, and the int-truncated ANMS keys are all 0 on C4 frames.  That the kernels build for sm_90a without spills
is checked for the whole library in tests/test_frontend.py.
GPU (tests/test_detection_gpu.py): every stage and the end-to-end result against the oracle.
"""
import os

import numpy as np
import pytest

import detection_oracle as DO
from dynosam_b200.synth_frames import SyntheticStream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _disc_half_widths(r):
    """make_disc: OpenCV's filled-circle spans (midpoint algorithm) as a half width per |dy|"""
    hw = [-1]*16
    err, dx, dy, plus, minus = 0, r, 0, 1, (r << 1) - 1
    while dx >= dy:
        hw[dy] = max(hw[dy], dx); hw[dx] = max(hw[dx], dy)
        dy += 1; err += plus; plus += 2
        m = -1 if err > 0 else 0
        err -= minus & m; dx += m; minus -= m & 2
    return hw


@pytest.mark.parametrize("radius", [8, 15])
def test_oracle_mask_matches_disc_rasteriser(radius):
    rng = np.random.default_rng(radius)
    H, W = 120, 200
    motion = np.zeros((H, W), np.int32); motion[40:60, 50:90] = 3
    boundary = np.full((H, W), 255, np.uint8); boundary[:, :7] = 0
    kp = np.concatenate([rng.uniform(-5, W + 5, (40, 2)) * [1, H/W],
                         [[10.5, 20.5], [11.5, 30.5], [-0.5, 2.5], [100.5, 119.5], [50.49999, 60.50001]]])
    got = DO.detection_mask(motion, boundary, kp, radius)
    hw = _disc_half_widths(radius)
    want = np.where((motion == 0) & (boundary != 0), 255, 0).astype(np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    for x, y in kp:
        cx, cy = int(np.rint(np.float32(x))), int(np.rint(np.float32(y)))        # round half to even
        ady = np.abs(yy - cy); adx = np.abs(xx - cx)
        cover = (ady <= radius) & (adx <= np.array(hw + [-1])[np.minimum(ady, 16)])
        want[cover] = 0
    assert np.array_equal(got, want)
    assert int(np.rint(np.float32(10.5))) == 10 and int(np.rint(np.float32(11.5))) == 12


def test_gftt_order_is_value_then_address_descending():
    """cv2.GFTTDetector's output order equals a numpy sort by (value desc, address desc) followed by the greedy strict
    minDistance filter, on an image built so that many eigenvalues tie (a periodic texture)."""
    import cv2
    rng = np.random.default_rng(5)
    tile = cv2.GaussianBlur(rng.integers(0, 256, (16, 16)).astype(np.uint8), (0, 0), 1.0)
    img = np.ascontiguousarray(np.tile(tile, (10, 14)))[:150, :221]
    H, W = img.shape
    mask = np.full((H, W), 255, np.uint8); mask[60:90, 100:140] = 0
    for md, mc in ((0, 5000), (5, 300), (9, 40)):
        eig = cv2.cornerMinEigenVal(img, 3, 3)
        thr = np.float32(np.float64(eig[mask > 0].max())*0.001)
        e = np.where(eig > thr, eig, np.float32(0))
        pad = np.pad(e, 1, constant_values=-np.inf)
        dil = np.max([pad[j:j + H, i:i + W] for j in range(3) for i in range(3)], axis=0)
        cand = (e != 0) & (e == dil) & (mask > 0)
        cand[0] = cand[-1] = False; cand[:, 0] = cand[:, -1] = False
        ys, xs = np.nonzero(cand); v = e[ys, xs]; addr = ys*W + xs
        o = np.lexsort((-addr, -v)); ys, xs, v = ys[o], xs[o], v[o]
        assert (np.diff(v) == 0).sum() > 50                      # plenty of ties
        kept = []
        for x, y in zip(xs.tolist(), ys.tolist()):
            if all((x - a)**2 + (y - b)**2 >= md*md for a, b in kept):
                kept.append((x, y))
                if len(kept) == mc:
                    break
        ref = [(int(k.pt[0]), int(k.pt[1])) for k in cv2.GFTTDetector_create(mc, 0.001, md, 3, False).detect(img, mask)]
        assert ref == kept, md


def test_gftt_responses_below_one_on_c4():
    for k in (1, 3, 7):
        g, m, _ = SyntheticStream(n_objects=10, seed=42).frame(k)
        mask = DO.detection_mask(m, None, np.zeros((0, 2)), 15)
        _, eig, pts, resp = DO.stages(np.ascontiguousarray(g.astype(np.uint8)), mask, DO.Params())
        assert len(resp) == 1000 and resp.max() < 1.0 and eig.max() < 1.0
        assert (resp.astype(np.int32) == 0).all()
        assert np.array_equal(pts, np.round(pts))                # the corners are whole pixels


def test_detection_exports():
    import __graft_entry__ as g
    if not os.path.exists(os.path.join(ROOT, "dynosam_b200", "libdynofront.so")):
        g.build()
    from dynosam_b200 import frontend
    lib = frontend.load()
    for s in ("dynofront_detect_static", "dynofront_detect_last_stages"):
        assert s in frontend.EXPORTS and hasattr(lib, s), s
