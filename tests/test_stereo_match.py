"""stereoTrack's restatement (tests/stereo_oracle.py) on the CPU: with cv2.findFundamentalMat it equals the one with
fundamental_oracle on C4 stereo frames, its per-feature loop equals an independent numpy statement, the synthetic right view
has the disparities its depth says, and hand-built LK results reach every state, both early returns, the LMedS path and a
failed RANSAC (where cv2 leaves the mask unwritten)."""
import numpy as np
import pytest

import fundamental_oracle as FO
import stereo_oracle as SO
from dynosam_b200.synth_frames import SyntheticStream

cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("k", [0, 7])
def test_cv2_fundamental_equals_oracle_on_c4(k):
    left, right, _, pts = SO.c4_stereo_frame(SyntheticStream(n_objects=10, seed=42), k)
    a = SO.stereo_match(left, right, pts, SO.FX, SO.BASELINE, which="oracle")
    b = SO.stereo_match(left, right, pts, SO.FX, SO.BASELINE, lk=(a["right_pts"], a["lk_status"]), which="cv2")
    assert a["matched"] and b["F"] is not None and a["fund_status"] == FO.OK
    assert np.array_equal(a["mask"], b["mask"])
    assert np.array_equal(a["state"], b["state"])
    assert np.array_equal(a["depth"], b["depth"], equal_nan=True) and np.array_equal(a["right_u"], b["right_u"], equal_nan=True)
    counts = np.bincount(a["state"], minlength=5)
    assert counts[SO.MATCHED] > 500 and counts[SO.EPIPOLAR] > 0, counts


def test_loop_equals_vectorised_statement():
    rng = np.random.default_rng(3)
    for trial in range(30):
        n = int(rng.integers(8, 400))
        left = np.stack([rng.uniform(0, 1242, n), rng.uniform(0, 375, n)], 1).astype(np.float32)
        disp = rng.choice([rng.uniform(-3, 40), 1.0, 0.5], n)
        right = np.stack([left[:, 0] - disp, left[:, 1]], 1).astype(np.float32)
        right[rng.random(n) < 0.05, 0] = -rng.uniform(0, 5)                  # uR < 0
        st = (rng.random(n) < 0.9).astype(np.uint8)
        mask = (rng.random(int(st.sum())) < 0.8).astype(np.uint8)
        s1, d1, u1 = SO.per_feature(left, right, st, mask, SO.FX, SO.BASELINE)
        s2, d2, u2 = SO.per_feature_vectorised(left, right, st, mask, SO.FX, SO.BASELINE)
        assert np.array_equal(s1, s2) and np.array_equal(d1, d2, equal_nan=True) and np.array_equal(u1, u2, equal_nan=True), trial
        assert set(np.unique(s1)) <= {SO.MATCHED, SO.LOST, SO.EPIPOLAR, SO.DISPARITY}


def test_synthetic_right_view_has_the_depth_disparities():
    from scipy.ndimage import maximum_filter, minimum_filter
    s = SyntheticStream(n_objects=10, seed=42)
    g0, _, _ = s.frame(3); d0 = s.depth(3)
    for k in (3, 11):
        left, right, mask, pts = SO.c4_stereo_frame(s, k)
        d = s.depth(k)
        good = np.isfinite(d) & (d > 0)
        disp = np.where(good, SO.FX*SO.BASELINE/np.where(good, d, 1.0), 0.0)
        rp, st, _, _ = __import__("oracle.frontend_oracle", fromlist=["x"]).stereo_track(left, right, pts, SO.FX, SO.BASELINE)
        x = pts[:, 0].astype(int); y = pts[:, 1].astype(int)
        # textured background away from object borders (no object within 65 px along the row, 15 rows across, whose right view
        # could cover or uncover the window) where the 21x21 window sees one disparity to within 2 px (LK fits one shift)
        far = ~maximum_filter(mask > 0, size=(31, 131))
        flat = (maximum_filter(disp, size=21) - minimum_filter(disp, size=21)) < 2.0
        sel = (st == 1) & far[y, x] & flat[y, x] & (pts[:, 0] > 60)
        err = np.abs((pts[:, 0] - rp[:, 0]) - disp[y, x])
        assert sel.sum() > 200 and (err[sel] < 0.25).mean() >= 0.9, (k, sel.sum(), (err[sel] < 0.25).mean())
    # the left view and the depth are those of frame() and depth()
    assert np.array_equal(s.frame(3)[0], g0) and np.array_equal(s.depth(3), d0, equal_nan=True)
    assert np.array_equal(s.right(3), s.right(3))


def _shifted(n, disp, rng, row=None):
    left = np.stack([rng.uniform(50, 1200, n), np.full(n, float(row)) if row is not None else rng.uniform(10, 360, n)], 1).astype(np.float32)
    right = left.copy(); right[:, 0] -= np.float32(disp)
    if row is None:
        right += rng.normal(0, 0.05, right.shape).astype(np.float32)
    return left, right


def test_hand_built_states_and_paths():
    rng = np.random.default_rng(11)
    # n = 7: nothing runs
    l7, r7 = _shifted(7, 9.0, rng)
    o = SO.stereo_match(None, None, l7, SO.FX, SO.BASELINE, lk=(r7, np.ones(7, np.uint8)))
    assert not o["matched"] and (o["state"] == SO.UNTOUCHED).all() and np.isnan(o["depth"]).all() and o["fund_status"] == -1
    # 8 inputs, 7 tracked: the second early return
    l8, r8 = _shifted(8, 9.0, rng)
    st = np.ones(8, np.uint8); st[3] = 0
    o = SO.stereo_match(None, None, l8, SO.FX, SO.BASELINE, lk=(r8, st))
    assert not o["matched"] and (o["state"] == SO.UNTOUCHED).all() and o["n_tracked"] == 7
    # 8-14 tracked: LMedS, with a lost point, an epipolar outlier and a disparity reject
    l12, r12 = _shifted(12, 9.0, rng)
    r12[0, 1] += 25.0                                                      # off its epipolar line
    r12[1, 0] = l12[1, 0] - np.float32(0.5)                                # disparity 0.5 <= 1
    st = np.ones(12, np.uint8); st[2] = 0
    o = SO.stereo_match(None, None, l12, SO.FX, SO.BASELINE, lk=(r12, st))
    c = SO.stereo_match(None, None, l12, SO.FX, SO.BASELINE, lk=(r12, st), which="cv2")
    assert o["matched"] and o["fund_status"] == FO.LMEDS and np.array_equal(o["state"], c["state"])
    assert o["state"][0] == SO.EPIPOLAR and o["state"][1] == SO.DISPARITY and o["state"][2] == SO.LOST
    ok = o["state"] == SO.MATCHED                                           # (LMedS's sigma is tight: noise makes a few more outliers)
    assert ok.sum() >= 5 and np.allclose(o["depth"][ok], SO.FX*SO.BASELINE/9.0, rtol=0.05) and np.isnan(o["depth"][~ok]).all()
    # a failed RANSAC: 20 points on one row under a pure horizontal shift, every subset collinear -> every tracked point EPIPOLAR
    lf, rf = _shifted(20, 9.0, rng, row=100.0)
    st = np.ones(20, np.uint8); st[5] = 0
    o = SO.stereo_match(None, None, lf, SO.FX, SO.BASELINE, lk=(rf, st))
    c = SO.stereo_match(None, None, lf, SO.FX, SO.BASELINE, lk=(rf, st), which="cv2")
    assert o["matched"] and o["fund_status"] == FO.FAILED and o["F"] is None and c["F"] is None
    want = np.full(20, SO.EPIPOLAR, np.uint8); want[5] = SO.LOST
    assert np.array_equal(o["state"], want) and np.array_equal(c["state"], want) and o["n_stereo"] == 0


def test_cv2_leaves_a_failed_mask_unwritten():
    """what the reference's std::vector mask holds after a failed findFundamentalMat: cv2 does not write a mask it is handed,
    so the vector keeps the m zeros it was resized to"""
    lf, rf = _shifted(20, 9.0, np.random.default_rng(2), row=100.0)
    for fill in (0, 7):
        mask = np.full((20, 1), fill, np.uint8)
        F, mk = cv2.findFundamentalMat(lf, rf, cv2.FM_RANSAC, 1.0, 0.99, 1000, mask=mask)
        assert F is None and (mask == fill).all()
    # and with a model, the handed-in mask is the one written
    a, b = FO.make_problem(5, 200, 0.2, "stereo")
    mask = np.full((200, 1), 7, np.uint8)
    F, mk = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, 1.0, 0.99, 1000, mask=mask)
    assert F is not None and set(np.unique(mask)) <= {0, 1} and np.array_equal(mask.ravel(), FO.find_fundamental(a, b).mask)
