"""tests/homography_oracle.py pinned against cv2: OpenCV's Jacobi bit for bit, the 4-point DLT bit for bit, the refinement to a
stated tolerance and cv::findHomography(RANSAC)'s returned masks on the parity set.  No GPU."""
import numpy as np
import pytest

import homography_oracle as HO

cv2 = pytest.importorskip("cv2")


PINNED = (4, 13)


def _pinned_opencv():
    """the cv2 release the restatement was pinned against (4.13): the returned-mask recomputation and the LM control are what
    that release was observed to do; other releases may differ (the mask recomputation is believed to date from 4.6, which has
    not been checked)"""
    return tuple(int(x) for x in cv2.__version__.split(".")[:2]) == PINNED


def ransac_stage_equals_cv2(a, b, R, Hc):
    """cv2.findHomography(src, dst, 0) on exactly the restatement's RANSAC inliers runs runKernel and OpenCV's own 10-step LM on
    them, which is what cv2's RANSAC path does after its RANSAC.  Returns True when that H equals cv2's RANSAC result bit for
    bit, i.e. cv2's RANSAC chose the same inlier set; None when the check does not apply (4 inliers: cv2 skips the LM for a
    4-point method-0 call)."""
    sel = R.ransac_mask.astype(bool)
    if sel.sum() <= 4:
        return None
    H0, _ = cv2.findHomography(a[sel], b[sel], 0)
    return H0 is not None and np.array_equal(H0, Hc)


def _ltl_matrices():
    out = []
    for name, a, b, mi in HO.parity_set("small")[:40]:
        if len(a) >= 4:
            L, *_ = HO.ltl(a[None], b[None]); out.append(L[0])
    return out


def test_jacobi_equals_cv2_eigen_bit_for_bit():
    rng = np.random.default_rng(0)
    mats = _ltl_matrices()
    for s in range(120):
        A = rng.normal(size=(9, 9)); A = A + A.T
        if s % 3 == 0:                                   # zero entries
            A[rng.random((9, 9)) < .4] = 0; A = np.triu(A) + np.triu(A, 1).T
        if s % 4 == 0:                                   # tied entries
            A = np.round(A)
        mats.append(A)
    mats.append(np.eye(9)); mats.append(np.ones((9, 9))); mats.append(np.zeros((9, 9)))
    W, V = HO.jacobi(np.array(mats))
    for i, A in enumerate(mats):
        _, w, v = cv2.eigen(A)
        assert np.array_equal(w.ravel(), W[i]) and np.array_equal(v, V[i]), i


def test_four_point_dlt_equals_cv2_bit_for_bit():
    """cv2.findHomography on exactly 4 points returns runKernel's H: normalisation, LtL, Jacobi, the 3x3 products, 1 / H22"""
    rng = np.random.default_rng(1)
    a = (rng.random((240, 4, 2))*[1242, 375]).astype(np.float32)
    b = (a + rng.normal(0, 20, a.shape)).astype(np.float32)
    H, ok, _ = HO.run_kernel(a, b)
    n = 0
    for i in range(len(a)):
        Hc, mk = cv2.findHomography(a[i], b[i], cv2.RANSAC, 5.0)
        assert (Hc is not None) == ok[i]
        if Hc is not None:
            assert np.array_equal(H[i], Hc), i; n += 1
            assert mk.all()
    assert n >= 200


def test_refinement_matches_cv2_method_0():
    """cv2.findHomography(src, dst, 0): the DLT over all points, then the 10-step LM.  OpenCV's LM solve is not restated bit for
    bit (the restatement sums and solves the normal equations as the kernel does), so H agrees to 1e-6 relative (1e-7 reached):
    the refined H lies on a flat minimum where solvers that converge stop at slightly different points."""
    rng = np.random.default_rng(2)
    worst = 0.0
    for s in range(40):
        n = int(rng.integers(5, 400))
        a = (rng.random((n, 2))*[1242, 375]).astype(np.float32); b = (a*1.01 + 3 + rng.normal(0, 1, a.shape)).astype(np.float32)
        Hc, _ = cv2.findHomography(a, b, 0)
        H, ok, _ = HO.run_kernel(a[None], b[None])
        Hr, _, _ = HO.refine(H[0], a, b)
        worst = max(worst, np.abs(Hr - Hc).max()/np.abs(Hc).max())
    assert worst <= 1e-6, worst


def test_block_sum_and_solve_restate_the_kernel_order():
    """the LM's reduction: strided per-thread sums, xor butterflies, warps in order -- against a literal scalar loop"""
    rng = np.random.default_rng(3)
    c = rng.normal(size=(1000, 2, 3))*10.0**rng.integers(-8, 8, (1000, 2, 3))
    acc = [[0.0]*3 for _ in range(256)]
    for i in range(1000):
        for row in range(2):
            for e in range(3):
                acc[i % 256][e] += float(c[i, row, e])
    warps = []
    for w in range(8):
        lanes = [list(acc[32*w + l]) for l in range(32)]
        for o in (16, 8, 4, 2, 1):
            lanes = [[lanes[l][e] + lanes[l ^ o][e] for e in range(3)] for l in range(32)]
        warps.append(lanes[0])
    want = [sum_w for sum_w in warps[0]]
    for w in range(1, 8):
        want = [want[e] + warps[w][e] for e in range(3)]
    assert np.array_equal(HO.block_sum(c), np.array(want))
    A = rng.normal(size=(8, 8)); A = A @ A.T + 8*np.eye(8); v = rng.normal(size=8)
    d = HO._cholesky_solve(A, v, 1e-3)
    Ap = A.copy(); Ap[np.diag_indices(8)] *= 1 + 1e-3
    assert np.allclose(Ap @ d, v, rtol=0, atol=1e-12)


def test_draw_stream_is_opencv_rng():
    """cv::RNG((uint64)-1): the first outputs of the multiply-with-carry generator against pure-Python integers, and the
    duplicate re-draw"""
    r = HO.RNG(); s = (1 << 64) - 1; ref = []
    for _ in range(20):
        s = ((s & 0xFFFFFFFF)*4164903690 + (s >> 32)) & ((1 << 64) - 1); ref.append(s & 0xFFFFFFFF)
    assert [r.next() for _ in range(20)] == ref
    g = HO.draw_groups(HO.RNG(), 5, 200)
    assert all(len(set(x)) == 4 for x in g.tolist())


@pytest.mark.skipif(not _pinned_opencv(), reason=f"restatement pinned against OpenCV {PINNED}")
def test_masks_equal_cv2_on_parity_set():
    """The returned masks equal cv2's on >= 200 problems (n 5 to 20 000, 0-70 % outliers, maxIters 1, 2, 3, 5, 2000, collinear,
    duplicated and identical points).  On every problem with more than 4 RANSAC inliers, cv2's RANSAC chose exactly the
    restatement's inlier set: cv2's own method-0 fit of those inliers reproduces cv2's H bit for bit.  Where the returned masks
    still differ, that proves the difference is the refinement alone -- OpenCV's 8x8 LM solve, which is not restated, and ten
    steps from a poor model (small maxIters) that end mid-descent -- and cv2's mask is err(H_cv2) <= thr^2 under the
    restatement's error function.  Those problems are named in homography_oracle.CV2_LM_DIFFERENCES."""
    probs = HO.parity_set("full")
    assert len(probs) >= 200
    differ = []; rejected = failed = pinned = 0
    for name, a, b, mi in probs:
        Hc, mk = cv2.findHomography(a, b, cv2.RANSAC, 5.0, maxIters=mi)
        R = HO.find_homography(a, b, max_iters=mi)
        rejected += R.rejected > 0; failed += R.status == HO.RANSAC_FAILED
        mk = np.zeros(len(a), np.uint8) if mk is None else mk.ravel()
        assert (Hc is None) == (R.status == HO.RANSAC_FAILED), name
        if R.status == HO.OK:
            same = ransac_stage_equals_cv2(a, b, R, Hc)
            assert same is not False, name
            pinned += same is True
        if np.array_equal(R.mask, mk):
            continue
        differ.append(name)
        assert R.status == HO.OK and mi <= 5 and ransac_stage_equals_cv2(a, b, R, Hc), name
        assert np.array_equal((HO.errors(Hc, a, b) <= np.float32(25.0)).astype(np.uint8), mk), name
    assert rejected >= 5 and failed >= 1 and pinned >= 150, (rejected, failed, pinned)
    print("masks that differ through the LM alone:", differ)
    assert set(differ) <= set(HO.CV2_LM_DIFFERENCES), differ
