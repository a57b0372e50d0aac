"""tests/fundamental_oracle.py against cv2 4.13 (CPU): OpenCV's 7x9 Jacobi SVD with its seeded completion bit for bit, solveCubic
and the 7-point models to the last bits, and the returned masks of cv2.findFundamentalMat(FM_RANSAC) on the parity set."""
import numpy as np
import pytest

import fundamental_oracle as FO

cv2 = pytest.importorskip("cv2")
pinned = pytest.mark.skipif(tuple(int(x) for x in cv2.__version__.split(".")[:2]) != (4, 13), reason="pinned against OpenCV 4.13")


@pinned
def test_svd_vt_equals_cv2_bit_for_bit():
    r = np.random.default_rng(3)
    A = [r.normal(size=(7, 9)) for _ in range(100)]
    for s in range(100):                               # the normalised systems run7Point builds
        a, b = FO.make_problem(s, 7, 0.0, ["general", "stereo", "planar"][s % 3])
        A.append(FO.normalise(a[None], b[None])[0][0])
    A = np.array(A)
    Vt = FO.svd_vt(A)
    for a, v in zip(A, Vt):
        assert np.array_equal(v, cv2.SVDecomp(a, flags=cv2.SVD_FULL_UV)[2])


@pinned
def test_solve_cubic_equals_cv2_bit_for_bit():
    """roots, root count and root order equal cv2.solveCubic bit for bit, including the zero thresholds (max|a| < DBL_EPSILON,
    and leading coefficients below DBL_EPSILON of the largest), NaN roots and the a0 == 0 branches"""
    r = np.random.default_rng(0)
    cs = [r.normal(size=4)*10.0**r.integers(-3, 3, 4) for _ in range(2000)]
    for _ in range(3000):
        c = r.normal(size=4)*10.0**r.integers(-18, 3, 4)
        c[r.random(4) < 0.3] = 0
        cs.append(c)
    cs += [np.array([e, 1., -3., 2.]) for e in (1e-10, 1e-13, 1e-14, 1e-16, 3*FO.DBL_EPS, 1e-17)]
    cs += [np.array([1., -6., 11., -6.])*s for s in (1e-15, 1e-16, 1e-17)]
    cs += [np.array(c, float) for c in ([0, 0, 0, FO.DBL_EPS], [-6.9e-17, 9.6e-17, -1.1e-16, 0], [0, 0, 0, 0], [0, 1, 0, 0], [1e-12, 1, -2, 1])]
    for c in cs:
        n, x, _ = FO.solve_cubic(c)
        nc, xc = cv2.solveCubic(c)
        assert n == nc, c
        assert np.array_equal(np.array(x[:max(n, 0)]), xc.ravel()[:max(n, 0)], equal_nan=True), c


@pinned
def test_seven_point_models_equal_cv2_bit_for_bit():
    for s in range(300):
        a, b = FO.make_problem(s, 7, 0.0, ["general", "stereo", "planar"][s % 3])
        res = FO.find_fundamental(a, b)
        Fc, mk = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, 1.0, 0.99)
        assert res.status == FO.SEVEN_POINT
        assert (Fc is None) == (not res.F), s
        if Fc is not None:
            assert np.array_equal(np.concatenate(res.F), Fc), s
            assert np.array_equal(mk.ravel(), res.mask)


@pinned
def test_raising_configuration():
    """cv2 raises (-215, rowRange) where run7Point's cubic has every coefficient below DBL_EPSILON: solveCubic returns -1 and
    FMEstimatorCallback::runKernel takes rowRange(0, -3).  The oracle reports that draw as one without a model (-1) at the same
    place: cv2 raises on the first drawn group's 7 points alone, and the oracle's first iteration is that group."""
    a, b = FO.raising_problem()
    with pytest.raises(cv2.error, match="rowRange"):
        cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, 1.0, 0.99)
    res = FO.find_fundamental(a, b)
    assert res.raised == 0 and res.models[0] == -1
    rng = FO.RNG()
    while True:                                       # the first group that passes the subset test is iteration 0
        g = FO.draw_groups(rng, len(a), 1)[0]
        if not (FO.collinear(a[g][None]) | FO.collinear(b[g][None]))[0]:
            break
    with pytest.raises(cv2.error, match="rowRange"):
        cv2.findFundamentalMat(a[g], b[g], cv2.FM_RANSAC, 1.0, 0.99)
    assert FO.run7(a[g][None], b[g][None])[0][0] == -1


@pinned
def test_parity_set_equals_cv2_bit_for_bit():
    """on the full parity set F and the returned mask equal cv2's bit for bit wherever cv2 returns a model; where cv2 raises, the
    oracle has met an all-zero cubic first"""
    checked = 0
    for name, a, b, mi in FO.parity_set("full"):
        res = FO.find_fundamental(a, b, max_iters=mi)
        try:
            Fc, mk = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, 1.0, 0.99, maxIters=mi)
        except cv2.error:
            assert res.raised >= 0, name
            continue
        if Fc is None:
            assert res.status == FO.FAILED or (res.status == FO.LMEDS and not res.success), name
            continue
        assert res.F and np.array_equal(res.F[0], Fc[:3]), name
        assert np.array_equal(mk.ravel(), res.mask), name
        checked += 1
    assert checked > 150


def test_statuses_and_paths():
    a, b = FO.make_problem(1, 40, 0.2)
    assert FO.find_fundamental(a[:6], b[:6]).status == FO.TOO_FEW
    assert FO.find_fundamental(a[:7], b[:7]).status == FO.SEVEN_POINT
    assert FO.find_fundamental(a[:10], b[:10]).status == FO.LMEDS
    r = FO.find_fundamental(a, b)
    assert r.status == FO.OK and r.n_inliers >= 7 and len(r.scores) >= r.iterations
    a, b = FO.make_problem(2, 50, 0.0, "identical")
    r = FO.find_fundamental(a, b)
    assert r.status == FO.FAILED and r.iterations == 0 and not r.mask.any()
