"""Feature selection on the device (SURVEY.md section 8f row 4, sampling half): range-tree ANMS and sampleDynamic.

CPU: the oracle's visiting order equals cv2.sortIdx on all-equal keys, and its range-tree ANMS equals a second
implementation that shares no code with it (cv2.sortIdx for the order, a scipy cKDTree Chebyshev ball query for the
square search, Decimal rounding for the bounds).  That the kernels build for sm_90a without spills is checked for the whole
library in tests/test_frontend.py.
GPU (tests/test_selection_gpu.py): the batched kernel and sample_dynamic bit-exact against the oracle.
"""
import os
from decimal import ROUND_HALF_UP, Decimal

import numpy as np

import selection_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 1242, 375


def test_sort_idx_equal_keys_matches_cv2():
    import cv2
    for n in list(range(1, 3001)) + [10000, 54321]:
        ref = cv2.sortIdx(np.zeros((1, n), np.int32), cv2.SORT_EVERY_ROW | cv2.SORT_DESCENDING).ravel().tolist()
        assert SO.sort_idx_equal_keys(n) == ref, n
    assert SO.sort_idx_equal_keys(20) == list(range(1, 10)) + [0] + list(range(11, 20)) + [10]


def _half_up(v):
    return int(Decimal(v).quantize(Decimal(1), rounding=ROUND_HALF_UP))


def _kdtree_anms(xy, k, tol, cols, rows):
    """Second implementation: same specification, no shared code with the oracle."""
    import cv2
    from scipy.spatial import cKDTree
    n = len(xy)
    if n == 0 or k == 0:
        return []
    order = cv2.sortIdx(np.zeros((1, n), np.int32), cv2.SORT_EVERY_ROW | cv2.SORT_DESCENDING).ravel()
    if k == 1:
        return [int(order[0])]
    pts = np.asarray(xy, np.float64)[order]
    tree = cKDTree(pts)
    disc = np.sqrt(np.float64(4*cols + 4*k + 4*rows*k + rows**2 + cols**2 - 2*rows*cols + 4*rows*cols*k))
    s = np.float64(rows + cols + 2*k)
    roots = [-_half_up(float((s + disc)/np.float64(k - 1))), -_half_up(float((s - disc)/np.float64(k - 1)))]
    hi = max(roots); lo = int(np.floor(np.sqrt(np.float64(n)/np.float64(k))))
    kf, tf = np.float32(k), np.float32(tol)
    kmin, kmax = _half_up(float(kf - kf*tf)), _half_up(float(kf + kf*tf))
    last, prev = [], None
    while lo <= hi:
        w = lo + int((hi - lo)/2)
        if w == prev:
            break
        nb = tree.query_ball_point(pts, r=w, p=np.inf)
        gone = np.zeros(n, bool); keep = []
        for i in range(n):
            if not gone[i]:
                keep.append(i); gone[nb[i]] = True
        last = keep
        if kmin <= len(keep) <= kmax:
            break
        if len(keep) < kmin:
            hi = w - 1
        else:
            lo = w + 1
        prev = w
    return [int(order[i]) for i in last]


def _anms_cases():
    rng = np.random.default_rng(12)
    cases = []
    for n in (300, 2000):                                             # random sets over the image
        flat = rng.choice(W*H, n, replace=False)
        cases += [(np.stack([flat % W, flat//W], 1), k, tol) for k in (5, 200) for tol in (0.01, 0.1)]
    yy, xx = np.mgrid[100:160, 400:470]                               # a dense object region: every pixel a candidate
    blob = np.stack([xx.ravel(), yy.ravel()], 1)
    cases += [(blob, k, 0.01) for k in (2, 37, 200)]
    small = np.stack([rng.integers(0, W, 50), rng.integers(0, H, 50)], 1)   # n < Kmin: the fall-back result
    cases += [(small, 200, 0.01), (small, 0, 0.01), (small, 1, 0.01), (small, 2, 0.1)]
    cases += [(np.zeros((0, 2), np.int64), 200, 0.01), (blob[:17], 5, 0.01)]
    return cases


def test_anms_oracle_matches_independent_kdtree():
    for xy, k, tol in _anms_cases():
        a = SO.anms_range_tree(xy, k, np.float32(tol), W, H)
        b = _kdtree_anms(xy, k, tol, W, H)
        assert a == b, (len(xy), k, tol)
    blob = _anms_cases()[8][0]
    assert len(SO.anms_range_tree(np.asarray(blob)[:50], 200, np.float32(0.01), W, H)) == 50   # fall-back keeps every point


def test_anms_oracle_semantics():
    """The visiting order is P_n, not the input order, and the square is inclusive."""
    xy = np.array([[10, 10], [12, 10], [20, 10]])       # P_3 = [2, 1, 0]
    assert SO.sort_idx_equal_keys(3) == [2, 1, 0]
    assert SO.anms_range_tree(xy, 1, np.float32(0.01), W, H) == [2]
    assert SO.anms_range_tree(xy, 0, np.float32(0.01), W, H) == []


def test_selection_exports():
    import __graft_entry__ as g
    if not os.path.exists(os.path.join(ROOT, "dynosam_b200", "libdynofront.so")):
        g.build()
    from dynosam_b200 import frontend
    lib = frontend.load()
    for s in ("dynofront_anms_range_tree", "dynofront_sample_dynamic"):
        assert s in frontend.EXPORTS and hasattr(lib, s), s
