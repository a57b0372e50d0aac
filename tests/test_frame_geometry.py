"""The frame-geometry rules of the front end's image kernels, on the CPU, at every size of tests/frame_cases.py: klt_top_level
against cv2.buildOpticalFlowPyramid, and the eigen-image float order (Sobel SIMD / tail split, sliding box sum, eigenvalue)
against cv2.cornerMinEigenVal bit for bit; the case list tells the Sobel tail rule from its neighbours and reaches every
boundary it names."""
import numpy as np
import pytest

import detection_oracle as DO
import frame_cases as FC

needs_opencv_orders = pytest.mark.skipif(not DO.opencv_float_orders_apply(),
                                         reason="cv2 does not run OpenCV's AVX2 + FMA3 code path, whose float orders the device reproduces")
NAMES = list(FC.CASES)


def _clahe_input(c: FC.Case):
    import cv2
    return cv2.createCLAHE(2.0, (8, 8)).apply(FC.frame(c, 3)[0])


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("win", [21, 31])
def test_klt_top_level_equals_opencv(name, win):
    import cv2
    c = FC.CASES[name]
    if min(c.w, c.h) < win + 1:
        pytest.skip("frame smaller than the window: refused by every LK entry point")
    img = FC.frame(c, 0)[0]
    for max_level in range(9):
        n, _ = cv2.buildOpticalFlowPyramid(img, (win, win), max_level, withDerivatives=False)
        assert FC.klt_top_level(c.w, c.h, max_level, win) == n, (max_level, n)


@needs_opencv_orders
@pytest.mark.parametrize("name", NAMES)
def test_min_eigen_image_order_equals_opencv(name):
    import cv2
    img = _clahe_input(FC.CASES[name])
    assert np.array_equal(DO.min_eigen_image(img), cv2.cornerMinEigenVal(img, 3, 3))


@needs_opencv_orders
@pytest.mark.parametrize("rule,where", [("(W-1)/32*32", "w_mult32"), ("W/16*16", "dataset")])
def test_case_list_tells_the_sobel_tail_rule_apart(rule, where):
    """the statement with a neighbouring tail rule mismatches cv2 on some case, and on the sizes predicted for it"""
    import cv2
    wrong = {"(W-1)/32*32": lambda W: ((W - 1)//32)*32, "W/16*16": lambda W: (W//16)*16}[rule]
    bad = []
    for c in FC.CASES.values():
        if wrong(c.w) == DO.sobel_simd_end(c.w):
            continue                                                 # the same split: no case can tell them apart here
        img = _clahe_input(c)
        if not np.array_equal(DO.min_eigen_image(img, wrong), cv2.cornerMinEigenVal(img, 3, 3)):
            bad.append(c.name)
    assert bad and any(where in FC.CASES[b].hits for b in bad), bad
    if rule == "(W-1)/32*32":
        assert {"tartan_aria_640x360", "camera_640x480"} <= set(bad), bad


def test_cases_reach_every_boundary():
    """every case reaches the boundaries it names, and together they reach every listed one; every case is large enough
    for the LK windows it runs and for CLAHE's reflected padding"""
    seen = set()
    for c in FC.CASES.values():
        h = FC.boundaries(c.w, c.h) | ({"dataset"} if c.dataset else set())
        assert set(c.hits) <= h, (c.name, set(c.hits) - h)
        seen |= set(c.hits)
        assert min(c.w, c.h) >= max(c.wins) + 1 and min(c.w, c.h) >= FC.CLAHE_MIN, c.name
    missing = set(FC.REQUIRED) - seen
    assert not missing, missing
    assert all(h in FC.REQUIRED for c in FC.CASES.values() for h in c.hits)
    assert {(c.w, c.h) for c in FC.CASES.values() if c.dataset} == {(1242, 375), (1238, 374), (1241, 376), (752, 480), (640, 480), (640, 360)}


def test_value_noise_shift_moves_the_surface():
    """the texture pair of the small cases: a whole-pixel shift is the same image moved, so sub-pixel shifts are the same surface"""
    a = FC.value_noise(80, 100, 5); b = FC.value_noise(80, 100, 5, (3.0, 2.0))
    assert np.array_equal(a[2:, 3:], b[:-2, :-3]) and a.std() > 20
