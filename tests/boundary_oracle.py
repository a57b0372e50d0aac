"""vision_tools::computeObjectMaskBoundaryMask on a provided motion mask (VisionTools.cc:286-449) as FeatureTracker::objectDetection
calls it (FeatureTracker.cc:1151-1210), composed literally from cv2 (TEST INFRASTRUCTURE).  It deliberately does not use the
restatement of dynosam_b200/frontend_csrc/boundary.cuh (column max, per-pixel morphology rules), so the tests that compare the
two show that the restatement holds.  Labels are visited in ascending order: the reference's getObjectLabels returns an
unordered_set's order, and so leaves the last writer of overlapping drawContours unspecified."""
from __future__ import annotations

import cv2
import numpy as np

INNER = 10                       # inner_thickness (VisionTools.cc:412)


def thickness(w, h):
    """objectDetection's scaled_boarder_thickness, as the reference writes it (int product, double ratio, std::round)"""
    image_ratio = float(np.int32(w)*np.int32(h))/(640.0*480.0)
    v = image_ratio*640.0/480.0*7.51
    return int(np.floor(v + 0.5))                  # std::round: half away from zero (v > 0)


def find_object_bounding_box(mask, object_id):
    """findObjectBoundingBox (VisionTools.cc:286-323): (found, (x, y, w, h), contours)"""
    obj = cv2.compare(mask, np.full_like(mask, object_id), cv2.CMP_EQ)
    dil = cv2.dilate(obj, cv2.getStructuringElement(cv2.MORPH_RECT, (1, 11)), anchor=(-1, -1))
    contours, _ = cv2.findContours(dil, cv2.RETR_TREE, cv2.CHAIN_APPROX_NONE)
    if len(contours) == 0:
        return False, (0, 0, 0, 0), contours
    rects = [cv2.boundingRect(c) for c in contours]
    x0 = min(r[0] for r in rects); y0 = min(r[1] for r in rects)
    x1 = max(r[0] + r[2] for r in rects); y1 = max(r[1] + r[3] for r in rects)
    return True, (x0, y0, x1 - x0, y1 - y0), contours


def object_labels(mask):
    """getObjectLabels without the background label, ascending"""
    return [int(v) for v in np.unique(mask) if v != 0]


def object_boundary(mask, t):
    """ObjectBoundaryMaskResult of computeObjectMaskBoundaryMask(mask, t, use_as_feature_detection_mask=true):
    (objects, bb [n][4], inner_bb [n][4], boundary_mask u8[H][W])"""
    mask = np.ascontiguousarray(mask, np.int32)
    objects = object_labels(mask)
    assert all(0 < j <= 255 for j in objects), "CHECK_LE(object_id, 255)"
    thicc = np.zeros(mask.shape, np.uint8)
    bb = []
    for j in objects:
        found, rect, contours = find_object_bounding_box(mask, j)
        assert found
        cv2.drawContours(thicc, contours, -1, int(j), cv2.FILLED)
        bb.append(rect)
    dilated = cv2.dilate(thicc, cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2*t + 1, 2*t + 1)))
    outer = cv2.subtract(dilated, thicc)
    eroded = cv2.erode(thicc, cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2*INNER + 1, 2*INNER + 1)))
    inner = cv2.subtract(thicc, eroded)
    inner_bb = [find_object_bounding_box(eroded, j)[1] for j in objects]
    boundary = np.full(mask.shape, 255, np.uint8)
    boundary[outer != 0] = 0
    boundary[inner != 0] = 0
    return (np.array(objects, np.int32), np.array(bb, np.int32).reshape(-1, 4), np.array(inner_bb, np.int32).reshape(-1, 4), boundary)
