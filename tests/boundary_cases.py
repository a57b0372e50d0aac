"""Motion masks for the object boundary mask (TEST INFRASTRUCTURE): each case names the rule of boundary.cuh it exercises.
cases() returns {name: (mask int32[H][W], thickness)}."""
from __future__ import annotations

import re
import os

import numpy as np

import boundary_oracle as BO
import frame_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUH = os.path.join(ROOT, "dynosam_b200", "frontend_csrc", "boundary.cuh")
CAP = int(re.search(r"#define BOUNDARY_MAX_THICKNESS (\d+)", open(CUH).read()).group(1))   # the largest thickness accepted


def ellipses(rng, h, w, n, labels=None, r=(1, 20)):
    """n filled ellipses with distinct labels in 1..255 (later ones on top)"""
    m = np.zeros((h, w), np.int32)
    labels = rng.choice(np.arange(1, 256), n, replace=False) if labels is None else labels
    yy, xx = np.mgrid[:h, :w]
    for j in labels:
        cx, cy, a, b = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(*r), rng.uniform(*r)
        m[((xx - cx)/a)**2 + ((yy - cy)/b)**2 <= 1] = j
    return m


def noisy(rng, h, w, n):
    """ellipses with 10 % salt holes and stray object pixels"""
    m = ellipses(rng, h, w, n)
    m[rng.random((h, w)) < 0.1] = 0
    stray = rng.random((h, w)) < 0.01
    m[stray] = rng.integers(1, 256, int(stray.sum()))
    return m


def diagonals(h, w):
    """one-pixel diagonal objects, both directions, and a two-pixel one"""
    m = np.zeros((h, w), np.int32)
    for i in range(min(h, w)):
        m[i, i] = 7
        m[i, w - 1 - i] = 200
        if i + 1 < w:
            m[i, (i + 20) % w] = 31; m[i, (i + 21) % w] = 31
    return m


def edges(h, w):
    """objects touching every edge and corner"""
    m = np.zeros((h, w), np.int32)
    m[:6, :9] = 1; m[:4, w - 12:] = 2; m[h - 7:, :5] = 3; m[h - 3:, w - 3:] = 4
    m[h//2 - 8:h//2 + 8, :3] = 5; m[h//2 - 2:h//2 + 2, w - 30:] = 6; m[:2, w//2 - 20:w//2 + 20] = 8; m[h - 1:, w//3:w//2] = 9
    return m


def singles(h, w, rng):
    """isolated single pixels, some at the border"""
    m = np.zeros((h, w), np.int32)
    m[0, 0] = 1; m[h - 1, w - 1] = 2; m[0, w - 1] = 3; m[h - 1, 0] = 4
    for j in range(5, 40):
        m[rng.integers(0, h), rng.integers(0, w)] = j
    return m


def all_labels(h=112, w=160):
    """every label 1..255 once, as small blocks (a 16 x 16 grid of 7 x 10 cells)"""
    m = np.zeros((h, w), np.int32)
    for j in range(1, 256):
        r, c = divmod(j, 16)
        m[r*7 + 1:r*7 + 5, c*10 + 2:c*10 + 8] = j
    return m


def stacked(h, w, gap, upper, lower):
    """two objects in the same columns, gap rows apart: their 1x11 dilations overlap for gap < 10"""
    m = np.zeros((h, w), np.int32)
    y = h//2 - gap//2
    m[y - 20:y, 20:80] = upper
    m[y + gap:y + gap + 20, 40:100] = lower
    return m


def thin(h, w):
    """objects narrower than the inner erosion's disc: erased by it (empty inner_bb), next to a large one"""
    m = np.zeros((h, w), np.int32)
    m[10:70, 20:24] = 3; m[40:42, 40:140] = 4; m[20:100, 60:120] = 9
    return m


def cases(dataset=True):
    rng = np.random.default_rng(2024)
    out = {}
    if dataset:
        for name in FC.DATASET:
            c = FC.CASES[name]
            out[f"stream_{name}"] = (FC.frame(c, 3)[1], BO.thickness(c.w, c.h))
    for k in range(6):
        out[f"noise_{k}"] = (noisy(rng, 120, 160, 11), [0, 1, 8, 15, 10, 4][k])
    for k in range(4):
        h, w = rng.integers(1, 80), rng.integers(1, 100)
        out[f"noise_small_{k}_{h}x{w}"] = (noisy(rng, h, w, 5), [0, 1, 8, 15][k])
    out["diagonals"] = (diagonals(96, 130), 8)
    out["edges"] = (edges(90, 150), 15)
    out["edges_t1"] = (edges(90, 150), 1)
    out["singles"] = (singles(60, 70, rng), 10)
    out["img_1x1_object"] = (np.full((1, 1), 9, np.int32), 15)
    out["img_1x1_empty"] = (np.zeros((1, 1), np.int32), 15)
    out["img_1xN"] = (np.where(np.arange(57) % 9 < 4, np.arange(57)//9 + 1, 0).astype(np.int32).reshape(1, 57), 8)
    out["img_Nx1"] = (np.where(np.arange(73) % 13 < 5, np.arange(73)//13 + 1, 0).astype(np.int32).reshape(73, 1), 8)
    out["label_255"] = (np.pad(np.full((30, 40), 255, np.int32), 30), 8)
    out["all_255_labels"] = (all_labels(), 8)
    for gap in (1, 5, 9, 10, 11):
        out[f"overlap_gap{gap}_small_on_top"] = (stacked(100, 120, gap, 3, 200), 8)
        out[f"overlap_gap{gap}_large_on_top"] = (stacked(100, 120, gap, 200, 3), 8)
    out["inner_erased"] = (thin(120, 160), 10)
    out["empty"] = (np.zeros((50, 64), np.int32), 15)
    base = ellipses(rng, 120, 160, 8, r=(4, 30))
    for t in (0, 1, 10, 15, 68):
        out[f"thickness_{t}"] = (base, t)
    out[f"thickness_cap{CAP}"] = (ellipses(rng, 90, 120, 6, r=(4, 25)), CAP)
    return {k: (np.ascontiguousarray(m, np.int32), int(t)) for k, (m, t) in out.items()}
