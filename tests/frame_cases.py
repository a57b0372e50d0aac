"""Frame sizes for the front end's image kernels (TEST INFRASTRUCTURE): the sizes the reference's data providers produce and
edge sizes chosen for the geometry rules of frontend.cu, each naming the boundaries it hits, in the style of
band_reference.Case; the image sources for them; the detection helpers the GPU tests share.

The boundaries:
  dataset             a frame size of a data provider of the reference (KITTI 00 / 18 / 20, VIODE, TartanAir, Aria, camera tests)
  w_mult32            W % 32 == 0: every column of the Sobel y-derivative row pass takes OpenCV's SIMD FMA chain
  w_mult32_minus1 / w_mult32_plus1   W one below / above a multiple of 32 (the longest / shortest scalar tail)
  w_below32           W < 32: no column takes the SIMD chain
  clahe_w8_only       W % 8 == 0, H % 8 != 0: CLAHE pads both sides, W by 8 reflected columns
  clahe_h8_only       H % 8 == 0, W % 8 != 0: likewise with 8 reflected rows
  clahe_both8         both sides multiples of 8: no padding, tile = side / 8
  lk_top1 / lk_top2 / lk_top3   klt_top_level(5, 21) stops at level 1 / 2 / 3
  lk_level_eq_win     the first level klt_top_level refuses is exactly win = 21 px on a side (84 -> 42 -> 21)
  lk_level_win_plus1  a level klt_top_level keeps is win + 1 = 22 px on a side (86 -> 43 -> 22)
  odd_level           an odd side at some pyramid level >= 1
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from dynosam_b200.synth_frames import SyntheticStream

REQUIRED = ("dataset", "w_mult32", "w_mult32_minus1", "w_mult32_plus1", "w_below32", "clahe_w8_only", "clahe_h8_only", "clahe_both8",
            "lk_top1", "lk_top2", "lk_top3", "lk_level_eq_win", "lk_level_win_plus1", "odd_level")
STREAM_MIN_W, STREAM_MIN_H = 160, 110            # SyntheticStream places objects up to 159 x 109 px
CLAHE_MIN = 16                                   # CLAHE reflects up to 8 rows / columns once


def klt_top_level(w, h, max_level, win):
    """frontend.cu's klt_top_level: buildOpticalFlowPyramid stops where the next level is not larger than the window"""
    levels = 0
    for lvl in range(min(max_level, 7) + 1):
        levels = lvl
        if lvl < max_level:
            w2, h2 = (w + 1)//2, (h + 1)//2
            if w2 <= win or h2 <= win:
                break
            w, h = w2, h2
    return levels


def level_sizes(w, h, top):
    out = [(w, h)]
    for _ in range(top):
        w, h = (w + 1)//2, (h + 1)//2
        out.append((w, h))
    return out


def boundaries(w, h, win=21, max_level=5):
    """the boundaries of the module docstring that a w x h frame reaches"""
    b = set()
    if w % 32 == 0: b.add("w_mult32")
    if w % 32 == 31: b.add("w_mult32_minus1")
    if w % 32 == 1 and w > 32: b.add("w_mult32_plus1")
    if w < 32: b.add("w_below32")
    if w % 8 == 0 and h % 8 != 0: b.add("clahe_w8_only")
    if h % 8 == 0 and w % 8 != 0: b.add("clahe_h8_only")
    if w % 8 == 0 and h % 8 == 0: b.add("clahe_both8")
    top = klt_top_level(w, h, max_level, win)
    if 1 <= top <= 3: b.add(f"lk_top{top}")
    sizes = level_sizes(w, h, top + 1)
    if top < max_level and min(sizes[top + 1]) == win: b.add("lk_level_eq_win")
    if any(min(s) == win + 1 for s in sizes[:top + 1]): b.add("lk_level_win_plus1")
    if any(s[0] % 2 or s[1] % 2 for s in sizes[1:top + 1]): b.add("odd_level")
    return b


@dataclass(frozen=True)
class Case:
    name: str
    w: int
    h: int
    hits: tuple
    wins: tuple = (21, 31)            # the LK windows run at this size (every side >= win + 1)

    @property
    def stream(self):
        """SyntheticStream frames when the size allows them, else the value-noise texture"""
        return self.w >= STREAM_MIN_W and self.h >= STREAM_MIN_H

    @property
    def dataset(self):
        return "dataset" in self.hits


CASES = {c.name: c for c in (
    Case("kitti00_1242x375", 1242, 375, ("dataset", "odd_level")),                                # the control
    Case("kitti18_1238x374", 1238, 374, ("dataset", "odd_level")),
    Case("kitti20_1241x376", 1241, 376, ("dataset", "clahe_h8_only", "odd_level")),
    Case("viode_752x480", 752, 480, ("dataset", "clahe_both8")),
    Case("tartan_aria_640x360", 640, 360, ("dataset", "w_mult32", "clahe_both8", "odd_level")),
    Case("camera_640x480", 640, 480, ("dataset", "w_mult32", "clahe_both8")),
    Case("w1248x200", 1248, 200, ("w_mult32", "clahe_both8")),
    Case("w1247x201", 1247, 201, ("w_mult32_minus1", "odd_level")),
    Case("w1249x199", 1249, 199, ("w_mult32_plus1",)),
    Case("w27x72", 27, 72, ("w_below32",), wins=(21,)),
    Case("w328x203_w8", 328, 203, ("clahe_w8_only", "odd_level")),
    Case("h8_245x168", 245, 168, ("clahe_h8_only", "lk_top2")),
    Case("lk_top1_96x64", 96, 64, ("lk_top1", "clahe_both8")),
    Case("lk_eq_win_120x84", 120, 84, ("lk_level_eq_win", "lk_top1", "clahe_w8_only")),
    Case("lk_win_plus1_130x86", 130, 86, ("lk_level_win_plus1", "lk_top2", "odd_level")),
    Case("lk_top3_180x172", 180, 172, ("lk_top3", "odd_level")),
)}
DATASET = [c.name for c in CASES.values() if c.dataset]


def value_noise(h, w, seed, shift=(0.0, 0.0)):
    """a seeded value-noise texture (uint8), sampled at (x + shift[0], y + shift[1]): a shift gives the same surface moved by a
    sub-pixel amount, a frame pair for the KLT at any size"""
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w))
    for cells, wt in ((2, 0.35), (5, 0.4), (11, 0.25)):
        nh, nw = h + 8*cells + 8, w + 8*cells + 8
        g = rng.uniform(0, 255, (nh//cells + 2, nw//cells + 2))
        ys = (np.arange(h) + shift[1] + 4*cells)/cells; xs = (np.arange(w) + shift[0] + 4*cells)/cells
        y0 = np.floor(ys).astype(int); x0 = np.floor(xs).astype(int); fy = (ys - y0)[:, None]; fx = (xs - x0)[None, :]
        img += wt*(g[y0][:, x0]*(1 - fx)*(1 - fy) + g[y0][:, x0 + 1]*fx*(1 - fy) + g[y0 + 1][:, x0]*(1 - fx)*fy + g[y0 + 1][:, x0 + 1]*fx*fy)
    return np.ascontiguousarray(np.clip(np.rint(img), 0, 255).astype(np.uint8))


def frame(case: Case, k, seed=42, n_objects=6):
    """frame k of the case: (gray uint8, motion mask int32, flow float32[H][W][2]), C-contiguous.  SyntheticStream at the
    case's size; below its minimum size the value-noise texture moved by (0.6 k, -0.35 k) px with an empty mask and that flow"""
    if case.stream:
        g, m, f = SyntheticStream(n_objects=n_objects, seed=seed, width=case.w, height=case.h).frame(k)
        return np.ascontiguousarray(g, np.uint8), np.ascontiguousarray(m, np.int32), np.ascontiguousarray(f, np.float32)
    g = value_noise(case.h, case.w, seed, (0.6*k, -0.35*k))
    f = np.zeros((case.h, case.w, 2), np.float32); f[..., 0] = -0.6; f[..., 1] = 0.35
    return g, np.zeros((case.h, case.w), np.int32), f


# ------------------------------------------------------------------------------------------------ detection helpers
def c4(k, seed=42):
    """frame k of the 1242 x 375 C4 stream (10 objects)"""
    g, m, f = SyntheticStream(n_objects=10, seed=seed).frame(k)
    return np.ascontiguousarray(g.astype(np.uint8)), np.ascontiguousarray(m.astype(np.int32)), np.ascontiguousarray(f.astype(np.float32))


def texture(h, w, seed):
    """blurred uniform noise: many strong corners"""
    import cv2
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(cv2.GaussianBlur(rng.integers(0, 256, (h, w)).astype(np.uint8), (0, 0), 1.2))


def cur_features(rng, m, n):
    """n current features on the background of motion mask m, at sub-pixel positions"""
    ys, xs = np.nonzero(m == 0)
    s = rng.choice(len(ys), n, replace=False)
    return np.stack([xs[s] + rng.uniform(0, 1, n), ys[s] + rng.uniform(0, 1, n)], 1)


def dev_params(p):
    """the device's DetectParams for detection_oracle.Params"""
    from dynosam_b200.frontend import DetectParams
    return DetectParams(use_clahe=p.use_clahe, use_anms=p.use_anms, use_subpix=p.use_subpix, max_corners=p.max_corners,
                        quality_level=p.quality_level, min_distance=p.min_distance, max_features=p.max_features,
                        shrink_row=p.shrink_row, shrink_col=p.shrink_col)
