"""Seeded synthetic RGB-D-like stream for the front-end rows (SURVEY.md 8d, config C4): procedurally textured
background (value noise), moving textured rectangles as objects, instance mask CV_32S, exact per-pixel flow CV_32FC2."""
from __future__ import annotations

import numpy as np

W, H = 1242, 375


def _value_noise(rng, h, w, cells):
    g = rng.uniform(0, 255, (h//cells + 2, w//cells + 2))
    ys = np.arange(h)/cells; xs = np.arange(w)/cells
    y0 = ys.astype(int); x0 = xs.astype(int); fy = (ys - y0)[:, None]; fx = (xs - x0)[None, :]
    a = g[y0][:, x0]; b = g[y0][:, x0 + 1]; c = g[y0 + 1][:, x0]; d = g[y0 + 1][:, x0 + 1]
    return a*(1 - fx)*(1 - fy) + b*fx*(1 - fy) + c*(1 - fx)*fy + d*fx*fy


class SyntheticStream:
    def __init__(self, n_objects=10, seed=42, width=W, height=H):
        self.rng = np.random.default_rng(seed); self.W, self.H = width, height; self.seed = seed
        rng = self.rng
        self.bg = (0.5*_value_noise(rng, height, width + 400, 8) + 0.3*_value_noise(rng, height, width + 400, 3)
                   + 0.2*rng.uniform(0, 255, (height, width + 400)))
        self.cam_v = 1.5                                     # background scroll, px / frame
        self.obj = []
        for j in range(n_objects):
            w = int(rng.integers(60, 160)); h = int(rng.integers(40, 110))
            tex = 0.6*_value_noise(rng, h, w, 5) + 0.4*rng.uniform(0, 255, (h, w))
            self.obj.append(dict(label=j + 1, w=w, h=h, tex=tex, x=float(rng.uniform(0, width - w)), y=float(rng.uniform(0, height - h)),
                                 vx=float(rng.uniform(-3, 3)), vy=float(rng.uniform(-1, 1))))

    def frame(self, k):
        """gray uint8, mask int32, flow float32[H,W,2] (flow from frame k to k+1)."""
        W_, H_ = self.W, self.H
        off = self.cam_v*k
        i0 = int(np.floor(off)); f = off - i0
        wb = self.bg.shape[1]                               # the background strip wraps around: streams of any length
        c0 = (i0 + np.arange(W_)) % wb; c1 = (i0 + 1 + np.arange(W_)) % wb
        gray = (1 - f)*self.bg[:, c0] + f*self.bg[:, c1]
        mask = np.zeros((H_, W_), np.int32)
        flow = np.zeros((H_, W_, 2), np.float32); flow[..., 0] = -self.cam_v; flow[..., 1] = 1e-3   # no exact zeros in the background
        for o in self.obj:
            x = o["x"] + o["vx"]*k; y = o["y"] + o["vy"]*k
            x = (x + o["w"]) % (W_ + o["w"]) - o["w"]; y = (y + o["h"]) % (H_ + o["h"]) - o["h"]   # objects re-enter on the other side
            xi, yi = int(round(x)), int(round(y))
            x0, y0 = max(xi, 0), max(yi, 0); x1, y1 = min(xi + o["w"], W_), min(yi + o["h"], H_)
            if x1 <= x0 or y1 <= y0:
                continue
            gray[y0:y1, x0:x1] = o["tex"][y0 - yi:y1 - yi, x0 - xi:x1 - xi]
            mask[y0:y1, x0:x1] = o["label"]
            flow[y0:y1, x0:x1, 0] = o["vx"]; flow[y0:y1, x0:x1, 1] = o["vy"] if o["vy"] != 0 else 1e-3
        return np.clip(gray, 0, 255).astype(np.uint8), mask, flow

    # fixed pixels of depth(k) that hold the values updateDepths / projectToDenseCloud treat specially (d == 30 and d == 200 are
    # the yaml thresholds max_object_depth / max_background_depth, kept by both)
    DEPTH_EDGE_VALUES = (0.0, -1.5, np.nan, np.inf, -np.inf, 30.0, 200.0)

    def depth_edge_pixels(self):
        """{value index: (rows, cols)} of the edge pixels of depth(k), the same in every frame"""
        t = np.arange(8)
        return {j: ((7 + 37*t + 3*j) % self.H, (11 + 131*j + 17*t) % self.W) for j in range(len(self.DEPTH_EDGE_VALUES))}

    def depth(self, k):
        """depth float64[H,W] in metres (CV_64F) for frame k, drawn from generators of its own (frame(k) is unchanged).
        Background 5-263 m, nearer towards the bottom rows; each object at its own depth in 8-60 m plus a small slope, so both
        classes lie on both sides of 30 m and 200 m.  The pixels of depth_edge_pixels() hold 0, -1.5, NaN, +-inf, 30 and 200."""
        _, mask, _ = self.frame(k)
        rng = np.random.default_rng([self.seed, 0x6465707468, k])
        r = (np.arange(self.H)/max(self.H - 1, 1))[:, None]; c = (np.arange(self.W)/max(self.W - 1, 1))[None, :]
        d = 8.0 + 252.0*(1.0 - r)**2 + 3.0*np.sin(2*np.pi*(c + 0.01*k)) + rng.normal(0.0, 0.05, (self.H, self.W))
        for o in self.obj:
            sel = mask == o["label"]
            if sel.any():
                base = np.random.default_rng([self.seed, 0x6f626a, o["label"]]).uniform(8.0, 60.0)
                ys, xs = np.nonzero(sel)
                d[ys, xs] = base + 0.08*(xs - xs.min()) + rng.normal(0.0, 0.02, len(ys))
        for j, (ys, xs) in self.depth_edge_pixels().items():
            d[ys, xs] = self.DEPTH_EDGE_VALUES[j]
        return d

    def right(self, k, fx=721.5377, baseline=0.5372):
        """the right view (gray uint8 [H,W]) of a rectified stereo pair whose left view is frame(k), rendered from frame(k) and
        depth(k): the left pixel (x, y) lands at x - fx * baseline / depth(x, y) on the same row (zero disparity where the depth is
        not finite or not positive).  Each row is resampled linearly between neighbouring left pixels of one surface (disparities
        within 1 px); where several surfaces cover a right pixel the nearer one (larger disparity) wins, and pixels no surface
        covers take seeded noise.  frame(k) and depth(k) are unchanged."""
        gray, _, _ = self.frame(k)
        d = self.depth(k)
        disp = np.where(np.isfinite(d) & (d > 0), fx*baseline/np.where(np.isfinite(d) & (d > 0), d, 1.0), 0.0)
        g = gray.astype(np.float64)
        H_, W_ = gray.shape
        xr = np.arange(W_)[None, :] - disp                             # right position of every left pixel
        a, b = xr[:, :-1], xr[:, 1:]                                   # one segment per pair of horizontal neighbours
        seg = np.abs(disp[:, 1:] - disp[:, :-1]) <= 1.0
        lo = np.ceil(np.minimum(a, b)).clip(0, W_); hi = np.floor(np.maximum(a, b)).clip(-1, W_ - 1)
        cnt = np.where(seg, np.maximum(hi - lo + 1, 0), 0).astype(np.int64).ravel()
        rows, cols = np.divmod(np.repeat(np.arange(cnt.size), cnt), W_ - 1)
        first = np.repeat(np.cumsum(cnt) - cnt, cnt)
        xp = lo.ravel()[rows*(W_ - 1) + cols] + (np.arange(cnt.sum()) - first)      # the covered right pixels of each segment
        x0, x1 = xr[rows, cols], xr[rows, cols + 1]
        t = np.where(x1 != x0, (xp - x0)/np.where(x1 != x0, x1 - x0, 1.0), 0.0)
        val = (1 - t)*g[rows, cols] + t*g[rows, cols + 1]
        dv = (1 - t)*disp[rows, cols] + t*disp[rows, cols + 1]
        pix = rows*W_ + xp.astype(np.int64)
        order = np.lexsort((dv, pix))                                  # by pixel, then disparity: the last of each pixel is the nearest
        pix, val = pix[order], val[order]
        last = np.r_[pix[1:] != pix[:-1], True]
        out = np.random.default_rng([self.seed, 0x7269676874, k]).uniform(0, 255, H_*W_)
        out[pix[last]] = val[last]
        return np.clip(np.rint(out), 0, 255).astype(np.uint8).reshape(H_, W_)
