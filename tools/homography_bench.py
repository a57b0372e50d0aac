"""Times dynofront_find_homography_batch and dynofront_klt_track_points and prints one JSON line:
  single_<p>     one 800-point problem at p % outliers (5, 30, 60): device time per call (CUDA events, copies included);
                 single_<p>_ransac_only the same call with refine = 0 (no final DLT, LM or mask recomputation)
  batch_400      400 problems of 50-800 points, 0-60 % outliers, in one call
  klt_c4         KltFeatureTracker::trackPoints on the synthetic C4 stream (1242 x 375, 800 points): klt_track_points against
                 klt_track_fb + host compaction + cv2.findHomography, wall clock per frame
  cv2_<p>        cv2.findHomography(RANSAC, 5.0) on the same 800-point problems, host time per call
Median / min over --iters calls after --warmup.  The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynosam_b200.frontend import FeatureTrackerGPU, HomographyParams  # noqa: E402
from dynosam_b200.synth_frames import SyntheticStream, W, H  # noqa: E402


def problem(rng, n, frac):
    a = rng.random((n, 2))*[W, H]
    Hm = np.array([[1 + rng.normal(0, .01), rng.normal(0, .01), rng.normal(0, 5)], [rng.normal(0, .01), 1 + rng.normal(0, .01), rng.normal(0, 5)],
                   [rng.normal(0, 1e-5), rng.normal(0, 1e-5), 1]])
    w = a @ Hm[2, :2] + 1
    b = np.stack([(a @ Hm[0, :2] + Hm[0, 2])/w, (a @ Hm[1, :2] + Hm[1, 2])/w], 1) + rng.normal(0, 1.0, a.shape)
    k = int(n*frac); b[:k] += rng.normal(0, 40, (k, 2))
    return a.astype(np.float32), b.astype(np.float32)


def stats(ts):
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), runs=len(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import cv2
    cv2.setNumThreads(1)
    rng = np.random.default_rng(1)
    t = FeatureTrackerGPU(W, H)
    out = {}
    for pct in (5, 30, 60):
        p = problem(rng, 800, pct/100)
        for _ in range(args.warmup):
            t.find_homography_batch([p])
        dev = []; cpu = []
        for _ in range(args.iters):
            r = t.find_homography_batch([p]); dev.append(t.last_ms)
            t0 = time.perf_counter(); cv2.findHomography(p[0], p[1], cv2.RANSAC, 5.0); cpu.append((time.perf_counter() - t0)*1e3)
        out[f"single_{pct}"] = dict(stats(dev), iterations=int(r["iterations"][0]), inliers=int(r["n_inliers"][0]))
        ran = []
        for _ in range(args.iters):
            t.find_homography_batch([p], HomographyParams(refine=False)); ran.append(t.last_ms)
        out[f"single_{pct}_ransac_only"] = stats(ran)
        out[f"cv2_{pct}"] = stats(cpu)
    batch = [problem(rng, int(rng.integers(50, 801)), float(rng.uniform(0, 0.6))) for _ in range(400)]
    for _ in range(args.warmup):
        t.find_homography_batch(batch)
    dev = []
    for _ in range(args.iters):
        r = t.find_homography_batch(batch); dev.append(t.last_ms)
    out["batch_400"] = dict(stats(dev), iterations=int(r["iterations"].sum()))
    # C4 stream: one tracker for each path
    stream = SyntheticStream(n_objects=10, seed=42)
    frames = [stream.frame(k) for k in range(20, 20 + 2 + args.warmup + args.iters)]
    pts = np.stack([rng.uniform(5, W - 5, 800), rng.uniform(5, H - 5, 800)], 1).astype(np.float32)
    age = np.zeros(800, np.int32)
    a = FeatureTrackerGPU(W, H); b = FeatureTrackerGPU(W, H)
    one = []; chain = []
    for k in range(1, len(frames)):
        g0 = frames[k - 1][0]; g1, m1, f1 = frames[k]
        a.set_frame(f1, m1, None); b.set_frame(f1, m1, None)
        t0 = time.perf_counter(); a.klt_track_points(g0, g1, pts, None, age, 25); t1 = time.perf_counter()
        nxt, st, _, keep = b.klt_track_fb(g0, g1, pts, None, age, 25)
        good = np.nonzero(st)[0]
        if len(good) >= 4:
            cv2.findHomography(pts[good], nxt[good], cv2.RANSAC, 5.0)
        t2 = time.perf_counter()
        if k > args.warmup:
            one.append((t1 - t0)*1e3); chain.append((t2 - t1)*1e3)
    out["klt_c4"] = dict(klt_track_points=stats(one), klt_track_fb_plus_cv2=stats(chain))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        out["gpu"] = q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        out["gpu"] = f"unknown ({e})"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
