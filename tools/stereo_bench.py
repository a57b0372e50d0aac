"""Times dynofront_find_fundamental_batch and prints one JSON line:
  single_<p>     one 800-point two-view problem at p % outliers (5, 30, 60): device time per call (CUDA events, copies included)
  cv2_<p>        cv2.findFundamentalMat(FM_RANSAC, 1.0, 0.99) on the same problem, one host thread, time per call
  batch_400      400 problems of 15-800 points, 0-60 % outliers, in one call
Median / min over --iters calls after --warmup.  The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from dynosam_b200.frontend import FeatureTrackerGPU  # noqa: E402
from dynosam_b200.synth_frames import W, H  # noqa: E402
from fundamental_oracle import make_problem  # noqa: E402


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
        p = make_problem(100 + pct, 800, pct/100)
        for _ in range(args.warmup):
            t.find_fundamental_batch([p])
        dev = []; cpu = []
        for _ in range(args.iters):
            r = t.find_fundamental_batch([p]); dev.append(t.last_ms)
            t0 = time.perf_counter(); cv2.findFundamentalMat(p[0], p[1], cv2.FM_RANSAC, 1.0, 0.99); cpu.append((time.perf_counter() - t0)*1e3)
        out[f"single_{pct}"] = dict(stats(dev), iterations=int(r["iterations"][0]), inliers=int(r["n_inliers"][0]))
        out[f"cv2_{pct}"] = stats(cpu)
    batch = [make_problem(1000 + i, int(rng.integers(15, 801)), float(rng.uniform(0, 0.6)), ["general", "stereo"][i % 2]) for i in range(400)]
    for _ in range(args.warmup):
        t.find_fundamental_batch(batch)
    dev = []
    for _ in range(args.iters):
        r = t.find_fundamental_batch(batch); dev.append(t.last_ms)
    cpu = []
    for p in batch:
        t0 = time.perf_counter(); cv2.findFundamentalMat(p[0], p[1], cv2.FM_RANSAC, 1.0, 0.99); cpu.append((time.perf_counter() - t0)*1e3)
    out["batch_400"] = dict(stats(dev), iterations=int(r["iterations"].sum()), cv2_sum_ms=float(np.sum(cpu)))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        out["gpu"] = q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        out["gpu"] = f"unknown ({e})"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
