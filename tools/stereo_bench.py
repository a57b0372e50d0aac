"""Times dynofront_find_fundamental_batch and prints one JSON line:
  single_<p>     one 800-point two-view problem at p % outliers (5, 30, 60): device time per call (CUDA events, copies included)
  cv2_<p>        cv2.findFundamentalMat(FM_RANSAC, 1.0, 0.99) on the same problem, one host thread, time per call
  batch_400      400 problems of 15-800 points, 0-60 % outliers, in one call
  c4_stereo_*    a C4 stereo stream (SyntheticStream with its right view, up to 800 GFTT background points per frame), per frame the
                 reference's two stereoTrack calls (the second on the points moved by (0.37, -0.21) px, as after solveCameraMotion),
                 wall clock per frame, three arms taken in turn on every frame (a rotating order):
                   c4_stereo_device       next_frame + set_right + two dynofront_stereo_match calls (resident images);
                                          device_ms = the two calls' CUDA-event time
                   c4_stereo_host_mix     two dynofront_stereo_track calls + host compaction + cv2.findFundamentalMat + the
                                          per-feature loop of tests/stereo_oracle.py in Python
                   c4_stereo_cv2          the whole composition in cv2 on one host thread (tests/stereo_oracle.py with cv2's LK
                                          and findFundamentalMat), twice
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
import stereo_oracle as SO  # noqa: E402
from dynosam_b200.synth_frames import SyntheticStream  # noqa: E402


def stats(ts):
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), runs=len(ts))


def c4_stereo(t, args):
    stream = SyntheticStream(n_objects=10, seed=42)
    frames = []
    for k in range(20):
        left, right, mask, pts = SO.c4_stereo_frame(stream, k)
        frames.append((np.ascontiguousarray(left), np.ascontiguousarray(right), np.ascontiguousarray(mask),
                       np.ascontiguousarray(stream.frame(k)[2]), pts, pts + np.float32([0.37, -0.21])))

    def device(f):
        left, right, mask, flow, p1, p2 = f
        t.next_frame(left, flow, mask); t.set_right(right)
        a = t.stereo_match(p1, SO.FX, SO.BASELINE); ms = t.last_ms
        b = t.stereo_match(p2, SO.FX, SO.BASELINE)
        return ms + t.last_ms, a["n_stereo"] + b["n_stereo"]

    def host_mix(f):
        left, right, _, _, p1, p2 = f
        import cv2
        n = 0
        for p in (p1, p2):
            rp, st, _, _ = t.stereo_track(left, right, p, SO.FX, SO.BASELINE)
            good = np.flatnonzero(st)
            if len(p) < 8 or len(good) < 8:
                continue
            mask = np.zeros((len(good), 1), np.uint8)
            cv2.findFundamentalMat(p[good], rp[good], cv2.FM_RANSAC, 1.0, 0.99, 1000, mask=mask)
            n += int((SO.per_feature(p, rp, st, mask.ravel(), SO.FX, SO.BASELINE)[0] == SO.MATCHED).sum())
        return 0.0, n

    def cv2_only(f):
        left, right, _, _, p1, p2 = f
        return 0.0, sum(SO.stereo_match(left, right, p, SO.FX, SO.BASELINE, which="cv2")["n_stereo"] for p in (p1, p2))

    arms = [("c4_stereo_device", device), ("c4_stereo_host_mix", host_mix), ("c4_stereo_cv2", cv2_only)]
    wall = {a: [] for a, _ in arms}; dev = []; nst = {a: [] for a, _ in arms}
    for it in range(args.warmup + args.iters):
        f = frames[it % len(frames)]
        for j in range(len(arms)):
            name, fn = arms[(it + j) % len(arms)]
            t0 = time.perf_counter(); d, n = fn(f); ms = (time.perf_counter() - t0)*1e3
            if it >= args.warmup:
                wall[name].append(ms); nst[name].append(n)
                if name == "c4_stereo_device":
                    dev.append(d)
    out = {a: dict(stats(wall[a]), stereo_features_per_frame=float(np.mean(nst[a]))) for a, _ in arms}
    out["c4_stereo_device"]["device_ms"] = stats(dev)
    out["c4_stereo_points_per_frame"] = float(np.mean([len(f[4]) for f in frames]))
    return out


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
    out.update(c4_stereo(t, args))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        out["gpu"] = q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        out["gpu"] = f"unknown ({e})"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
