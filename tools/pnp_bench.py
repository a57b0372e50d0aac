"""Times dynoba_pnp_ransac_batch (one call = copies in, one launch, copies out) on seeded frames and prints one JSON line:
  frame         camera (1 500 correspondences) + 10 objects (~200 each), 10 % gross outliers
  heavy_frame   the same sizes at 40 % outliers (the 500-iteration cap)
  batch_400     400 problems of 50-400 correspondences, 0-50 % outliers
Median / min ms per call over --iters calls after --warmup, hypotheses evaluated per call, and cv2.solvePnPRansac (CPU,
SOLVEPNP_P3P, 500 iterations, 1 px, 0.995) over the problems of `frame` one by one as a CPU reference point -- not OpenGV.
The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynosam_b200 import binding  # noqa: E402
from dynosam_b200.synth_star import K5, make_pnp_problem  # noqa: E402


def frame(seed, outliers):
    rng = np.random.default_rng(seed)
    return [make_pnp_problem(rng, 1500, outliers=outliers)] + [make_pnp_problem(rng, int(n), outliers=outliers) for n in rng.integers(180, 221, 10)]


def time_calls(probs, iters, warmup):
    for _ in range(warmup):
        out = binding.pnp_ransac_batch(probs)
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter(); out = binding.pnp_ransac_batch(probs); ts.append((time.perf_counter() - t0)*1e3)
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), problems=len(probs),
                correspondences=int(sum(len(q["kp"]) for q in probs)), hypotheses=int(sum(r["iterations"] + r["skipped"] for r in out)),
                evaluated_models=int(sum(r["iterations"] for r in out)), max_iterations_hit=int(sum(r["iterations"] == 501 for r in out)))


def cv2_frame(probs, iters):
    import cv2
    Km = np.array([[K5[0], K5[2], K5[3]], [0, K5[1], K5[4]], [0, 0, 1.0]])
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        for q in probs:
            cv2.solvePnPRansac(q["points"], q["kp"], Km, None, iterationsCount=500, reprojectionError=1.0, confidence=0.995, flags=cv2.SOLVEPNP_P3P)
        ts.append((time.perf_counter() - t0)*1e3)
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), threads=cv2.getNumThreads())


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        name, power = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power)
    except Exception as e:          # pragma: no cover
        return dict(gpu=f"unknown ({e})", power_limit="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    f, h = frame(1, 0.1), frame(2, 0.4)
    rng = np.random.default_rng(3)
    b = [make_pnp_problem(rng, int(n), outliers=float(o)) for n, o in zip(rng.integers(50, 401, 400), rng.choice([0.0, 0.1, 0.3, 0.5], 400))]
    res = dict(metric="pnp_ransac_batch", launches_per_call=1, **gpu_info())
    res["frame"] = time_calls(f, a.iters, a.warmup)
    res["heavy_frame"] = time_calls(h, a.iters, a.warmup)
    res["batch_400"] = time_calls(b, max(a.iters//5, 3), a.warmup)
    res["cv2_cpu_frame"] = cv2_frame(f, max(a.iters//5, 3))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
