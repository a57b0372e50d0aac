"""Timing of dynoba_marginal_covariance on the synthetic configurations (default C3 and C5, hybrid formulation).

Per configuration, on one handle at the initial values:
    latest pose     the first call (the latest camera pose, as ParallelHybridBackendModule asks for it): linearise,
                    build the undamped reduced system, plain band factorisation, selected inversion, gather
    all poses       every pose-like block, from the kept selected inverse
    all points      every point: landmark kernels + gather
and the CUDA-event times of the stages (DYNOBA_TIMING lines of the library), the device memory the handle holds
after the calls beyond what it held before them, the GPU's name, power limit and SM clock.  Repeated `--reps` times
after one warm-up on fresh values (dynoba_set_variables invalidates the kept inverse).  There is no GTSAM or CPU
number at this scale: the CPU oracle's dense normal equations do not fit.

    python tools/covariance_bench.py [--configs C3 C5] [--reps 3] [--out covariance_bench.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from dynosam_b200 import synth  # noqa: E402
from dynosam_b200.binding import POINT3, POSE6, Solver  # noqa: E402


class StderrCapture:
    """the library prints its stage times to fd 2"""
    def __enter__(self):
        self.f = tempfile.TemporaryFile(mode="w+b")
        sys.stderr.flush()
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        return self

    def __exit__(self, *a):
        sys.stderr.flush()
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read().decode(errors="replace")
        self.f.close()


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unavailable ({e})"


def mem_used():
    """bytes in use on the device (every process: read it on an otherwise idle GPU)"""
    import torch
    free, total = torch.cuda.mem_get_info()
    return total - free


def stage_times(text):
    out = {}
    for m in re.finditer(r"reduced system ([\d.]+) ms\s+factor ([\d.]+) ms\s+selected inversion ([\d.]+) ms", text):
        out = {"build_ms": float(m.group(1)), "factor_ms": float(m.group(2)), "selinv_ms": float(m.group(3))}
    for m in re.finditer(r"landmarks ([\d.]+) ms", text):
        out["landmarks_ms"] = float(m.group(1))
    return out


def run(cfg, reps):
    p = synth.make_config(cfg, formulation="hybrid")
    order = p.pose_order if p.pose_order is not None else np.arange(p.n_pose)
    latest = int(np.argsort(order, kind="stable")[-1])
    s = Solver(p)
    info = s.info()
    s.finalize()
    rows = []
    for r in range(reps + 1):
        s.reset_values()                        # fresh values: the kept inverse goes
        m0 = mem_used()
        with StderrCapture() as cap:
            t0 = time.perf_counter(); s.marginal_covariance(POSE6, [latest]); t1 = time.perf_counter()
            s.marginal_covariance(POSE6); t2 = time.perf_counter()
            s.marginal_covariance(POINT3); t3 = time.perf_counter()
        m1 = mem_used()
        row = {"latest_pose_ms": 1e3*(t1 - t0), "all_poses_ms": 1e3*(t2 - t1), "all_points_ms": 1e3*(t3 - t2),
               "held_bytes": m1 - m0, **stage_times(cap.text)}
        if r:
            rows.append(row)
    s.close()
    med = {k: float(np.median([x[k] for x in rows])) for k in rows[0]}
    return {"config": cfg, "n_pose": p.n_pose, "n_point": p.n_point, "reduced_dim": info["reduced_dim"],
            "bandwidth": info["bandwidth"], "median": med, "runs": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["C3", "C5"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    os.environ["DYNOBA_TIMING"] = "1"
    os.environ.setdefault("DYNOBA_NO_DEVCACHE", "1")     # freed blocks go back to the device: held_bytes is what a call keeps
    res = {"gpu (name, power limit, SM clock, max SM clock)": gpu_info(), "results": [run(c, a.reps) for c in a.configs]}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
