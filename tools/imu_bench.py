"""Cost of the IMU chain on the device: the same synthetic graph with and without the visual-inertial chain
(synth.make_problem(imu=True): velocities, biases, their priors and one COMBINED_IMU15 per frame pair in place of the
odometry), arms alternating, CUDA-event times from dynoba_lm_stats.  Prints one JSON line.

    python tools/imu_bench.py --config C3 --runs 2 --iterations 5
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynosam_b200 import synth                      # noqa: E402
from dynosam_b200.binding import Solver             # noqa: E402
from dynosam_b200.problem import COMBINED_IMU15     # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def run(p, iterations):
    s = Solver(p)
    s.finalize()
    st = s.optimize(max_iterations=iterations, relative_error_tol=0.0, absolute_error_tol=0.0)
    r = dict(ms_per_iteration=st["ms_total"]/max(st["inner_iterations"], 1), iterations=st["iterations"],
             inner_iterations=st["inner_iterations"], ms_factor=st["ms_factor"]/max(st["inner_iterations"], 1),
             reduced_dim=st["reduced_dim"], bandwidth=st["bandwidth"], error_final=st["error_final"])
    imu = [i for i, b in enumerate(p.blocks) if b.type == COMBINED_IMU15]
    if imu:
        s.linearize_block(imu[0])
        r["imu_linearize_block_ms"] = float(np.median([s.linearize_block(imu[0])[0] for _ in range(20)]))
    s.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0)
    a = ap.parse_args()
    probs = {arm: synth.make_config(a.config, scale=a.scale, imu=(arm == "imu")) for arm in ("plain", "imu")}
    out = {arm: [] for arm in probs}
    run(probs["plain"], 1)                         # warm-up: module load, allocation cache
    for _ in range(a.runs):
        for arm in ("plain", "imu"):
            out[arm].append(run(probs[arm], a.iterations))
    res = dict(config=a.config, scale=a.scale, gpu=gpu_info(), runs=out,
               n_imu_factors=int(sum(b.n for b in probs["imu"].blocks if b.type == COMBINED_IMU15)))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
