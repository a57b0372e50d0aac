"""Time one window of the sliding-window optimiser on a visual-inertial graph: ingest + finalize, optimize, and the typed
marginal (dynoba_marginal_vars, with its constant f) of the frames the next window keeps.

Settings of the reference's SLIDING_WINDOW mode (RegularBackendModule.cc:50-51): window 10 frames, overlap 4.  The window
is a synthetic visual-inertial problem (synth.make_problem(imu=True)) at the per-frame density of the C1 configuration
(35 static and 15 dynamic tracklets per frame, one object).  Times are host clocks around calls that end in a device
synchronise; each is the median of --repeats runs after one warm-up run, a fresh handle per run.  The card's name and
power limit are read in the same run.  Needs an sm_90 device: without one it fails.

    python tools/window_bench.py [--repeats 5] [--frames 10] [--overlap 4] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynosam_b200 import synth  # noqa: E402
from dynosam_b200.binding import BIAS6, POSE6, VEL3, Solver  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:                          # the timings stand without it; say so
        return f"unknown ({e})", "unknown"


def kept_set(p, overlap):
    """(kinds, idx) of X, H, V, b of the last `overlap` frames: the next window's marginal prior"""
    F = p.meta["n_frames"]
    kinds, idx = [], []
    for kind, order in ((POSE6, p.pose_order), (VEL3, p.vel_order), (BIAS6, p.bias_order)):
        sel = np.flatnonzero(order >= F - overlap)
        kinds += [kind]*sel.size; idx += list(sel)
    return np.array(kinds, np.int32), np.array(idx, np.int32)


def one_run(p, kinds, idx):
    t0 = time.perf_counter()
    s = Solver(p)
    s.finalize()                                    # ends in a device synchronise
    t1 = time.perf_counter()
    st = s.optimize()                               # returns after the last error read-back
    t2 = time.perf_counter()
    G, g, f = s.marginal_vars(kinds, idx)           # returns after the host has the marginal
    t3 = time.perf_counter()
    s.close()
    return dict(ingest_finalize_ms=1e3*(t1 - t0), optimize_ms=1e3*(t2 - t1), optimize_device_ms=st["ms_total"],
                marginal_ms=1e3*(t3 - t2), iterations=st["iterations"], error_initial=st["error_initial"],
                error_final=st["error_final"], marginal_dim=int(G.shape[0]), f=f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--overlap", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=21)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    p = synth.make_problem(n_frames=a.frames, n_objects=1, n_static=35*a.frames, n_dynamic=15*a.frames, seed=a.seed, imu=True)
    kinds, idx = kept_set(p, a.overlap)
    one_run(p, kinds, idx)                          # warm-up: module load, allocation cache
    runs = [one_run(p, kinds, idx) for _ in range(a.repeats)]
    med = {k: float(np.median([r[k] for r in runs])) for k in ("ingest_finalize_ms", "optimize_ms", "optimize_device_ms", "marginal_ms")}
    name, power = card()
    res = dict(tool="window_bench", card=name, power_limit=power, frames=a.frames, overlap=a.overlap, repeats=a.repeats,
               n_pose=p.n_pose, n_point=p.n_point, n_vel=p.n_vel, n_bias=p.n_bias, n_factors=p.n_factors,
               iterations=runs[-1]["iterations"], error_initial=runs[-1]["error_initial"], error_final=runs[-1]["error_final"],
               marginal_dim=runs[-1]["marginal_dim"], f=runs[-1]["f"], **med)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
