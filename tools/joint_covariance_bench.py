"""Timing of dynoba_joint_marginal_covariance on the synthetic configurations (default C3 and C5, hybrid formulation).

Three queries, each on a fresh linearisation point (dynoba_set_variables drops the kept factor, so every query builds
and factors S):
    (a) latest      the latest frame's camera pose X, every object motion H of that frame, and 10 landmarks seen in it
    (b) ends        the first and last camera poses: the sweeps span the whole band
    (c) spread      20 camera poses spread evenly over the trajectory
Per query: the wall time of the call (host clock), the CUDA-event times of its stages (the DYNOBA_TIMING line of the
library: build S, factor, sweeps, strips), the sweep span in tiles, |C| (requested scalars plus the poses the landmarks'
factors touch), and the device memory the handle holds after the call beyond what it held before it (the kept plain
layout).  Medians of `--reps` runs after one warm-up; the GPU's name, power limit and SM clock are printed with them.

    python tools/joint_covariance_bench.py [--configs C3 C5] [--reps 3] [--out joint_covariance_bench.json]
"""
import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from covariance_bench import StderrCapture, gpu_info, mem_used  # noqa: E402
from dynosam_b200 import synth  # noqa: E402
from dynosam_b200.binding import POINT3, POSE6, Solver  # noqa: E402
from dynosam_b200.problem import SLOT_CLASS  # noqa: E402


def queries(p):
    """(name, kinds, idx) of the three queries; camera poses are poses 0 .. n_frames-1 of the synthetic graphs"""
    N = p.meta["n_frames"]
    order = np.asarray(p.pose_order)
    last = N - 1
    motions = [int(i) for i in np.flatnonzero(order == order[last]) if i >= N]
    pts = []
    for b in p.blocks:
        cl = SLOT_CLASS[b.type]
        if 1 not in cl or 0 not in cl:
            continue
        kp, kl = cl.index(0), cl.index(1)
        pts += [int(v) for v in b.idx[b.idx[:, kp] == last, kl]]
        if len(dict.fromkeys(pts)) >= 10:
            break
    pts = list(dict.fromkeys(pts))[:10]
    a = ([POSE6]*(1 + len(motions)) + [POINT3]*len(pts), [last] + motions + pts)
    b = ([POSE6, POSE6], [0, last])
    spread = np.unique(np.linspace(0, last, 20).round().astype(int))
    c = ([POSE6]*spread.size, spread.tolist())
    return [("a_latest", *a), ("b_ends", *b), ("c_spread", *c)]


def stage_times(text):
    m = re.search(r"reduced system ([\d.]+) ms\s+factor ([\d.]+) ms(?: \(earlier call\))?\s+sweeps ([\d.]+) ms\s+strips ([\d.]+) ms"
                  r"\s+\(span (\d+) tiles, \|C\| (\d+)", text)
    if not m:
        return {}
    return {"build_ms": float(m.group(1)), "factor_ms": float(m.group(2)), "sweeps_ms": float(m.group(3)),
            "strips_ms": float(m.group(4)), "span_tiles": int(m.group(5)), "C": int(m.group(6))}


def run(cfg, reps):
    p = synth.make_config(cfg, formulation="hybrid")
    s = Solver(p)
    info = s.info()
    s.finalize()
    out = {"config": cfg, "n_pose": p.n_pose, "n_point": p.n_point, "reduced_dim": info["reduced_dim"],
           "bandwidth": info["bandwidth"], "queries": {}}
    for name, kinds, idx in queries(p):
        rows = []
        for r in range(reps + 1):
            s.reset_values()                    # fresh values: the kept factor goes
            m0 = mem_used()
            with StderrCapture() as cap:
                t0 = time.perf_counter(); C, _ = s.joint_marginal_covariance(kinds, idx); t1 = time.perf_counter()
            row = {"call_ms": 1e3*(t1 - t0), "held_bytes": mem_used() - m0, **stage_times(cap.text)}
            if r:
                rows.append(row)
        med = {k: float(np.median([x[k] for x in rows])) for k in rows[0]}
        out["queries"][name] = {"n_vars": len(idx), "D": int(C.shape[0]), "median": med, "runs": rows}
    s.close()
    return out


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
