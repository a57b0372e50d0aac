"""Time dynoba_object_srif_batch (ObjectMotionSolverFilter's predict + IRLS update for every object of a frame, one CTA per
object) on the GPU.

Workloads: a frame of 10 objects of 200 inliers (NEW: two updates each) and 400 objects of 200 inliers.  Per workload, after a
warm-up: the whole call (host-to-device copies, one launch, device-to-host copies, stream synchronise) by a host clock around
the C call on pre-packed arrays, repeated; and the host build of srif.cuh on one CPU thread over the same objects (the
reference's per-object host loop without its Eigen / GTSAM overheads).  Card name and power limit are read in the same run.
Prints one JSON line per workload (and writes the list to --out if given).

    python tools/srif_bench.py [--reps 50] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import pathlib
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from dynosam_b200 import binding as B
    from dynosam_b200 import synth_srif as SS
    import test_srif as TS
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True)
    if card.returncode != 0:
        raise SystemExit("no CUDA device: srif_bench measures the GPU only")
    card = card.stdout.strip().splitlines()[0]
    L = B.load()
    host = TS.build_shim(pathlib.Path(tempfile.mkdtemp()))
    prm = B.SrifParams(); L.dynoba_object_srif_default_params(C.byref(prm))
    out = []
    for n_obj in (10, 400):
        objs = SS.random_frame(n_obj, 200, seed=1)
        arr, total = B.srif_arrays(objs)
        for _ in range(3):
            assert B.srif_call(L.dynoba_object_srif_batch, arr, prm, 0) == 0
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rc = B.srif_call(L.dynoba_object_srif_batch, arr, prm, 0)      # returns after its stream synchronise
            ts.append(time.perf_counter() - t0)
            assert rc == 0
        harr, _ = B.srif_arrays(objs)
        th = []
        for _ in range(max(3, a.reps//10)):
            t0 = time.perf_counter()
            B.srif_call(host.host_srif_batch, harr, prm)
            th.append(time.perf_counter() - t0)
        dev = B.srif_results(arr); hst = B.srif_results(harr)
        worst = max(TS.compare(d, h, 16.0) for d, h in zip(dev, hst))
        r = dict(workload=f"{n_obj} objects x 200 inliers (NEW)", correspondences=total, card=card,
                 call_ms_median=1e3*float(np.median(ts)), call_ms_min=1e3*float(np.min(ts)),
                 host_one_thread_ms_median=1e3*float(np.median(th)), device_vs_host_worst_in_16eps_kappa=float(worst))
        print(json.dumps(r), flush=True)
        out.append(r)
    B.load().dynoba_batch_release(0)
    if a.out:
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
