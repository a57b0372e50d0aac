"""Time dynoba_imu_preintegrate_batch (combined IMU preintegration, one warp per frame interval) on the GPU.

Workloads: 2 000 and 10 000 intervals (the C3 / C5 frame counts) at 10, 20 and 200 samples per interval, and ragged lengths
(2..40 samples).  Per workload, after a warm-up: the whole call (host-to-device copies, one launch, device-to-host copies)
by CUDA events around it, repeated; the kernel alone by torch.profiler's device time of preint_kernel in a separate
profiled pass; and the host build of preint.cuh on one CPU thread (a prefix of the intervals, scaled).  Card name and
power limit are read in the same run.  Prints one JSON line per workload (and writes the list to --out if given).

    python tools/preint_bench.py [--reps 20] [--cpu-intervals 200] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def workload(n, m, seed=0):
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 41, n) if m == "ragged" else np.full(n, m)
    st, ag = [], []
    for k in lens:
        st.append(np.cumsum(np.concatenate([[0.0], rng.uniform(0.004, 0.006, k - 1)])))
        ag.append(np.concatenate([rng.normal(0, 3, (k, 3)) + [0, 0, 9.81], rng.normal(0, 0.5, (k, 3))], 1))
    return st, ag


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cpu-intervals", type=int, default=200, help="intervals the one-thread host build times (scaled up)")
    a = ap.parse_args()
    import ctypes as C

    import torch
    from dynosam_b200 import binding
    import test_preint as TP
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: preint_bench measures the GPU only")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    T = np.eye(4); T[:3, :3] = np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]])
    P = binding.imu_frontend_params((0.0, 9.8, 0.0), 0.2, 0.05, 0.02, 4e-5, 1e-3, T)
    L = binding.load()
    host = TP.build_shim(__import__("pathlib").Path(tempfile.mkdtemp()))
    out = []
    for n in (2000, 10000):
        for m in (10, 20, 200, "ragged"):
            st, ag = workload(n, m)
            off, sts, ags = binding._preint_args(st, ag)
            rec = np.zeros((n, 70)); cov = np.zeros((n, 225)); R = np.zeros((n, 225)); status = np.zeros(n, np.int32)
            dp, ip = binding._dp, binding._ip

            def call():
                rc = L.dynoba_imu_preintegrate_batch(0, C.byref(P), n, ip(off), dp(sts), dp(ags), None, dp(rec), dp(cov), dp(R), ip(status))
                assert rc == 0, rc
            for _ in range(3):
                call()                                   # warm-up: module load, workspace growth
            times = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize(); e0.record(); call(); e1.record(); torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    call()
                torch.cuda.synchronize()
            kern = [e.device_time_total for e in prof.key_averages() if "preint_kernel" in e.key]
            kernel_ms = sum(kern)/1e3/3 if kern else float("nan")
            k = min(a.cpu_intervals, n)
            h0 = time.perf_counter()
            TP.host_batch(host, P, [(st[i], ag[i], None) for i in range(k)])
            cpu_ms = (time.perf_counter() - h0)*1e3*n/k
            steps = int(sum(len(s) - 1 for s in st))
            r = dict(intervals=n, samples=m, steps=steps, call_ms_median=float(np.median(times)), call_ms_min=float(np.min(times)),
                     call_ms_max=float(np.max(times)), kernel_ms=kernel_ms, input_MB=(8*7*int(off[-1]) + 4*(n + 1))/1e6, output_MB=8*520*n/1e6,
                     cpu_one_thread_ms=cpu_ms, card=card)
            print(json.dumps(r), flush=True)
            out.append(r)
    if a.out:
        json.dump(out, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
