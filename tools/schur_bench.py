"""Where one damped solve's landmark elimination spends its time: the kernels of dynoba_solve on a BASELINE config,
per kernel name, from torch.profiler (CUDA activities) in a run of its own, after warm-up LM iterations.  Prints the
GPU name and power limit beside the numbers, and the window-path census the library reports (Solver.info()).

    python tools/schur_bench.py --config C5 --solves 3 --warmup 2 [--trace /tmp/schur_trace.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynosam_b200 import synth                      # noqa: E402
from dynosam_b200.binding import Solver             # noqa: E402

# kernels of the elimination, by the name the profiler shows (template arguments kept: one line per NP)
ELIMINATION = ("band_clear", "pose_factors", "schur_stage_kernel", "schur_accum_kernel", "schur_simple", "schur_general")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def short_name(name):
    """'void dynoba::schur_accum_kernel<2>(dynoba::DevWindows, ...)' -> 'schur_accum_kernel<2>'"""
    m = re.search(r"(\w+(<[^()]*>)?)\(", name)
    return m.group(1) if m else name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C5")
    ap.add_argument("--formulation", default="hybrid")
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2, help="LM iterations before the profiled solves")
    ap.add_argument("--solves", type=int, default=3, help="damped solves profiled (times are per solve)")
    ap.add_argument("--lam", type=float, default=1e-4)
    ap.add_argument("--trace", default="", help="also write the Chrome trace here")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("schur_bench.py needs a CUDA device")
    p = synth.make_config(a.config, formulation=a.formulation, seed=a.seed, scale=a.scale)
    s = Solver(p)
    s.finalize()
    s.optimize(max_iterations=a.warmup, relative_error_tol=0.0, absolute_error_tol=0.0)
    s.linearize()
    s.solve(a.lam)                                  # one unprofiled solve: every kernel of the timed ones loaded
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.solves):
            s.solve(a.lam)
        torch.cuda.synchronize()
    if a.trace:
        os.makedirs(os.path.dirname(os.path.abspath(a.trace)), exist_ok=True)
        prof.export_chrome_trace(a.trace)
    per = defaultdict(lambda: [0.0, 0])              # short name -> [total us, launches]
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = short_name(ev.name)
            per[k][0] += ev.device_time; per[k][1] += 1
    total_us = sum(v[0] for v in per.values())
    rows = {k: {"ms_per_solve": v[0]/1e3/a.solves, "launches_per_solve": v[1]/a.solves}
            for k, v in sorted(per.items(), key=lambda kv: -kv[1][0])}
    elim = {k: r for k, r in rows.items() if any(k.startswith(e) for e in ELIMINATION)}
    out = dict(config=a.config, scale=a.scale, gpu=gpu_info(), solves=a.solves, lam=a.lam,
               ms_per_solve_all_kernels=total_us/1e3/a.solves,
               ms_per_solve_elimination=sum(r["ms_per_solve"] for r in elim.values()),
               elimination=elim, info=s.info(),
               other_kernels={k: r for k, r in rows.items() if k not in elim})
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
