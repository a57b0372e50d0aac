"""Where the band factorisation of one damped solve spends its time, on a BASELINE config (C5 by default).

For each split of the worker CTAs (`--ctas`: band_ctas_per_chain values, 0 = the library's default split) it prints
  * ms_factor per damped solve (the reduced solve: factorisation + sweeps) from LM iterations with the profile off;
  * with the band profile on (dynoba_set_tuning "band_profile", which synchronises after every stage and so runs after
    all the profile-off timings), each factorisation launch: its grid split, the finish time of every spine (plain or
    spiked chain) and of the two worker pools, in ms from the launch's first worker CTA, median over `--solves` solves;
plus the GPU name and power limit, read in the same process.

    python tools/band_bench.py --config C5 --warmup 2 --iters 3 --solves 3 [--ctas 0,16,22,28]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynosam_b200 import synth                      # noqa: E402
from dynosam_b200.binding import Solver             # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


class CaptureStderr:
    """the library prints its profile with fprintf(stderr): redirect file descriptor 2 into a temporary file"""
    def __enter__(self):
        sys.stderr.flush()
        self.f = tempfile.TemporaryFile(mode="w+b")
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        return self

    def __exit__(self, *exc):
        sys.stderr.flush()
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read().decode(errors="replace")
        self.f.close()


def parse_profile(text):
    """[band] lines of one solve -> list of launches {problems, WB, grid split, spines [(columns, spiked, ms)], pools}"""
    launches = []
    for line in text.splitlines():
        if m := re.match(r"\[band\]\s+launch: (\d+) problems, WB (\d+), grid (\d+) = (\d+) spines \+ (\d+) band CTAs \+ (\d+) spike CTAs", line):
            launches.append(dict(problems=int(m[1]), WB=int(m[2]), grid=int(m[3]), band_ctas=int(m[5]), spike_ctas=int(m[6]), spines=[]))
        elif (m := re.match(r"\[band\]\s+spine (\d+) \((\d+) columns(, spiked)?\) done at\s+([-\d.]+) ms", line)) and launches:
            launches[-1]["spines"].append((int(m[2]), bool(m[3]), float(m[4])))
        elif (m := re.match(r"\[band\]\s+band pool done at\s+([-\d.]+) ms, spike pool at\s+([-\d.]+) ms", line)) and launches:
            launches[-1]["pool_a_ms"] = float(m[1]); launches[-1]["pool_b_ms"] = float(m[2])
    return launches


def summarise(runs):
    """median over solves of each launch's finish times; spines split into plain and spiked chains"""
    out = []
    for li in range(min(len(r) for r in runs)):
        ls = [r[li] for r in runs]
        l0 = ls[0]
        plain = [max([t for c, sp, t in l["spines"] if not sp], default=0.0) for l in ls]
        spiked = [max([t for c, sp, t in l["spines"] if sp], default=0.0) for l in ls]
        cols_plain = max([c for c, sp, _ in l0["spines"] if not sp], default=0)
        cols_spiked = max([c for c, sp, _ in l0["spines"] if sp], default=0)
        med = lambda v: float(np.median(v))
        row = dict(problems=l0["problems"], WB=l0["WB"], grid=l0["grid"], band_ctas=l0["band_ctas"], spike_ctas=l0["spike_ctas"],
                   plain_chain_columns=cols_plain, spiked_chain_columns=cols_spiked,
                   plain_spines_done_ms=med(plain), spiked_spines_done_ms=med(spiked),
                   pool_a_done_ms=med([l.get("pool_a_ms", 0.0) for l in ls]), pool_b_done_ms=med([l.get("pool_b_ms", 0.0) for l in ls]))
        if cols_plain and row["plain_spines_done_ms"] > 0:
            row["plain_us_per_column"] = 1e3*row["plain_spines_done_ms"]/cols_plain
        if cols_spiked and row["spiked_spines_done_ms"] > 0:
            row["spiked_us_per_column"] = 1e3*row["spiked_spines_done_ms"]/cols_spiked
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C5")
    ap.add_argument("--formulation", default="hybrid")
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--cells", type=int, default=0, help="cells of the reduced solve (0 automatic, -1 plain band)")
    ap.add_argument("--warmup", type=int, default=2, help="LM iterations before anything is timed")
    ap.add_argument("--iters", type=int, default=3, help="LM iterations timed per split, profile off")
    ap.add_argument("--solves", type=int, default=3, help="damped solves profiled per split")
    ap.add_argument("--lam", type=float, default=1e-4)
    ap.add_argument("--ctas", default="0", help="comma-separated band_ctas_per_chain values (0: default split)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("band_bench.py needs a CUDA device")
    ctas = [int(x) for x in a.ctas.split(",") if x.strip()]
    p = synth.make_config(a.config, formulation=a.formulation, seed=a.seed, scale=a.scale)
    s = Solver(p)
    s.set_partition(a.cells)
    s.finalize()
    prm = dict(relative_error_tol=0.0, absolute_error_tol=0.0)
    s.optimize(max_iterations=a.warmup, **prm)
    res = {k: {"band_ctas_per_chain": k} for k in ctas}
    for k in ctas:                                  # ---- profile off: ms_factor per damped solve
        s.set_tuning("band_ctas_per_chain", k)
        s.reset_values()
        s.optimize(max_iterations=1, **prm)         # warm this split
        s.reset_values()
        torch.cuda.synchronize()
        st = s.optimize(max_iterations=a.iters, **prm)
        solves = max(st["inner_iterations"], 1)
        res[k].update(ms_factor_per_solve=st["ms_factor"]/solves, ms_schur_per_solve=st["ms_schur"]/solves,
                      inner_iterations=st["inner_iterations"], lm_iterations=st["iterations"])
    s.set_tuning("band_profile", 1)                 # ---- profile on (process-wide from here)
    s.reset_values()
    s.linearize()
    for k in ctas:
        s.set_tuning("band_ctas_per_chain", k)
        s.solve(a.lam)                              # warm
        runs = []
        for _ in range(a.solves):
            with CaptureStderr() as cap:
                s.solve(a.lam)
                torch.cuda.synchronize()
            runs.append(parse_profile(cap.text))
        res[k]["launches"] = summarise(runs)
    s.set_tuning("band_ctas_per_chain", 0)
    out = dict(config=a.config, scale=a.scale, gpu=gpu_info(), torch_device=torch.cuda.get_device_name(0),
               reduced_dim=s.info()["reduced_dim"], bandwidth=s.info()["bandwidth"], splits=list(res.values()))
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
