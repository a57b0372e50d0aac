"""Time one window of the sliding-window optimiser on a visual-inertial graph: ingest + finalize, optimize, and the typed
marginal (dynoba_marginal_vars, with its constant f) of the frames the next window keeps.

Settings of the reference's SLIDING_WINDOW mode (RegularBackendModule.cc:50-51): window 10 frames, overlap 4.  The window
is a synthetic visual-inertial problem (synth.make_problem(imu=True)) at the per-frame density of the C1 configuration
(35 static and 15 dynamic tracklets per frame, one object).  Times are host clocks around calls that end in a device
synchronise; each is the median of --repeats runs after one warm-up run, a fresh handle per run.  The card's name and
power limit are read in the same run.  Needs an sm_90 device: without one it fails.

    python tools/window_bench.py [--repeats 5] [--frames 10] [--overlap 4] [--out result.json] [--keep-landmarks]

--keep-landmarks keeps the reference's retained set (isRecentKey, SlidingWindowOptimization.cc:125-130): the pose-like
variables of the last `overlap` frames and the points first observed in them.  The marginal is then
dynoba_marginal_keep_points, and a second window -- the next `frames - overlap` frames' factors, the HessianFactor prior
and the exported LINEAR_PP3 / LINEAR_PPP3 factors -- is optimised too; its time is reported as window2_optimize_ms.
Observations at the new frames of points inserted before the kept frames are left out of the graph, as the reference's
window has no such keys.
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
from dynosam_b200.problem import SLOT_CLASS, FactorBlock, Problem  # noqa: E402


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


def _take(b, m, idx=None):
    return FactorBlock(b.type, b.idx[m] if idx is None else idx, None if b.meas is None else b.meas[m],
                       b.sigma if b.sigma_bcast else b.sigma[m], b.robust_k, None if b.aux_idx is None else b.aux_idx[m])


def _sub(p, blocks, keep):
    """the variables kept by the masks keep[class] (0 pose, 1 point, 3 velocity, 4 bias), blocks re-indexed"""
    new = {c: np.cumsum(m) - 1 for c, m in keep.items()}
    out = []
    for b in blocks:
        idx = b.idx.copy()
        for k, c in enumerate(SLOT_CLASS[b.type]):
            assert keep[c][idx[:, k]].all()         # a window's factors touch only its own variables
            idx[:, k] = new[c][idx[:, k]]
        out.append(FactorBlock(b.type, idx, b.meas, b.sigma, b.robust_k, b.aux_idx))
    return Problem(p.pose[keep[0]], p.point[keep[1]], aux_pose=p.aux_pose, calib=p.calib, blocks=out, pose_order=p.pose_order[keep[0]],
                   vel=p.vel[keep[3]], bias=p.bias[keep[4]], vel_order=p.vel_order[keep[3]], bias_order=p.bias_order[keep[4]])


def two_windows(p, F, overlap):
    """window 1 = the factors of frames < F, window 2 = the rest; kept = frames [F - overlap, F) and their new points"""
    fr = {0: p.pose_order, 3: p.vel_order, 4: p.bias_order}
    frames = lambda b: np.stack([fr[c][b.idx[:, k]] if c in fr else np.full(b.n, -1) for k, c in enumerate(SLOT_CLASS[b.type])], 1).max(1)
    first = np.full(p.n_point, 1 << 30)
    for b in p.blocks:
        if 1 in SLOT_CLASS[b.type]:
            np.minimum.at(first, b.idx[:, SLOT_CLASS[b.type].index(1)], frames(b))
    w1, w2 = [], []
    for b in p.blocks:
        f = frames(b)
        drop = (first[b.idx[:, SLOT_CLASS[b.type].index(1)]] < F - overlap) & (f >= F) if 1 in SLOT_CLASS[b.type] else np.zeros(b.n, bool)
        if (f < F).any(): w1.append(_take(b, f < F))
        if ((f >= F) & ~drop).any(): w2.append(_take(b, (f >= F) & ~drop))
    K1 = {c: fr[c] < F for c in fr}; K1[1] = first < F
    K2 = {c: fr[c] >= F - overlap for c in fr}; K2[1] = (first >= F - overlap) & (first < (1 << 30))
    pa = _sub(p, w1, K1)
    pa.meta = dict(n_frames=F)
    kinds, idx = kept_set(pa, overlap)
    pts = np.flatnonzero(first[K1[1]] >= F - overlap).astype(np.int32)
    return pa, kinds, idx, pts, w2, K1, K2


def window2(p, w2, K1, K2, kinds, idx, G, g, f, blocks):
    """the second window: its own factors, the HessianFactor prior and the exported factors, in its own indices"""
    w1_of = {c: np.flatnonzero(m) for c, m in K1.items()}
    lin = []
    for b in blocks:
        jidx = b.idx.copy()
        for k, c in enumerate(SLOT_CLASS[b.type]):
            jidx[:, k] = w1_of[c][b.idx[:, k]]
        lin.append(FactorBlock(b.type, jidx, b.meas, b.sigma))
    pb = _sub(p, w2 + lin, K2)
    new = {c: np.cumsum(m) - 1 for c, m in K2.items()}
    kc = {POSE6: 0, VEL3: 3, BIAS6: 4}
    idx_b = np.array([new[kc[k]][w1_of[kc[k]][i]] for k, i in zip(kinds, idx)], np.int32)
    lp = np.concatenate([(pb.pose, None, None, pb.vel, pb.bias)[kc[k]][i] for k, i in zip(kinds, idx_b)])
    pb.linear_priors = [dict(kind=kinds, idx=idx_b, lin=lp, G=G, g=g, f=f)]
    return pb


def keep_run(p, pa, kinds, idx, pts, w2, K1, K2):
    s = Solver(pa)
    s.finalize()
    s.optimize()
    t0 = time.perf_counter()
    G, g, f, blocks = s.marginal_keep_points(kinds, idx, pts)   # returns after the host has the marginal and the factors
    t1 = time.perf_counter()
    s.close()
    pb = window2(p, w2, K1, K2, kinds, idx, G, g, f, blocks)
    s2 = Solver(pb)
    s2.finalize()
    t2 = time.perf_counter()
    st = s2.optimize()
    t3 = time.perf_counter()
    s2.close()
    return dict(marginal_ms=1e3*(t1 - t0), window2_optimize_ms=1e3*(t3 - t2), window2_optimize_device_ms=st["ms_total"],
                exported_factors=int(sum(b.n for b in blocks)), kept_points=int(pts.size), window2_iterations=st["iterations"],
                window2_error_initial=st["error_initial"], window2_error_final=st["error_final"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--overlap", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=21)
    ap.add_argument("--out", default=None)
    ap.add_argument("--keep-landmarks", action="store_true")
    a = ap.parse_args()
    if a.keep_landmarks:
        F2 = 2*a.frames - a.overlap                 # two windows of `frames` frames sharing `overlap`
        p = synth.make_problem(n_frames=F2, n_objects=1, n_static=35*F2, n_dynamic=15*F2, seed=a.seed, imu=True)
        pa, kinds, idx, pts, w2, K1, K2 = two_windows(p, a.frames, a.overlap)
        keep_run(p, pa, kinds, idx, pts, w2, K1, K2)            # warm-up
        runs = [keep_run(p, pa, kinds, idx, pts, w2, K1, K2) for _ in range(a.repeats)]
        med = {k: float(np.median([r[k] for r in runs])) for k in ("marginal_ms", "window2_optimize_ms", "window2_optimize_device_ms")}
        spread = {k + "_range": [float(min(r[k] for r in runs)), float(max(r[k] for r in runs))] for k in ("marginal_ms", "window2_optimize_ms")}
        name, power = card()
        res = dict(tool="window_bench", mode="keep_landmarks", card=name, power_limit=power, frames=a.frames, overlap=a.overlap,
                   repeats=a.repeats, **{k: runs[-1][k] for k in ("exported_factors", "kept_points", "window2_iterations",
                                                                  "window2_error_initial", "window2_error_final")}, **med, **spread)
        line = json.dumps(res)
        print(line)
        if a.out:
            with open(a.out, "w") as fh:
                fh.write(line + "\n")
        return
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
