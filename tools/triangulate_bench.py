"""Time dynoba_triangulate_batch (one warp per problem) and the builder's STEREO_PROJECTION finalize on the GPU.

Workloads:
  (a) C5-shaped problems: 1 M static landmarks with synth.py's track ages (2 to 15 frames) on a 10 000-frame trajectory,
      one problem per landmark over its whole track (left and right camera per frame, 5 % right key-points missing).
      The whole call (copies, one launch, synchronise) by a host clock after a warm-up, the kernel alone by torch.profiler
      in a separate call, and the host build of triangulate.cuh on one CPU thread over the first --host-problems problems.
  (b) builder finalize at --frames frames / --landmarks static landmarks: point-to-point (add_static) against stereo with the
      triangulation rounds on the device and on the host build.
The card name, power limit and maximum SM clock are read in the same run.  Prints one JSON line (and writes it to --out).

    python tools/triangulate_bench.py [--landmarks-c5 1000000] [--out results.json]
"""
import argparse
import ctypes as C
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--landmarks-c5", type=int, default=1_000_000)
    ap.add_argument("--frames-c5", type=int, default=10_000)
    ap.add_argument("--host-problems", type=int, default=20_000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--landmarks", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from dynosam_b200 import binding as B
    from dynosam_b200 import lie, synth, synth_stereo
    from dynosam_b200.builder import GraphBuilder
    import test_triangulate as TT
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True)
    if card.returncode != 0:
        raise SystemExit("no CUDA device: triangulate_bench measures the GPU only")
    res = dict(card=card.stdout.strip().splitlines()[0])
    L = B.load()

    # (a) C5-shaped batch
    N = a.frames_c5
    xi = np.array([0.0, 0.004, 0.0, 0.02, 0.0, 1.0])
    X = lie.se3_exp(np.arange(N)[:, None]*xi[None])
    st = synth_stereo.make_static_stereo(X, a.landmarks_c5, seed=1, nan_right=0.05, outlier_fraction=0.01)
    off, poses, kp, cal = synth_stereo.full_track_problems(X, st)
    n = off.size - 1
    arr = dict(off=off, poses=poses, kp=kp, calib=cal, point=np.zeros((n, 3)), status=np.zeros(n, np.int32),
               reproj=np.zeros(n), sv=np.zeros((n, 4)))
    res.update(problems=int(n), cameras=int(off[-1]))
    assert B.triangulate_call(L.dynoba_triangulate_batch, arr, 1.0, 3.0, 0) == 0           # warm-up (workspace, module)
    wall = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        assert B.triangulate_call(L.dynoba_triangulate_batch, arr, 1.0, 3.0, 0) == 0
        wall.append(time.perf_counter() - t0)
    res["call_ms"] = [round(1e3*w, 2) for w in sorted(wall)]
    res["status_counts"] = np.bincount(arr["status"], minlength=4).tolist()
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        B.triangulate_call(L.dynoba_triangulate_batch, arr, 1.0, 3.0, 0)
        torch.cuda.synchronize()
    res["kernel_ms"] = round(sum(e.device_time_total for e in prof.key_averages() if "triangulate_kernel" in e.key)/1e3, 3)
    with tempfile.TemporaryDirectory() as tmp:
        import pathlib
        shim = TT.build_shim(pathlib.Path(tmp))
        m = min(a.host_problems, n)
        sub = dict(arr, off=off[:m + 1], point=np.zeros((m, 3)), status=np.zeros(m, np.int32), reproj=np.zeros(m), sv=np.zeros((m, 4)))
        t0 = time.perf_counter()
        B.triangulate_call(shim.host_triangulate_batch, sub, 1.0, 3.0)
        res["host_1thread_ms"] = round(1e3*(time.perf_counter() - t0), 1)
        res["host_problems"] = m
        res["host_equals_device"] = bool(all(np.array_equal(sub[k], arr[k][:m], equal_nan=True) for k in ("status", "point", "reproj", "sv")))

    # (b) builder finalize: point-to-point against stereo (device, host build)
    p, sst = synth_stereo.make_scene(n_frames=a.frames, n_static=a.landmarks, seed=3, nan_right=0.05)
    pts = sst["points"]
    fin = {}
    for mode in ("ptp", "stereo_device", "stereo_host"):
        b = GraphBuilder()
        if mode != "ptp":
            b.set_static_stereo(synth.KITTI_K, 1.0, 0 if mode == "stereo_device" else -1)
        for k in range(a.frames):
            b.add_frame(k, p.pose[k], None if k == 0 else p.pose[k])
            sel = np.flatnonzero(sst["frame"] == k)
            if mode == "ptp":
                z = lie.transform_to(np.repeat(p.meta["gt_camera"][k][None], sel.size, 0), pts[sst["tracklet"][sel]])
                b.add_static(k, sst["tracklet"][sel], z)
            else:
                b.add_static_stereo(k, sst["tracklet"][sel], sst["stereo"][sel])
        t0 = time.perf_counter()
        assert L.dynoba_builder_finalize(b.h) == 0
        fin[mode] = round(1e3*(time.perf_counter() - t0), 1)
        if mode != "ptp":
            fin[mode + "_stats"] = b.static_stereo_stats()
        b.close()
    res["builder_finalize_ms"] = fin
    res["builder_frames"], res["builder_landmarks"] = a.frames, a.landmarks
    line = json.dumps(res)
    print(line)
    if a.out:
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
