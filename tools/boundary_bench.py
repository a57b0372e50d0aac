"""Time dynofront_object_boundary (computeObjectMaskBoundaryMask on the resident motion mask) on the GPU.

Per frame size (the reference's dataset sizes of tests/frame_cases.py and 1920 x 1080, SyntheticStream masks at the reference's
scaled thickness): the call's device time (CUDA events around its two kernels and the table reset), its wall clock (host clock
around the C call, the table download and the stream synchronise included), and the literal cv2 composition of
tests/boundary_oracle.py on this host's CPU with 1 thread and with cv2's default thread count.  Then the C4 streaming loop of
bench_frontend.py (next_frame, propagate_mask, track_dynamic, sample_candidates, klt_track_fb) in frames/s three ways: without a
boundary mask, with object_boundary after next_frame, and with the cv2 mask computed on the host and uploaded through next_frame.
The three loops alternate over --rounds rounds, so the spread shows.  Card name and power limit are read in the same run.

    python tools/boundary_bench.py [--reps 200] [--frames 200] [--rounds 3] [--out results.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def size_row(w, h, reps, n_objects=10):
    import cv2
    import boundary_oracle as BO
    import frame_cases as FC
    from dynosam_b200.frontend import FeatureTrackerGPU
    case = FC.Case(f"{w}x{h}", w, h, ())
    masks = [FC.frame(case, k, n_objects=n_objects)[1] for k in range(4)]
    t = BO.thickness(w, h)
    tr = FeatureTrackerGPU(w, h)
    flow = np.zeros((h, w, 2), np.float32)
    dev_ms, wall_ms = [], []
    for i in range(reps + 20):
        tr.set_frame(flow, masks[i % 4], None)
        t0 = time.perf_counter()
        objs, bb, ib, _ = tr.object_boundary(-1)
        t1 = time.perf_counter()
        if i >= 20:
            dev_ms.append(tr.last_ms); wall_ms.append(1e3*(t1 - t0))
    got = tr.object_boundary(-1, want_mask=True)
    ref = BO.object_boundary(masks[3], t)
    same = all(np.array_equal(a, b) for a, b in zip(got, ref))
    tr.close()
    cpu = {}
    default_threads = cv2.getNumThreads()
    for label, n in (("1_thread", 1), ("default_threads", default_threads)):
        cv2.setNumThreads(n)
        ts = []
        for i in range(max(5, min(30, reps//5)) + 2):
            t0 = time.perf_counter(); BO.object_boundary(masks[i % 4], t); ts.append(1e3*(time.perf_counter() - t0))
        cpu[label] = float(np.median(ts[2:]))
    cv2.setNumThreads(default_threads)
    return {"size": f"{w}x{h}", "thickness": t, "objects": int(len(objs)), "device_ms_median": float(np.median(dev_ms)),
            "wall_ms_median": float(np.median(wall_ms)), "wall_ms_p90": float(np.percentile(wall_ms, 90)),
            "cv2_ms_median_1_thread": cpu["1_thread"], "cv2_ms_median_default_threads": cpu["default_threads"],
            "cv2_default_threads": int(default_threads), "bit_identical_to_cv2": bool(same)}


def stream_loops(n, rounds):
    import bench_frontend as BF
    import boundary_oracle as BO
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    W, H = BF.W, BF.H
    frames, static_pts, feats = BF.make_inputs(n + 1)
    frames = [(np.ascontiguousarray(g, np.uint8), np.ascontiguousarray(m, np.int32), np.ascontiguousarray(f, np.float32)) for g, m, f in frames]
    t = FeatureTrackerGPU(W, H); prm = TrackParams()
    for g, m, f in frames:
        t.pin(g); t.pin(m); t.pin(f)
    static_age = np.zeros(len(static_pts), np.int32)
    thick = BO.thickness(W, H)

    def loop(mode):
        t.next_frame(frames[0][0], frames[0][2], frames[0][1])
        t0 = time.perf_counter()
        for k in range(1, n + 1):
            g1, m1, f1 = frames[k]
            kp, lab, age, tid = feats[k - 1]
            if mode == "host_mask":
                t.next_frame(g1, f1, m1, BO.object_boundary(m1, thick)[3])
            else:
                t.next_frame(g1, f1, m1)
            if mode == "device":
                t.object_boundary(-1)
            t.propagate_mask_resident(kp, lab, prm)
            t.track_dynamic(kp, lab, age, tid, prm, 10**6, want_masks=False)
            t.sample_candidates(list(range(1, 11)), prm, capacity=W*H//2)
            t.klt_track_fb(None, None, static_pts, prm, static_age, 25)
        return n/(time.perf_counter() - t0)

    modes = ("none", "device", "host_mask")
    for mode in modes:                                  # warm-up of every path
        loop(mode)
    fps = {m: [] for m in modes}
    for _ in range(rounds):
        for mode in modes:
            fps[mode].append(loop(mode))
    return {"c4_frames": n, "c4_fps_without_boundary": fps["none"], "c4_fps_with_object_boundary": fps["device"],
            "c4_fps_with_host_cv2_mask_uploaded": fps["host_mask"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: boundary_bench measures the GPU only")
    import bench_frontend as BF
    import frame_cases as FC
    info = BF.card()
    rows = []
    for name in FC.DATASET:
        c = FC.CASES[name]
        rows.append(size_row(c.w, c.h, a.reps))
        print(json.dumps(rows[-1]), flush=True)
    for n_obj in (5, 20):
        rows.append(dict(size_row(1920, 1080, a.reps, n_obj), n_objects_generated=n_obj))
        print(json.dumps(rows[-1]), flush=True)
    loops = stream_loops(a.frames, a.rounds)
    print(json.dumps(loops), flush=True)
    res = {"card": info, "sizes": rows, "stream": loops}
    print(json.dumps({"card": info}), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
