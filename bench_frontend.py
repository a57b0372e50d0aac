#!/usr/bin/env python
"""bench_frontend.py -- front-end frames/s at 1242x375 (BASELINE.json second metric, config C4).

Per frame (what FeatureTracker::track does on the hot path, dynosam/src/frontend/vision/FeatureTracker.cc:73-192):
upload flow / instance mask / gray, propogateMask, trackDynamic over the previous dynamic features, sampleDynamic
candidate scan, and pyramidal KLT of the static features (forward 21x21 L3 + backward check L5 as in
StaticFeatureTracker.cc:486-534).  CPU arm (--impl reference): cv2.calcOpticalFlowPyrLK on all host threads plus the
literal numpy restatement of the dense passes on a bounded number of frames.
    python bench_frontend.py [--frames N] [--impl dynoba|reference]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from dynosam_b200.synth_frames import SyntheticStream, W, H  # noqa: E402

N_STATIC, PER_OBJECT = 800, 200          # params/FrontendParams.yaml:50-66


def make_inputs(n_frames, seed=42):
    st = SyntheticStream(n_objects=10, seed=seed)
    rng = np.random.default_rng(seed)
    frames = [st.frame(k) for k in range(n_frames + 1)]
    static_pts = np.stack([rng.uniform(20, W - 20, N_STATIC), rng.uniform(20, H - 20, N_STATIC)], 1).astype(np.float32)
    feats = []
    for k in range(n_frames):
        _, m0, f0 = frames[k]
        kps, labs = [], []
        for lab in range(1, 11):
            ys, xs = np.nonzero(m0 == lab)
            if len(ys) == 0:
                continue
            sel = rng.choice(len(ys), size=min(PER_OBJECT, len(ys)), replace=False)
            kps.append(np.stack([xs[sel] + 0.5 + f0[ys[sel], xs[sel], 0], ys[sel] + 0.5 + f0[ys[sel], xs[sel], 1]], 1))
            labs.append(np.full(len(sel), lab, np.int32))
        kp = np.concatenate(kps) if kps else np.zeros((0, 2)); lab = np.concatenate(labs) if labs else np.zeros(0, np.int32)
        ok = (kp[:, 0] > 1) & (kp[:, 0] < W - 1) & (kp[:, 1] > 1) & (kp[:, 1] < H - 1)
        feats.append((kp[ok], lab[ok], rng.integers(0, 21, ok.sum()).astype(np.int32), np.arange(ok.sum(), dtype=np.int64)))
    return frames, static_pts, feats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="dynoba", choices=["dynoba", "reference"])
    ap.add_argument("--call-by-call", action="store_true", help="round-1 path: every image re-uploaded by every call")
    args = ap.parse_args()
    n = args.frames
    frames, static_pts, feats = make_inputs(max(n, args.warmup) + 1)
    config = {"workload": f"C4: 1242x375 synthetic stream, {n} frames, 10 objects, {N_STATIC} static KLT points (fwd L3 + bwd L5), "
                          f"<= {PER_OBJECT} dynamic features/object", "data": "synthetic"}
    per_frame_bytes = 21*W*H + 2*W*H          # dense passes ~21 B/px (SURVEY 8d) + two gray uploads
    if args.impl == "reference":
        import cv2
        from oracle import frontend_oracle as FO
        nb = min(n, 20); t0 = time.perf_counter()
        for k in range(1, nb + 1):
            g0 = frames[k-1][0]; g1, m1, f1 = frames[k]
            p1, st, _ = FO.klt_track(g0, g1, static_pts, 21, 3, 30, 0.03)
            FO.klt_track(g1, g0, p1, 21, 5, 30, 0.01)
        t_klt = (time.perf_counter() - t0)/nb
        # dense passes: vectorised numpy equivalent of the literal loops (the literal Python loops take minutes/frame)
        t0 = time.perf_counter()
        for k in range(1, nb + 1):
            _, m1, f1 = frames[k]
            ok = (m1 != 0) & (f1[..., 0] != 0) & (f1[..., 1] != 0)
            [np.flatnonzero(ok & (m1 == o)) for o in range(1, 11)]
            kp, lab, age, tid = feats[k-1]
            x = kp[:, 0].astype(int); y = kp[:, 1].astype(int); _ = (m1[y, x] == lab) & (f1[y, x, 0] != 0)
        t_dense = (time.perf_counter() - t0)/nb
        fps = 1.0/(t_klt + t_dense)
        print(json.dumps({"impl": "reference", "metric": "frontend fps at 1242x375", "value": fps, "unit": "frames/s", "n_gpus": 1,
                          "higher_is_better": True, "dtype": "u8/int16/fp32 (OpenCV)", "config": config,
                          "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": os.cpu_count(), "kind": "reference",
                                           "sample": f"{nb} frames: cv2.calcOpticalFlowPyrLK fwd+bwd ({1e3*t_klt:.1f} ms) + numpy dense passes ({1e3*t_dense:.1f} ms)"}}))
        return
    print(json.dumps(run_dynoba(n, args.warmup, streaming=not args.call_by_call)))


def run_dynoba(n, warmup, streaming=True):
    """front-end frames/s through the C ABI (libdynofront) over n frames of the synthetic stream.
    streaming: frames arrive in pinned host buffers, only the NEW frame crosses PCIe (dynofront_next_frame), the previous
    frame's flow / mask / gray pyramid stay on the device, the forward-backward KLT with its checks is one call and the
    propagated mask stays on the device.  Otherwise: the call-by-call path of round 1 (every image re-uploaded per call)."""
    frames, static_pts, feats = make_inputs(max(n, warmup) + 1)
    config = {"workload": f"C4: 1242x375 synthetic stream, {n} frames, 10 objects, {N_STATIC} static KLT points (fwd L3 + bwd L5 + round-trip / label / border checks), "
                          f"<= {PER_OBJECT} dynamic features/object", "data": "synthetic", "mode": "streaming (resident previous frame, pinned uploads)" if streaming else "call by call"}
    import torch  # noqa: F401  (device selection / presence check only)
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    t = FeatureTrackerGPU(W, H); prm = TrackParams()
    static_age = np.zeros(N_STATIC, np.int32)
    if streaming:
        frames = [(np.ascontiguousarray(g, np.uint8), np.ascontiguousarray(m, np.int32), np.ascontiguousarray(f, np.float32)) for g, m, f in frames]
        for g, m, f in frames:
            t.pin(g); t.pin(m); t.pin(f)
        t.next_frame(frames[0][0], frames[0][2], frames[0][1])
        def one(k):
            g1, m1, f1 = frames[k]
            kp, lab, age, tid = feats[k-1]
            t.next_frame(g1, f1, m1)                                   # H2D of the new frame only
            t.propagate_mask_resident(kp, lab, prm)
            acc, *_ = t.track_dynamic(kp, lab, age, tid, prm, 10**6, want_masks=False)
            cand, _ = t.sample_candidates(list(range(1, 11)), prm, capacity=W*H//2)
            p1, st, back, keep = t.klt_track_fb(None, None, static_pts, prm, static_age, 25)
            return t.last_ms, int(acc.sum()), int(keep.sum())
        h2d = W*H*(1 + 8 + 4)
    else:
        def one(k):
            g0 = frames[k-1][0]; _, m0, f0 = frames[k-1]; g1, m1, f1 = frames[k]
            kp, lab, age, tid = feats[k-1]
            cur = t.propagate_mask(kp, lab, m0, f0, m1, prm)
            t.set_frame(f1, cur, None)
            acc, *_ = t.track_dynamic(kp, lab, age, tid, prm, 10**6, want_masks=False)
            cand, _ = t.sample_candidates(list(range(1, 11)), prm, capacity=W*H//2)
            p1, st, _ = t.klt_track(g0, g1, static_pts, 21, 3, 30, 0.03); ms = t.last_ms
            p0, st2, _ = t.klt_track(g1, g0, p1, 21, 5, 30, 0.01)
            return ms + t.last_ms, int(acc.sum()), int(st.sum())
        h2d = W*H*(2*(8 + 4) + 4 + 4)
    for k in range(1, warmup + 1):
        one(k)
    klt_ms = []; t0 = time.perf_counter()
    for k in range(1, n + 1):
        ms, na, ns = one(k); klt_ms.append(ms)
    dt = time.perf_counter() - t0
    fps = n/dt
    dense_bytes = 21*W*H                    # SURVEY 8d: flow 8 + prev mask 4 + cur mask 4 + det mask 1 + scatter 4 per pixel
    out = {"metric": "frontend fps at 1242x375", "value": fps, "unit": "frames/s", "n_gpus": 1, "frames": n, "ms_per_frame": 1e3*dt/n,
           "higher_is_better": True, "dtype": "u8/int16/int32 fixed point + fp32 (OpenCV semantics)", "config": config,
           "klt_device_ms_per_frame": float(np.mean(klt_ms)), "h2d_bytes_per_frame": int(h2d),
           "note": "end to end through the C ABI from host images (H2D/D2H inside the timed region); a frame moves a few MB and "
                   "launches ~40 small kernels, so it is PCIe / launch bound, not HBM bound: the dense passes' 21 B/px "
                   f"({dense_bytes/1e6:.1f} MB) would take {dense_bytes/3.35e12*1e6:.1f} us at the H100 data-sheet HBM rate (3.35 TB/s)"}
    if streaming:
        out.update(full_frame(t, frames, static_pts, feats, n, warmup))
        out.update(static_detection(t, frames, static_pts, n, warmup))
        out.update(depth_stage(t, frames, static_pts, feats, n, warmup))
        out.update(dynamic_klt(t, frames, n, warmup))
    out.update(card())
    return out


def full_frame(t, frames, static_pts, feats, n, warmup):
    """The streaming frame loop again, with sampleDynamic completed on the device (scan + range-tree ANMS + new features,
    dynofront_sample_dynamic) in place of the candidate scan: per object K = 200 - the features track_dynamic kept."""
    from dynosam_b200.frontend import TrackParams
    prm = TrackParams(); static_age = np.zeros(N_STATIC, np.int32); objs = list(range(1, 11))
    t.next_frame(frames[0][0], frames[0][2], frames[0][1])

    def one(k):
        g1, m1, f1 = frames[k]
        kp, lab, age, tid = feats[k-1]
        t.next_frame(g1, f1, m1)
        t.propagate_mask_resident(kp, lab, prm)
        acc, *_ = t.track_dynamic(kp, lab, age, tid, prm, 10**6, want_masks=False)
        num_track = np.bincount(lab[acc.astype(bool)], minlength=11)[1:11].astype(np.int32)
        r = t.sample_dynamic(objs, num_track, prm, 10**6, max_features=PER_OBJECT); sd_ms = t.last_ms
        t.klt_track_fb(None, None, static_pts, prm, static_age, 25)
        return sd_ms, int(r["num_sampled"].sum())
    for k in range(1, warmup + 1):
        one(k)
    sd = []; sampled = []; t0 = time.perf_counter()
    for k in range(1, n + 1):
        ms, s = one(k); sd.append(ms); sampled.append(s)
    dt = time.perf_counter() - t0
    return {"full_frame_fps": n/dt, "sample_dynamic_ms": float(np.mean(sd)), "sampled_per_frame": float(np.mean(sampled)),
            "full_frame_note": "streaming loop with dynofront_sample_dynamic in place of dynofront_sample_candidates; static "
                               "feature detection (dynofront_detect_static) runs on the device but is timed in its own loop "
                               "(detect_static_ms), not in this one"}


def static_detection(t, frames, static_pts, n, warmup):
    """KltFeatureTracker::detectFeatures on the device over the streaming frames: after the forward-backward KLT, the kept
    static tracks are the current features (n_cur = the keep count), as on the reference's trigger path; plus the first-frame
    case n_cur = 0.  detect_static_ms is the device time of one call (CUDA events), detected_per_frame the new features."""
    from dynosam_b200.frontend import DetectParams, TrackParams
    prm = DetectParams(); tprm = TrackParams(); static_age = np.zeros(N_STATIC, np.int32)
    t.next_frame(frames[0][0], frames[0][2], frames[0][1])

    def one(k):
        g1, m1, f1 = frames[k]
        t.next_frame(g1, f1, m1)
        p1, st, back, keep = t.klt_track_fb(None, None, static_pts, tprm, static_age, 25)
        kp, tid, _, _ = t.detect_static(None, p1[keep.astype(bool)], prm, 0)
        return t.last_ms, len(kp)
    for k in range(1, warmup + 1):
        one(k)
    ms, det = [], []
    for k in range(1, n + 1):
        a, b = one(k); ms.append(a); det.append(b)
    first = []
    for k in range(1, min(n, 20) + 1):
        t.detect_static(None, np.zeros((0, 2)), prm, 0); first.append(t.last_ms)
    return {"detect_static_ms": float(np.mean(ms)), "detected_per_frame": float(np.mean(det)),
            "detect_static_first_frame_ms": float(np.mean(first)), "detected_first_frame": len(t.detect_static(None, np.zeros((0, 2)), prm, 0)[0])}


def depth_stage(t, frames, static_pts, feats, n, warmup):
    """Depth and back-projection on the device over the streaming frames (Frame::updateDepths, the per-feature half of
    fillOutputPacketWithTracks, Frame::projectToDenseCloud): after next_frame the frame's depth image (float64, from pinned host
    memory) is uploaded with set_depth, then update_depths runs over the 800 static points and the dynamic features, back_project
    over what it kept (RGB-D right key-points, KITTI-like intrinsics) and dense_cloud over the whole image, its four planar
    outputs copied to the host.  The *_ms keys are the device time of one call (CUDA events, including its copies)."""
    cal, baseline = (718.856, 718.856, 0.0, 607.1928, 185.2157), 0.537
    stream = SyntheticStream(n_objects=10, seed=42)             # the stream make_inputs draws its frames from
    bufs = [np.empty((H, W)), np.empty((H, W))]
    for b in bufs:
        t.pin(b)
    t.next_frame(frames[0][0], frames[0][2], frames[0][1])

    def one(k):
        g1, m1, f1 = frames[k]
        kp, lab, _, _ = feats[k-1]
        buf = bufs[k % 2]; np.copyto(buf, stream.depth(k))    # (the other buffer's copy finished inside the previous frame's calls)
        t.next_frame(g1, f1, m1)
        t.set_depth(buf)
        allkp = np.concatenate([static_pts.astype(np.float64), kp]); alllab = np.concatenate([np.zeros(N_STATIC, np.int32), lab])
        d, v, _, _ = t.update_depths(allkp, alllab); ud = t.last_ms
        r = t.back_project(allkp, d, v, cal, baseline, True); bp = t.last_ms
        nv = t.dense_cloud(cal)[4]
        return ud, bp, t.last_ms, len(allkp), r["m"], nv
    for k in range(1, warmup + 1):
        one(k)
    rows = np.array([one(k) for k in range(1, n + 1)], np.float64)
    for b in bufs:
        t.unpin(b)
    return {"depth_update_ms": float(rows[:, 0].mean()), "back_project_ms": float(rows[:, 1].mean()), "dense_cloud_ms": float(rows[:, 2].mean()),
            "depth_h2d_bytes_per_frame": int(8*W*H), "dense_cloud_d2h_bytes_per_frame": int(W*H*(12 + 3 + 4 + 1)),
            "depth_features_per_frame": float(rows[:, 3].mean()), "measurements_per_frame": float(rows[:, 4].mean()),
            "dense_points_per_frame": float(rows[:, 5].mean())}


def _objects(m):
    """objects_detected and inner bounding boxes (x, y, w, h) of a motion mask: each label's box shrunk by 2 px"""
    objs, bb = [], []
    for oid in range(1, 11):
        ys, xs = np.nonzero(m == oid)
        if len(ys):
            x0, y0, x1, y1 = xs.min(), ys.min(), xs.max(), ys.max()
            objs.append(oid); bb.append((x0 + 2, y0 + 2, max(x1 - x0 - 3, 1), max(y1 - y0 - 3, 1)))
    return objs, np.array(bb, np.int32).reshape(-1, 4)


def dynamic_klt(t, frames, n, warmup):
    """FeatureTracker::trackDynamicKLT + requiresSampling on the device (dynofront_track_dynamic_klt) over the streaming frames, the
    features carried from frame to frame as the reference does; track_dynamic_klt_ms is the device time of one call (CUDA events,
    copies included).  Beside it, on the first frames, the host composition it replaces: dynofront_klt_track for the LK plus the
    test oracle's cv2 / numpy stages (tests/dynamic_klt_oracle.py: per-feature loop, cv2.circle, requiresSampling,
    cv2.goodFeaturesToTrack per sampled object, range-tree ANMS), wall clock on one host thread."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dynamic_klt_oracle as KO
    objs_of = [_objects(m) for _, m, _ in frames]
    empty = (np.zeros((0, 2), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int64))
    t.next_frame(frames[0][0], frames[0][2], frames[0][1])
    state = {"prev": empty, "nid": 0}

    def one(k):
        g1, m1, f1 = frames[k]
        t.next_frame(g1, f1, m1)
        r = t.track_dynamic_klt(None, None, *state["prev"], *objs_of[k], state["nid"], want_masks=False)
        state["prev"] = (r["keypoint"].astype(np.float32), r["label"], r["age"], r["tracklet"]); state["nid"] = r["next_tracklet_id"]
        return t.last_ms, len(r["keypoint"]), int(r["tracked"].sum()), int(r["status"]["sampled"].sum())
    for k in range(1, warmup + 1):
        one(k)
    state["prev"] = empty; state["nid"] = 0
    rows = np.array([one(k) for k in range(1, n + 1)], np.float64)
    # the host composition on the first frames, from the same carried-forward inputs
    nb = min(n, 10); prev = empty; nid = 0; lk_ms = []; host_s = []
    for k in range(1, nb + 1):
        g0 = frames[k - 1][0]; g1, m1, _ = frames[k]; objs, bb = objs_of[k]
        p1, st, _ = t.klt_track(g0, g1, prev[0], 21, 3, 30, 0.03); lk_ms.append(t.last_ms)
        t0 = time.perf_counter()
        r = KO.track_dynamic_klt(g1, m1, None, *prev, p1, st, objs, bb, KO.Params(), nid)
        host_s.append(time.perf_counter() - t0)
        prev = (r["keypoint"].astype(np.float32), r["label"], r["age"], r["tracklet"]); nid = r["next_tracklet_id"]
    return {"track_dynamic_klt_ms": float(rows[:, 0].mean()), "track_dynamic_klt_features_per_frame": float(rows[:, 1].mean()),
            "track_dynamic_klt_tracked_per_frame": float(rows[:, 2].mean()), "track_dynamic_klt_sampled_objects_per_frame": float(rows[:, 3].mean()),
            "track_dynamic_klt_host_composition_ms": float(np.mean(lk_ms) + 1e3*np.mean(host_s)),
            "track_dynamic_klt_host_composition_note": f"{nb} frames: dynofront_klt_track {np.mean(lk_ms):.3f} ms (device) + the oracle's "
                                                       f"cv2 / numpy stages {1e3*np.mean(host_s):.1f} ms (one host thread, Python loops)"}


def card():
    """name and power limit of the GPU the numbers were measured on, read in the same run"""
    import subprocess
    import torch
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        info["power_limit"] = r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        pass
    return info


if __name__ == "__main__":
    main()
