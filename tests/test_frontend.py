"""Front-end rows a13 (dense-flow track / sample scan / mask propagation) and a14 (pyramidal KLT).

Bar (north_star): bit-exact on track / association indices (accept flags, ages, tracklet ids, labels, masks, candidate
index sets, KLT status flags); KLT sub-pixel positions within 1e-2 px of cv2 (OpenCV accumulates the 21x21 sums in
float with a SIMD lane order we do not replicate; our sums are exact integers).
"""
import os
import re
import shlex
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from dynosam_b200.synth_frames import SyntheticStream

W, H = 1242, 375
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dynosam_b200", "frontend_csrc")


def _features_from_mask(rng, mask, flow, per_object=200, jitter=True):
    """Previous-frame dynamic features: sampled on the objects of frame k-1, predicted key-point = kp + flow."""
    kps, labs = [], []
    for lab in np.unique(mask):
        if lab == 0:
            continue
        ys, xs = np.nonzero(mask == lab)
        sel = rng.choice(len(ys), size=min(per_object, len(ys)), replace=False)
        for y, x in zip(ys[sel], xs[sel]):
            kx = x + (rng.uniform(0, 0.9) if jitter else 0.0); ky = y + (rng.uniform(0, 0.9) if jitter else 0.0)
            kps.append((kx + flow[y, x, 0], ky + flow[y, x, 1])); labs.append(lab)
    kps = np.array(kps); labs = np.array(labs, dtype=np.int32)
    keep = (kps[:, 0] > 1) & (kps[:, 0] < W - 1) & (kps[:, 1] > 1) & (kps[:, 1] < H - 1)
    return kps[keep], labs[keep]


def test_filled_circle_stencil_matches_opencv():
    """The per-row half widths the kernels use reproduce cv::circle(..., FILLED) for every radius we accept."""
    import cv2
    for r in range(0, 16):
        # same midpoint recurrence as frontend.cu::make_disc
        hw = [-1]*16
        err, dx, dy, plus, minus = 0, r, 0, 1, (r << 1) - 1
        while dx >= dy:
            hw[dy] = max(hw[dy], dx); hw[dx] = max(hw[dx], dy)
            dy += 1; err += plus; plus += 2
            m = -1 if err > 0 else 0
            err -= minus & m; dx += m; minus -= m & 2
        img = np.zeros((41, 41), np.uint8); cv2.circle(img, (20, 20), r, 255, cv2.FILLED)
        ref = np.zeros_like(img)
        for ddy in range(-r, r + 1):
            w = hw[abs(ddy)]
            ref[20 + ddy, 20 - w:20 + w + 1] = 255
        assert np.array_equal(img, ref), r


def test_frontend_oracle_sequential_semantics():
    """Oracle self-checks: suppression by earlier accepted features and tracklet renewal order."""
    from oracle import frontend_oracle as FO
    mask = np.zeros((40, 60), np.int32); mask[5:35, 5:55] = 3
    flow = np.zeros((40, 60, 2), np.float32); flow[..., 0] = 1.5; flow[..., 1] = 0.5
    kp = np.array([[10.2, 10.1], [11.0, 10.9], [20.5, 20.5], [30.0, 12.0]])
    acc, pk, fl, age, tid, lab, nid, det, trk = FO.track_dynamic(kp, [3, 3, 3, 3], [1, 2, 20, 5], [100, 101, 102, 103], flow, mask, None,
                                                                 FO.TrackParams(), 500)
    assert list(acc) == [1, 0, 1, 1]                      # second feature sits inside the first one's circle
    assert list(tid) == [100, 0, 500, 103] and nid == 501  # age 21 > 20 -> new tracklet id, age reset
    assert list(age) == [2, 0, 0, 6]
    assert det[10, 10] == 0 and trk[10, 10] == 3 and det[0, 0] == 255


def test_c_abi_frontend_exports():
    import os
    import __graft_entry__ as g
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(os.path.join(root, "dynosam_b200", "libdynofront.so")):
        g.build()
    from dynosam_b200 import frontend
    lib = frontend.load()
    for s in frontend.EXPORTS:
        assert hasattr(lib, s), s


def test_frontend_kernels_compile_without_spills():
    """Every kernel of libdynofront, compiled with the Makefile's code-generation flags, keeps its values in registers:
    ptxas reports 0 bytes of spill stores and loads (a stack frame alone, such as a local patch array, is not a spill)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not available")
    with open(os.path.join(CSRC, "Makefile")) as f:
        flags = shlex.split(re.search(r"^NVFLAGS\s*:=(.*)$", f.read(), re.M).group(1))
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, *flags, "-Xptxas", "-v", "-cubin", "-o", os.path.join(d, "f.cubin"), os.path.join(CSRC, "frontend.cu")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    props = re.findall(r"Function properties for (\S+)\n\s+\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) >= 30, len(props)
    spills = [(name, int(st), int(ld)) for name, st, ld in props if int(st) or int(ld)]
    assert not spills, spills


# ------------------------------------------------------------------------------------------------ GPU parity
@pytest.mark.gpu
@pytest.mark.parametrize("with_det,min_dist", [(False, 2), (True, 3), (True, 0)])
def test_track_dynamic_bit_exact(with_det, min_dist):
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(1)
    st = SyntheticStream(n_objects=10, seed=7)
    _, m0, f0 = st.frame(4); _, m1, f1 = st.frame(5)
    f1[100:140, 300:360] = 0.0                              # exact-zero flow region (skipped features)
    kp, lab = _features_from_mask(rng, m0, f0, per_object=400)
    age = rng.integers(0, 22, len(lab)).astype(np.int32); tid = np.arange(1000, 1000 + len(lab), dtype=np.int64)
    det = None
    if with_det:
        det = np.full((H, W), 255, np.uint8); det[:, 500:520] = 0; det[150:160, :] = 0
    prm = TrackParams(max_dynamic_feature_age=20, min_distance=min_dist)
    t = FeatureTrackerGPU(W, H); t.set_frame(f1, m1, det)
    a, pk, fl, oa, ot, ol, nid, dm, tm = t.track_dynamic(kp, lab, age, tid, prm, 5000)
    ra, rpk, rfl, roa, rot, rol, rnid, rdm, rtm = FO.track_dynamic(kp, lab, age, tid, f1, m1, det, FO.TrackParams(20, min_dist, 0, 0), 5000)
    assert 0 < ra.sum() < len(ra)
    assert np.array_equal(a, ra) and np.array_equal(oa, roa) and np.array_equal(ot, rot) and np.array_equal(ol, rol) and nid == rnid
    assert np.array_equal(pk, rpk) and np.array_equal(fl, rfl)          # fp32 -> fp64 adds are exact on both sides
    assert np.array_equal(dm, rdm) and np.array_equal(tm, rtm)


@pytest.mark.gpu
def test_growing_feature_count_reuses_device_memory():
    """A stream whose feature count creeps upward: each growth of the scratch buffers frees the old ones, so the device's
    free memory falls by about the final buffers (~30 MB at 300 000 features), not by every size seen on the way."""
    import torch
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    rng = np.random.default_rng(8)
    _, m, f = SyntheticStream(n_objects=4, seed=1).frame(1)
    t = FeatureTrackerGPU(W, H); t.set_frame(f, m, None)

    def call(n):
        kp = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
        t.track_dynamic(kp, np.zeros(n, np.int32), np.zeros(n, np.int32), np.arange(n, dtype=np.int64), TrackParams(), 0, want_masks=False)
    call(100)                                                 # module load and the first buffers
    torch.cuda.synchronize(); free0, _ = torch.cuda.mem_get_info()
    for n in np.linspace(4097, 300000, 64).astype(int):
        call(int(n))
    torch.cuda.synchronize(); free1, _ = torch.cuda.mem_get_info()
    t.close()
    assert free0 - free1 < 200e6, (free0 - free1)/1e6


@pytest.mark.gpu
def test_sample_candidates_sets():
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    from oracle import frontend_oracle as FO
    st = SyntheticStream(n_objects=6, seed=3)
    _, m1, f1 = st.frame(2)
    f1[50:80, 200:260] = 0.0
    det = np.full((H, W), 255, np.uint8); det[::7, :] = 0
    small = (slice(0, 200), slice(100, 500))                     # the literal Python oracle is slow: crop
    m = np.ascontiguousarray(m1[small]); f = np.ascontiguousarray(f1[small]); d = np.ascontiguousarray(det[small])
    hh, ww = m.shape
    objs = [int(o) for o in np.unique(m) if o != 0][:4] + [99]
    t = FeatureTrackerGPU(ww, hh); t.set_frame(f, m, d)
    prm = TrackParams(shrink_row=3, shrink_col=5)
    cand, zero = t.sample_candidates(objs, prm)
    rc, rz = FO.sample_dynamic_candidates(f, m, d, objs, FO.TrackParams(20, 2, 3, 5))
    for o in objs:
        assert np.array_equal(cand[o], np.array(rc[o], dtype=np.int32)), o      # ascending pixel order on both sides
        assert zero[o] == rz[o]
    assert sum(len(v) for v in cand.values()) > 0


@pytest.mark.gpu
def test_propagate_mask_bit_exact():
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(5)
    st = SyntheticStream(n_objects=5, seed=11, width=400, height=200)
    _, m0, f0 = st.frame(3); _, m1, _ = st.frame(4)
    cur = m1.copy()
    labs = [int(l) for l in np.unique(m0) if l != 0]
    cur[cur == labs[0]] = 0                                   # the detector lost the first object in the current frame
    if len(labs) > 1:
        cur[cur == labs[1]] = 0
    kps, lab = [], []
    for l in labs:
        ys, xs = np.nonzero(m0 == l)
        sel = rng.choice(len(ys), size=min(220, len(ys)), replace=False)
        kps += [(x + 0.3 + f0[y, x, 0], y + 0.4 + f0[y, x, 1]) for y, x in zip(ys[sel], xs[sel])]; lab += [l]*len(sel)
    kps = np.array(kps); lab = np.array(lab, dtype=np.int32)
    ok = (kps[:, 0] > 1) & (kps[:, 0] < 399) & (kps[:, 1] > 1) & (kps[:, 1] < 199)
    kps, lab = kps[ok], lab[ok]
    t = FeatureTrackerGPU(400, 200)
    out = t.propagate_mask(kps, lab, m0, f0, cur, TrackParams())
    ref = FO.propagate_mask(kps, lab, m0, f0, cur, FO.TrackParams())
    assert np.array_equal(out, ref)
    assert (out != cur).sum() > 0


@pytest.mark.gpu
def test_pyramid_and_scharr_bit_exact():
    import cv2
    from dynosam_b200.frontend import FeatureTrackerGPU
    st = SyntheticStream(n_objects=4, seed=2)
    g0, _, _ = st.frame(0); g1, _, _ = st.frame(1)
    t = FeatureTrackerGPU(W, H)
    t.klt_track(g0, g1, np.array([[100.0, 100.0]], np.float32))
    ref = g0
    for lvl in range(4):
        img, der = t.pyramid_level(0, lvl)
        assert np.array_equal(img, ref), lvl
        # calcSharrDeriv == Scharr with BORDER_REFLECT_101, unnormalised, int16
        dx = cv2.Scharr(ref, cv2.CV_16S, 1, 0, borderType=cv2.BORDER_REFLECT_101)
        dy = cv2.Scharr(ref, cv2.CV_16S, 0, 1, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(der[..., 0], dx) and np.array_equal(der[..., 1], dy), lvl
        ref = cv2.pyrDown(ref)


@pytest.mark.gpu
@pytest.mark.parametrize("max_level,initial", [(3, False), (5, False), (3, True)])
def test_klt_matches_opencv(max_level, initial):
    from dynosam_b200.frontend import FeatureTrackerGPU
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(9)
    st = SyntheticStream(n_objects=10, seed=42)
    g0, _, _ = st.frame(10); g1, _, _ = st.frame(11)
    n = 1000
    pts = np.stack([rng.uniform(-5, W + 5, n), rng.uniform(-5, H + 5, n)], 1).astype(np.float32)     # includes border cases
    pts[:50] = np.stack([rng.uniform(0, 12, 50), rng.uniform(0, H, 50)], 1)                        # windows hanging over the edge
    init = (pts + rng.normal(0, 1.0, pts.shape)).astype(np.float32) if initial else None
    t = FeatureTrackerGPU(W, H)
    nxt, stt, err = t.klt_track(g0, g1, pts, win=21, max_level=max_level, max_count=30, eps=0.03, initial=init)
    rn, rs, re = FO.klt_track(g0, g1, pts, 21, max_level, 30, 0.03, init)
    agree = stt == rs
    # status flags: bit-exact except where cv2's float accumulation (its 21x21 sums run in fp32 SIMD lanes, ours are exact
    # integers) lands on the other side of a threshold.  The one tolerated deviation, proven per point: a mismatching point
    # has its level-0 min eigenvalue within fp32 accumulation error of minEigThreshold (the error of a 441-term fp32 sum
    # relative to the matrix trace), or both sides agree that it is tracked but the final position left the image by a
    # sub-pixel amount (positions differ by < 1e-2 px).
    assert agree.mean() >= 0.998, agree.mean()
    eig = t.klt_last_min_eig(n)
    for i in np.flatnonzero(~agree):
        near_threshold = abs(float(eig[i, 0]) - 1e-4) <= 441*2.0**-24*max(float(eig[i, 1]), 1e-4)
        x, y = (rn[i] if rs[i] else nxt[i])
        at_border = min(x, y, W - 1 - x, H - 1 - y) < 22 + 1e-2
        assert near_threshold or at_border, (i, eig[i], stt[i], rs[i], nxt[i], rn[i])
    both = (stt == 1) & (rs == 1)
    d = np.abs(nxt[both] - rn[both]).max(axis=1)
    assert np.percentile(d, 99) < 1e-2 and np.median(d) < 1e-3, (np.percentile(d, 99), np.median(d))
    assert np.abs(err[both] - re[both]).max() < 0.5


def _static_inputs(rng, st_k, n_prev=1500, n_det=2500):
    _, mask, flow = st_k
    kp = np.stack([rng.uniform(-3, W + 3, n_prev), rng.uniform(-3, H + 3, n_prev)], 1)      # some outside the image
    kp[:200] = kp[200:400] + rng.uniform(-1.5, 1.5, (200, 2))                               # several features per grid cell
    age = rng.integers(0, 30, n_prev).astype(np.int32)
    usable = (rng.uniform(0, 1, n_prev) > 0.1).astype(np.uint8)
    det = np.stack([rng.integers(0, W, n_det), rng.integers(0, H, n_det)], 1).astype(np.int32)
    return kp, age, usable, det, mask, flow


def test_static_flow_oracle_first_come_per_cell():
    """Oracle self-check: of two usable background features in one grid cell the first in iteration order wins; a feature
    that fails a check does not occupy its cell; detections only fill free cells and stop at max_features."""
    from oracle import frontend_oracle as FO
    mask = np.zeros((60, 90), np.int32); mask[:, 60:] = 2
    flow = np.zeros((60, 90, 2), np.float32); flow[..., 0] = 1.25; flow[..., 1] = -0.5
    flow[10, 10] = (0.0, 1.0)                                        # zero x-flow at (10, 10): constructStaticFeature fails
    kp = np.array([[10.4, 10.2], [12.0, 11.0], [13.0, 12.0], [70.0, 5.0], [31.0, 31.0]])
    r = FO.track_static_flow(kp, [3, 4, 5, 6, 7], [1, 1, 1, 1, 0], [(12, 12), (40, 40), (41, 41), (50, 10), (20, 50)], flow, mask, 15, 4, 100)
    assert list(r["acc"]) == [0, 1, 0, 0, 0]           # 0: zero flow (cell stays free), 1 takes cell 0, 2 same cell, 3 on object, 4 unusable
    assert list(r["age"]) == [0, 5, 0, 0, 0]
    assert list(r["det_acc"]) == [0, 1, 0, 1, 1] and list(r["det_tracklet"]) == [0, 100, 0, 101, 102]   # (12,12) occupied, (41,41) same cell as (40,40)
    assert r["next_tracklet_id"] == 103 and r["n_tracked"] == 1 and r["n_detected"] == 3


@pytest.mark.gpu
@pytest.mark.parametrize("max_features", [400, 900, 3000])
def test_track_static_flow_bit_exact(max_features):
    """ExternalFlowFeatureTracker::trackStatic on the device: accept flags, ages, flows, predicted key-points and the new
    tracklet ids equal the literal loops, with and without the max_features cut."""
    from dynosam_b200.frontend import FeatureTrackerGPU
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(21)
    stream = SyntheticStream(n_objects=10, seed=42)
    kp, age, usable, det, mask, flow = _static_inputs(rng, stream.frame(7))
    flow = flow.copy(); flow[::7, ::5, 0] = 0.0                      # exact zeros in the flow field
    t = FeatureTrackerGPU(W, H); t.set_frame(flow, mask, None)
    g = t.track_static_flow(kp, age, usable, det, 15, max_features, 5000)
    o = FO.track_static_flow(kp, age, usable, det, flow, mask, 15, max_features, 5000)
    for k in ("acc", "age", "det_acc", "det_tracklet"):
        assert np.array_equal(g[k], o[k]), k
    for k in ("flow", "pred", "det_flow", "det_pred"):
        assert np.array_equal(g[k], o[k]), k                          # doubles formed from the same floats: bit-exact
    assert (g["next_tracklet_id"], g["n_tracked"], g["n_detected"]) == (o["next_tracklet_id"], o["n_tracked"], o["n_detected"])
    assert g["n_tracked"] > 100 and (g["n_detected"] == 0 if max_features == 400 else g["n_detected"] > 100)   # 767 tracked: the 400 cut admits no detection


@pytest.mark.gpu
@pytest.mark.parametrize("initial", [False, True])
def test_klt_forward_backward_on_device(initial):
    """KltFeatureTracker::trackPoints as one device call: the forward-backward status and the label / border / age checks
    agree with cv2 + the literal checks wherever the two LK passes themselves agree (see test_klt_matches_opencv for the
    one tolerated deviation of the LK status)."""
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(4)
    stream = SyntheticStream(n_objects=10, seed=42)
    g0, _, _ = stream.frame(20); g1, m1, f1 = stream.frame(21)
    n = 800
    pts = np.stack([rng.uniform(5, W - 5, n), rng.uniform(5, H - 5, n)], 1).astype(np.float32)
    age = rng.integers(0, 30, n).astype(np.int32)
    init = (pts + rng.normal(0, 0.7, pts.shape)).astype(np.float32) if initial else None
    prm = TrackParams(shrink_row=20, shrink_col=20)
    t = FeatureTrackerGPU(W, H); t.set_frame(f1, m1, None)
    nxt, stt, back, keep = t.klt_track_fb(g0, g1, pts, prm, age, 25, initial=init)
    fprm = FO.TrackParams(shrink_row=20, shrink_col=20)
    rn, rs, rb, rk = FO.klt_track_fb(g0, g1, pts, m1, age, 25, fprm, initial=init)
    agree = stt == rs
    assert agree.mean() >= 0.99, agree.mean()
    both = (stt == 1) & (rs == 1)
    assert np.percentile(np.abs(nxt[both] - rn[both]).max(axis=1), 99) < 1e-2
    # the per-point checks are integer logic on the truncated key-point: identical wherever the key-points truncate alike
    same_px = both & (nxt.astype(np.float64).astype(np.int64) == rn.astype(np.float64).astype(np.int64)).all(axis=1)
    assert same_px.sum() > 0.8*both.sum()
    assert np.array_equal(keep[same_px], rk[same_px])
    assert 0 < keep.sum() < stt.sum()                                # the checks removed something and kept something
    assert t.last_counts == (int(stt.sum()), int(keep.sum()))


@pytest.mark.gpu
def test_streaming_mode_equals_call_by_call():
    """dynofront_next_frame keeps the previous frame on the device (buffers swap roles, only the new frame is uploaded):
    mask propagation, dynamic tracking and the forward-backward KLT on the resident pair give exactly what the
    call-by-call entry points give on re-uploaded images, over several consecutive frames."""
    from dynosam_b200.frontend import FeatureTrackerGPU, TrackParams
    rng = np.random.default_rng(3)
    stream = SyntheticStream(n_objects=6, seed=5)
    frames = [stream.frame(k) for k in range(4)]
    frames = [(np.ascontiguousarray(g, np.uint8), np.ascontiguousarray(m, np.int32), np.ascontiguousarray(f, np.float32)) for g, m, f in frames]
    prm = TrackParams()
    pts = np.stack([rng.uniform(25, W - 25, 300), rng.uniform(25, H - 25, 300)], 1).astype(np.float32)
    age = rng.integers(0, 30, 300).astype(np.int32)
    a = FeatureTrackerGPU(W, H); b = FeatureTrackerGPU(W, H)
    for arr in frames[1]:
        a.pin(arr)                                            # pinned and pageable host buffers both work
    a.next_frame(frames[0][0], frames[0][2], frames[0][1])
    for k in range(1, 4):
        g0, m0, f0 = frames[k-1]; g1, m1, f1 = frames[k]
        kp, lab = _features_from_mask(rng, m0, f0, per_object=120)
        fage = rng.integers(0, 22, len(lab)).astype(np.int32); tid = np.arange(len(lab), dtype=np.int64)
        a.next_frame(g1, f1, m1)
        a.propagate_mask_resident(kp, lab, prm, min_votes=20)
        ra = a.track_dynamic(kp, lab, fage, tid, prm, 9000)
        ka = a.klt_track_fb(None, None, pts, prm, age, 25)
        cur = b.propagate_mask(kp, lab, m0, f0, m1, prm, min_votes=20)
        b.set_frame(f1, cur, None)
        rb = b.track_dynamic(kp, lab, fage, tid, prm, 9000)
        kb = b.klt_track_fb(g0, g1, pts, prm, age, 25)
        assert np.array_equal(a.motion_mask(), cur), k
        for x, y in zip(ra, rb):
            assert np.array_equal(x, y), k
        for x, y in zip(ka, kb):
            assert np.array_equal(x, y), k
    a.unpin(frames[1][0]); a.unpin(frames[1][1]); a.unpin(frames[1][2])


@pytest.mark.gpu
def test_stereo_track_matches_opencv():
    """FeatureTracker::stereoTrack: left -> right LK, disparity / depth test (the RANSAC in between is host code)."""
    from dynosam_b200.frontend import FeatureTrackerGPU
    from oracle import frontend_oracle as FO
    rng = np.random.default_rng(17)
    left, _, _ = SyntheticStream(n_objects=6, seed=3).frame(5)
    right = np.empty_like(left)                                     # a fronto-parallel scene: constant disparity of 9 px, except for
    right[:, :-9] = left[:, 9:]; right[:, -9:] = left[:, -9:]        # the bottom 70 rows, which are infinitely far away (zero disparity)
    right[H - 70:] = left[H - 70:]
    n = 600
    pts = np.stack([rng.uniform(15, W - 15, n), rng.uniform(15, H - 15, n)], 1).astype(np.float32)
    t = FeatureTrackerGPU(W, H)
    rp, st, depth, valid = t.stereo_track(left, right, pts, 721.5377, 0.5372)
    orp, ost, odepth, ovalid = FO.stereo_track(left, right, pts, 721.5377, 0.5372)
    agree = st == ost
    assert agree.mean() >= 0.99, agree.mean()
    both = (st == 1) & (ost == 1)
    assert np.percentile(np.abs(rp[both] - orp[both]).max(axis=1), 99) < 1e-2
    # the disparity test is a threshold on uL - uR: identical wherever the disparities are not within 1e-2 px of it
    clear = both & (np.abs((pts[:, 0] - orp[:, 0]) - 1.0) > 2e-2) & (np.abs(orp[:, 0]) > 2e-2)
    assert np.array_equal(valid[clear], ovalid[clear]) and valid[clear].sum() > 300 and (valid[clear] == 0).sum() > 0
    ok = clear & (valid == 1)
    assert np.abs(depth[ok] - odepth[ok]).max() <= 2e-3*np.abs(odepth[ok]).max()
    assert abs(np.median(depth[ok]) - 721.5377*0.5372/9.0) < 0.05
