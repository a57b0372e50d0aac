"""dynofront_find_homography_batch and dynofront_klt_track_points on the device against tests/homography_oracle.py and cv2:
the draw trace, every model's count, the RANSAC mask and model, the refined H and the returned mask; the composition with the
forward-backward KLT; determinism and the batch."""
import numpy as np
import pytest

import homography_oracle as HO
from dynosam_b200.synth_frames import SyntheticStream, W, H

pytestmark = pytest.mark.gpu
NEAR = 1e-3          # px^2: a final mask may differ only on a point whose error lies this close to thr^2
H_REL = 1e-12        # refined H: the oracle restates the kernel's LM (block-ordered sums, Cholesky, host lambdas) operation
                     # for operation, so the two agree to the last bit; the bound is the issue's contract


def _pinned_opencv():
    import cv2
    return tuple(int(x) for x in cv2.__version__.split(".")[:2]) == (4, 13)


def _tracker():
    from dynosam_b200.frontend import FeatureTrackerGPU
    return FeatureTrackerGPU(W, H)


def _run(t, probs, refine=True):
    from dynosam_b200.frontend import HomographyParams
    out = []
    for mi in sorted(set(p[3] for p in probs)):
        idx = [i for i, p in enumerate(probs) if p[3] == mi]
        t.homography_record_counts(max(mi, 1))
        r = t.find_homography_batch([(probs[i][1], probs[i][2]) for i in idx], HomographyParams(max_iters=mi, refine=refine))
        tr = t.homography_trace(max(mi, 1))
        for j, i in enumerate(idx):
            out.append((i, dict(H=r["H"][j], mask=r["masks"][j], n_inl=int(r["n_inliers"][j]), status=int(r["status"][j]),
                                iterations=int(r["iterations"][j]), groups=int(tr["groups"][j]), rejected=int(tr["rejected"][j]),
                                best=int(tr["best"][j]), counts=tr["counts"][j])))
    return [d for _, d in sorted(out, key=lambda x: x[0])]


def _same_trace(d, o):
    k = len(o.counts)
    return (d["status"], d["iterations"], d["groups"], d["rejected"], d["best"]) == (o.status, o.iterations, o.groups, o.rejected, o.best) \
        and np.array_equal(d["counts"][:k], np.asarray(o.counts, np.int32)) and (d["counts"][k:] == -1).all()


def _check(name, d, o, refine):
    """None when the device equals the oracle, else the reason the oracle proves the difference (or raises)"""
    if not _same_trace(d, o):
        # the models are plain IEEE arithmetic on both sides; only RANSACUpdateNumIters' pow / log may round differently
        assert o.niters_margin <= 1e-9, (name, d["iterations"], o.iterations, o.niters_margin)
        return f"{name}: iterations {d['iterations']} vs {o.iterations} on a cvRound tie"
    if o.status != HO.OK:
        assert np.array_equal(d["mask"], o.mask), name
        if o.H is not None:
            assert np.array_equal(d["H"], o.H), name
        return None
    if not refine:
        assert np.array_equal(d["H"], o.H), name                       # the RANSAC model: bit for bit
        assert np.array_equal(d["mask"], o.mask), name
        return None
    rel = np.abs(d["H"] - o.H).max()/np.abs(o.H).max()
    assert rel <= H_REL, (name, rel)
    bad = d["mask"] != o.mask
    if bad.any():
        assert (o.margin[bad] <= NEAR).all(), (name, o.margin[bad])
        return f"{name}: {int(bad.sum())} point(s) within {NEAR} px^2 of the threshold"
    return None


@pytest.mark.parametrize("refine", [False, True])
def test_device_matches_oracle(refine):
    probs = HO.parity_set("small")
    t = _tracker()
    dev = _run(t, probs, refine)
    named = []
    for (name, a, b, mi), d in zip(probs, dev):
        o = HO.find_homography(a, b, max_iters=mi, refine_model=refine)
        why = _check(name, d, o, refine)
        if why:
            named.append(why)
    print("differences the oracle proves:", named)


@pytest.mark.skipif(not _pinned_opencv(), reason="restatement pinned against OpenCV 4.13")
def test_device_matches_cv2():
    """the device's masks equal cv2's on the full parity set; where they differ, the device's RANSAC inliers reproduce cv2's H
    through cv2's own method-0 fit (same RANSAC result, the refinement alone differs) and the problem is one the CPU suite names"""
    import cv2
    from test_homography import ransac_stage_equals_cv2
    probs = HO.parity_set("full")
    t = _tracker()
    dev = _run(t, probs, True)
    ran = _run(t, probs, False)
    differ = []
    for (name, a, b, mi), d, q in zip(probs, dev, ran):
        Hc, mk = cv2.findHomography(a, b, cv2.RANSAC, 5.0, maxIters=mi)
        mk = np.zeros(len(a), np.uint8) if mk is None else mk.ravel()
        assert (Hc is None) == (d["status"] == HO.RANSAC_FAILED or not d["H"].any()), name
        if not np.array_equal(d["mask"], mk):
            differ.append(name)
            R = HO.Result(q["status"], ransac_mask=q["mask"])
            assert ransac_stage_equals_cv2(a, b, R, Hc), name
    print("masks that differ from cv2 through the LM alone:", differ)
    assert set(differ) <= set(HO.CV2_LM_DIFFERENCES), differ


def test_batch_of_400_in_one_launch_equals_single_calls():
    from dynosam_b200.frontend import HomographyParams
    rng = np.random.default_rng(5)
    probs = [HO.make_problem(1000 + i, int(rng.integers(3, 600)), float(rng.uniform(0, 0.6))) for i in range(400)]
    t = _tracker()
    r = t.find_homography_batch(probs)
    assert r["status"].shape == (400,)
    for i in range(0, 400, 37):
        s = t.find_homography_batch([probs[i]])
        assert np.array_equal(s["H"][0], r["H"][i]) and np.array_equal(s["masks"][0], r["masks"][i]) and s["iterations"][0] == r["iterations"][i]
    again = t.find_homography_batch(probs)                              # two calls: bit-identical
    assert np.array_equal(again["H"], r["H"]) and all(np.array_equal(x, y) for x, y in zip(again["masks"], r["masks"]))
    t.find_homography_batch(probs, HomographyParams(refine=False))
    assert (t.homography_trace()["status"] == r["status"]).all()


def _c4_points(stream, k, n, rng):
    g0, _, _ = stream.frame(k - 1); g1, m1, f1 = stream.frame(k)
    pts = np.stack([rng.uniform(5, W - 5, n), rng.uniform(5, H - 5, n)], 1).astype(np.float32)
    return g0, g1, m1, f1, pts


def _host_chain(t, g0, g1, pts, age, prm):
    """klt_track_fb + host compaction + cv2.findHomography + &: what KltFeatureTracker::trackPoints does today"""
    import cv2
    nxt, st, _, keep = t.klt_track_fb(g0, g1, pts, prm, age, 25)
    good = np.nonzero(st)[0]
    if len(good) >= 4:
        Hc, mk = cv2.findHomography(pts[good], nxt[good], cv2.RANSAC, 5.0)
        mk = np.zeros(len(good), np.uint8) if mk is None else mk.ravel()
    else:
        Hc, mk = None, np.ones(len(good), np.uint8)
    ver = np.zeros(len(pts), np.uint8); ver[good] = mk
    return nxt, st, ver, keep & ver, Hc


@pytest.mark.parametrize("streaming", [False, True])
def test_klt_track_points_equals_host_chain(streaming):
    from dynosam_b200.frontend import TrackParams
    rng = np.random.default_rng(8)
    stream = SyntheticStream(n_objects=10, seed=42)
    prm = TrackParams(shrink_row=20, shrink_col=20)
    a = _tracker(); b = _tracker()
    if streaming:
        g, m, f = stream.frame(19)
        a.next_frame(np.ascontiguousarray(g, np.uint8), np.ascontiguousarray(f, np.float32), np.ascontiguousarray(m, np.int32))
    for k in (20, 21, 22):
        g0, g1, m1, f1, pts = _c4_points(stream, k, 800, rng)
        age = rng.integers(0, 30, len(pts)).astype(np.int32)
        b.set_frame(f1, m1, None)
        if streaming:
            a.next_frame(np.ascontiguousarray(g1, np.uint8), np.ascontiguousarray(f1, np.float32), np.ascontiguousarray(m1, np.int32))
            out = a.klt_track_points(None, None, pts, prm, age, 25)
        else:
            a.set_frame(f1, m1, None)
            out = a.klt_track_points(g0, g1, pts, prm, age, 25)
        nxt, st, ver, keep, Hd = out
        rn, rs, rv, rk, Hc = _host_chain(b, g0, g1, pts, age, prm)
        assert np.array_equal(nxt, rn) and np.array_equal(st, rs), k
        assert np.array_equal(ver, rv), (k, int((ver != rv).sum()))
        assert np.array_equal(keep, rk), k
        assert Hd is not None and Hc is not None and np.abs(Hd - Hc).max() <= 1e-6*np.abs(Hc).max(), k
        assert a.last_counts == (int(st.sum()), int(ver.sum()), int(keep.sum()))
        assert 0 < ver.sum() <= st.sum()


def test_klt_track_points_small_and_failed_frames():
    """n < 4 and n == 4 surviving points, and a frame where RANSAC fails (all points identical)"""
    from dynosam_b200.frontend import TrackParams, HOM_TOO_FEW, HOM_FOUR_POINT, HOM_RANSAC_FAILED
    rng = np.random.default_rng(9)
    stream = SyntheticStream(n_objects=10, seed=42)
    g0, g1, m1, f1, pts = _c4_points(stream, 30, 200, rng)
    t = _tracker(); b = _tracker(); t.set_frame(f1, m1, None); b.set_frame(f1, m1, None)
    _, st, _, _ = b.klt_track_fb(g0, g1, pts)
    good = pts[st == 1]
    for npts, want in ((3, HOM_TOO_FEW), (4, HOM_FOUR_POINT)):
        p = good[:npts]
        nxt, s, ver, keep, Hd = t.klt_track_points(g0, g1, p)
        assert t.last_hom_status == want and t.homography_trace()["status"][0] == want
        rn, rs, rv, rk, Hc = _host_chain(b, g0, g1, p, np.zeros(npts, np.int32), TrackParams())
        assert np.array_equal(ver, rv) and s.sum() == npts
        if want == HOM_FOUR_POINT:
            assert np.array_equal(Hd, Hc)
    same = np.repeat(good[:1], 50, axis=0)
    nxt, s, ver, keep, Hd = t.klt_track_points(g0, g1, same)
    assert t.last_hom_status == HOM_RANSAC_FAILED and Hd is None
    assert s.sum() == 50 and ver.sum() == 0
