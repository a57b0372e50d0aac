"""dynofront_find_fundamental_batch on the device against tests/fundamental_oracle.py and cv2: the draw trace (groups, rejections,
iterations, models per draw, every model's count or median, the best (draw, root)), F and the mask; the batch against single calls;
the refusals."""
import numpy as np
import pytest

import fundamental_oracle as FO
from dynosam_b200.synth_frames import W, H

pytestmark = pytest.mark.gpu


def _tracker():
    from dynosam_b200.frontend import FeatureTrackerGPU
    return FeatureTrackerGPU(W, H)


def _run(t, probs):
    from dynosam_b200.frontend import FundamentalParams
    out = {}
    for mi in sorted(set(p[3] for p in probs)):
        idx = [i for i, p in enumerate(probs) if p[3] == mi]
        cap = max(mi, 3)
        t.fundamental_record(cap)
        r = t.find_fundamental_batch([(probs[i][1], probs[i][2]) for i in idx], FundamentalParams(max_iters=mi))
        tr = t.fundamental_trace(cap)
        for j, i in enumerate(idx):
            out[i] = dict(F=r["F"][j], n_models=int(r["n_models"][j]), mask=r["masks"][j], n_inl=int(r["n_inliers"][j]),
                          status=int(r["status"][j]), iterations=int(r["iterations"][j]), groups=int(tr["groups"][j]),
                          rejected=int(tr["rejected"][j]), best=(int(tr["best"][j]), int(tr["best_root"][j])),
                          success=int(tr["success"][j]), record=tr["record"][j])
    return [out[i] for i in range(len(probs))]


def _check(name, a, b, d, o):
    """None when the device equals the oracle, else the reason, proven at the first point where the two part: a draw's root
    count on its discriminant margin, a model's inlier count on its threshold margin, the iteration count on the stopping rule's
    cvRound margin, an LMedS best on a median tie, an F by explain_F (the C library's acos / cos / pow within 2 ulp) and a mask
    point on its threshold margin"""
    rec = d["record"]
    k = min(len(o.models), len(rec))
    j = 0
    for i in range(k):
        km = int(rec[i, 0])
        if km != o.models[i]:
            assert o.draw_margins[i] <= 1e-12, (name, i, km, o.models[i], o.draw_margins[i])
            return f"{name}: iteration {i} root count {km} vs {o.models[i]} on a discriminant tie"
        for r in range(max(km, 0)):
            if o.status == FO.OK and float(rec[i, 1 + r]) != float(o.scores[j]):
                assert o.model_margins[j] <= 1e-6, (name, i, r, rec[i, 1 + r], o.scores[j], o.model_margins[j])
                return f"{name}: iteration {i} root {r} count on a threshold tie"
            j += 1
    if (d["status"], d["iterations"], d["groups"], d["rejected"]) != (o.status, o.iterations, o.groups, o.rejected):
        assert o.niters_margin <= 1e-9, (name, d["iterations"], o.iterations, o.niters_margin)
        return f"{name}: iterations {d['iterations']} vs {o.iterations} on a cvRound tie"
    if o.status in (FO.OK, FO.LMEDS) and d["best"] != tuple(o.best):
        assert o.status == FO.LMEDS, name
        flat = {}
        for i, km in enumerate(o.models):
            for r in range(max(km, 0)):
                flat[(i, r)] = len(flat)
        x, y = o.scores[flat[d["best"]]], o.scores[flat[tuple(o.best)]]
        # two medians whose order the roots' last bits decide: equal to 1e-6, or both at the rounding floor of an exact fit
        assert abs(x - y) <= 1e-6*max(abs(x), abs(y)) or max(x, y) <= 1e-12, (name, d["best"], o.best, x, y)
        return f"{name}: LMedS best {d['best']} vs {tuple(o.best)} on a median tie ({x} vs {y})"
    assert d["n_models"] == (len(o.F) if o.status == FO.SEVEN_POINT else (1 if o.F else 0)), name
    why = None
    for r, F in enumerate(o.F):
        if not np.array_equal(d["F"][r], F):
            group, root = (np.arange(7), r) if o.status == FO.SEVEN_POINT else (o.draws[o.best[0]], o.best[1])
            assert FO.explain_F(a, b, group, root, d["F"][r]), (name, r, d["F"][r], F)
            why = f"{name}: F differs in the C library's acos / cos / pow last bits"
    bad = d["mask"] != o.mask
    if bad.any():
        assert why, name
        thr2 = np.float32(1.0)
        if o.status == FO.LMEDS:
            import math
            jb = sum(max(km, 0) for km in o.models[:o.best[0]]) + o.best[1]        # the best model's median
            sg = max(2.5*1.4826*(1 + 5./(len(a) - 7))*math.sqrt(o.scores[jb]), 0.001)
            thr2 = np.float32(sg*sg)
        e = FO.errors(o.F[0], np.asarray(a, np.float32), np.asarray(b, np.float32)).astype(np.float64)
        assert (np.abs(e[bad] - float(thr2)) <= 1e-6).all(), (name, e[bad])
    else:
        assert d["n_inl"] == o.n_inliers, name
    if o.status == FO.LMEDS:
        assert d["success"] == int(o.success), name
    return why


def test_device_matches_oracle():
    probs = FO.parity_set("small")
    probs += [(f"seven_s{s}", *FO.make_problem(900 + s, 7, 0.0, "general"), 1000) for s in range(5)]
    probs += [("few", *FO.make_problem(950, 5, 0.0), 1000), ("empty", np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32), 1000)]
    t = _tracker()
    dev = _run(t, probs)
    named = []
    for (name, a, b, mi), d in zip(probs, dev):
        o = FO.find_fundamental(a, b, max_iters=mi)
        why = _check(name, a, b, d, o)
        if why:
            named.append(why)
    # every difference above is proven by _check; most problems match bit for bit
    assert len(named) <= len(probs)//4, named


def test_masks_match_cv2():
    cv2 = pytest.importorskip("cv2")
    probs = FO.parity_set("small")
    dev = _run(_tracker(), probs)
    for (name, a, b, mi), d in zip(probs, dev):
        Fc, mk = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, 1.0, 0.99, maxIters=mi)
        if Fc is not None:
            assert np.array_equal(d["mask"], mk.ravel()), name


def test_batch_equals_single_calls():
    from dynosam_b200.frontend import FundamentalParams
    r = np.random.default_rng(5)
    probs = [FO.make_problem(2000 + i, int(r.integers(5, 300)), float(r.uniform(0, 0.6)), ["general", "stereo", "planar"][i % 3])
             for i in range(400)]
    t = _tracker()
    big = t.find_fundamental_batch(probs, FundamentalParams())
    for i in range(0, 400, 37):
        one = t.find_fundamental_batch([probs[i]], FundamentalParams())
        assert np.array_equal(one["F"][0], big["F"][i]) and np.array_equal(one["masks"][0], big["masks"][i])
        assert (one["status"][0], one["iterations"][0], one["n_inliers"][0]) == (big["status"][i], big["iterations"][i], big["n_inliers"][i])


def test_large_problem_and_refusals():
    from dynosam_b200.frontend import FundamentalParams, FrontendError
    a, b = FO.make_problem(77, 20000, 0.3)
    t = _tracker()
    d = _run(t, [("n20000", a, b, 1000)])[0]
    why = _check("n20000", a, b, d, FO.find_fundamental(a, b))
    assert why is None or "last bits" in why, why
    for bad in (FundamentalParams(threshold_px=0.0), FundamentalParams(confidence=1.0), FundamentalParams(confidence=0.0)):
        with pytest.raises(FrontendError):
            t.find_fundamental_batch([(a[:20], b[:20])], bad)
