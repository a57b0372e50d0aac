"""dynoba_pnp_ransac_batch on the device against tests/pnp_oracle.py under the same seeded hypothesis stream: parity, determinism
and the hand-off into dynoba_flow_pose_batch."""
import numpy as np
import pytest

import pnp_oracle as PO
from dynosam_b200 import binding, lie
from dynosam_b200.synth_star import K5, make_pnp_problem, pnp_parity_set

pytestmark = pytest.mark.gpu


def _proven(q, o, r):
    """None if the device equals the oracle; otherwise the reason the oracle proves the difference is a last-bit comparison,
    or raises.  Every differing count must be within the number of points the oracle finds within NEAR of the threshold under
    that model, the first differing model must be an ambiguous disambiguation or such a count, and a differing final inlier
    must have a margin <= NEAR."""
    hc = r["hyp_counts"]; oc = o["hyp_counts"]
    m = min(len(hc), len(oc))
    diff = np.nonzero(hc[:m] != oc[:m])[0]
    same_run = len(hc) == len(oc) and not len(diff) and r["iterations"] == o["iterations"] and r["skipped"] == o["skipped"] \
        and r["best_hypothesis"] == o["best_hypothesis"]
    if same_run:
        bad = r["inlier"] != o["inlier"]
        if not bad.any():
            return None
        assert (o["point_margin"][bad] <= PO.NEAR).all(), "final inliers differ beyond the proven margin"
        return "final inliers at the threshold"
    first = int(diff[0]) if len(diff) else m
    assert first < len(o["hyp_near"]), "run lengths differ without a differing count"
    ok = abs(int(hc[first]) - int(oc[first])) <= int(o["hyp_near"][first]) or o["hyp_gap"][first] <= PO.NEAR
    assert ok, (first, hc[first], oc[first], o["hyp_near"][first], o["hyp_gap"][first])
    return f"model {first}: count {hc[first]} vs {oc[first]}"


def _check_parity(probs, out, max_named=1, **kw):
    named = []
    for i, (q, r) in enumerate(zip(probs, out)):
        o = PO.ransac(q["points"], q["kp"], q["calib"], p_index=i, **kw)
        why = _proven(q, o, r)
        if why is not None:
            named.append((i, len(q["kp"]), why))
            continue
        assert r["status"] == o["status"], (i, r["status"], o["status"])
        assert (r["iterations"], r["skipped"], r["best_hypothesis"], r["n_inliers"]) == (o["iterations"], o["skipped"], o["best_hypothesis"], o["n_inliers"]), i
        assert np.array_equal(r["hyp_counts"], o["hyp_counts"])
        assert np.array_equal(r["inlier"], o["inlier"])
        assert np.abs(r["pose"] - o["pose"]).max() <= 1e-9*max(1.0, np.abs(o["pose"]).max()), (i, np.abs(r["pose"] - o["pose"]).max())
    print("problems whose difference the oracle proves:", named)
    assert len(named) <= max_named, named
    return named


def test_parity_set_matches_oracle():
    probs = pnp_parity_set()
    out = binding.pnp_ransac_batch(probs, hyp_counts=True)
    assert len(out) == len(probs)
    _check_parity(probs, out)
    st = [r["status"] for r in out]
    assert st[0] == st[1] == binding.TRACK_FEW_MATCHES                       # n = 0, 4
    assert out[-3]["status"] == binding.TRACK_INVALID and out[-3]["skipped"] == 5000   # all collinear: the skip cap
    assert out[-2]["iterations"] == 501                                        # 70 % outliers: max_iterations + 1
    assert sum(s == binding.TRACK_VALID for s in st) >= 10


def test_parameters_match_oracle():
    """other threshold, iteration cap, probability, minimum and seed"""
    probs = pnp_parity_set()[5:13]
    kw = dict(threshold_px=2.0, max_iterations=40, probability=0.99, min_inliers=20, seed=1234567)
    out = binding.pnp_ransac_batch(probs, hyp_counts=True, **kw)
    _check_parity(probs, out, **kw)


def test_determinism_and_independence():
    probs = pnp_parity_set()
    a = binding.pnp_ransac_batch(probs, hyp_counts=True)
    b = binding.pnp_ransac_batch(probs, hyp_counts=True)
    for x, y in zip(a, b):
        for k in x:
            assert np.array_equal(x[k], y[k]), k
    # problem p's outputs do not depend on the other problems of the batch (the stream is indexed by p)
    rng = np.random.default_rng(9)
    other = [make_pnp_problem(rng, int(n), outliers=0.3) for n in rng.integers(5, 900, len(probs))]
    mixed = [probs[i] if i % 2 == 0 else other[i] for i in range(len(probs))]
    c = binding.pnp_ransac_batch(mixed, hyp_counts=True)
    for i in range(0, len(probs), 2):
        for k in a[i]:
            assert np.array_equal(a[i][k], c[i][k]), (i, k)
    # another seed draws other hypotheses
    d = binding.pnp_ransac_batch(probs, hyp_counts=True, seed=99)
    assert sum(x["best_hypothesis"] != y["best_hypothesis"] or not np.array_equal(x["hyp_counts"], y["hyp_counts"])
               for x, y in zip(a, d) if len(x["inlier"]) >= 30) >= 8


def test_batch_of_400_equals_one_by_one():
    rng = np.random.default_rng(13)
    probs = [make_pnp_problem(rng, int(n), outliers=float(f)) for n, f in zip(rng.integers(5, 400, 400), rng.choice([0.0, 0.1, 0.3, 0.5], 400))]
    allb = binding.pnp_ransac_batch(probs, hyp_counts=True)
    # problem index p seeds the stream: call one by one with the same index by padding with empty problems
    for p in range(0, 400, 37):
        one = binding.pnp_ransac_batch([dict(calib=K5, points=np.zeros((0, 3)), kp=np.zeros((0, 2)))]*p + [probs[p]], hyp_counts=True)[-1]
        for k in one:
            assert np.array_equal(one[k], allb[p][k]), (p, k)
    one0 = binding.pnp_ransac_batch([probs[0]], hyp_counts=True)[0]
    for k in one0:
        assert np.array_equal(one0[k], allb[0][k])


def test_large_problem_and_refusals():
    rng = np.random.default_rng(17)
    q = make_pnp_problem(rng, 20000, outliers=0.4)
    r = binding.pnp_ransac_batch([q], hyp_counts=True)[0]
    o = PO.ransac(q["points"], q["kp"], q["calib"])
    if _proven(q, o, r) is None:
        assert r["iterations"] == o["iterations"] and np.array_equal(r["inlier"], o["inlier"])
    assert r["status"] == binding.TRACK_VALID
    with pytest.raises(binding.DynobaError):
        binding.pnp_ransac_batch([q], threshold_px=0.0)


def test_hand_off_to_flow_pose_batch():
    """camera + 10 objects: the RANSAC pose and inlier set of every problem become the initial pose and the tracklets of
    dynoba_flow_pose_batch; the device chain equals the oracle chain (pnp_oracle -> star_oracle.flow_pose_lm)"""
    from oracle import star_oracle as SO
    rng = np.random.default_rng(23)
    probs = [make_pnp_problem(rng, 1500, outliers=0.1)] + [make_pnp_problem(rng, int(n), outliers=0.1) for n in rng.integers(150, 250, 10)]
    rs = binding.pnp_ransac_batch(probs, hyp_counts=True)
    flows, ref = [], []
    for i, (q, r) in enumerate(zip(probs, rs)):
        o = PO.ransac(q["points"], q["kp"], q["calib"], p_index=i)
        assert _proven(q, o, r) is None, i
        assert np.array_equal(r["inlier"], o["inlier"]) and r["status"] == binding.TRACK_VALID
        # the flow problem of the inliers: previous camera pose, depths of the world points seen from it, measured flow
        sel = r["inlier"]
        Xp = lie.compose(q["gt"][None], lie.se3_exp(np.array([[0.0, 0.0, 0.0, 0.0, 0.0, -0.5]])))[0]
        pc = lie.transform_to(np.tile(Xp, (sel.sum(), 1)), q["points"][sel])
        kp_prev = np.stack([K5[0]*pc[:, 0]/pc[:, 2] + K5[3], K5[1]*pc[:, 1]/pc[:, 2] + K5[4]], 1)
        flows.append(dict(pose_init=r["pose"], pose_prev=Xp, calib=K5, kp_prev=kp_prev, depth=pc[:, 2], flow=q["kp"][sel] - kp_prev))
        ref.append(o)
    fo = binding.flow_pose_batch(flows, flow_sigma=1.0, flow_prior_sigma=0.5, huber_k=1.0, outlier_rounds=0)
    for f, o, g in zip(flows, ref, fo):
        oo = SO.flow_pose_lm(o["pose"], f["pose_prev"], K5, f["kp_prev"], f["depth"], f["flow"], 1.0, 0.5, 1.0, max_iterations=10)
        assert (g["iterations"], g["inner_iterations"]) == (oo["iterations"], oo["inner_iterations"])
        assert abs(g["error_final"] - oo["error_final"]) <= 1e-9*max(oo["error_final"], 1e-12) + 1e-12
        assert np.abs(g["pose"] - oo["pose"]).max() < 1e-7
