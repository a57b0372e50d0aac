"""dynoba_object_srif_batch on the device: every object of every frame of 30-frame sequences against the numpy statement of the
reference (tests/srif_reference.py), bit-identical repeats, a 400-object batch against the same objects one by one, the empty
batch, the hand-off from dynoba_pnp_ransac_batch, and the refusals."""
import numpy as np
import pytest

import srif_reference as SR
from dynosam_b200 import binding as B
from dynosam_b200 import synth_srif as SS
from test_srif import REFUSALS, assert_same

pytestmark = pytest.mark.gpu


def gpu(objs, **kw):
    return B.object_srif_batch(objs, device=0, **kw)


def _same_bits(a, b):
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), k


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_sequences_match_reference(seed):
    seq = SS.make_sequence(n_frames=30, n_objects=4, seed=seed, few_first=seed == 1)
    ref = SR.run_sequence(seq, SR.reference_batch)
    dev = SR.run_sequence(seq, gpu)
    modes = set()
    for (objs, rr), (_, rd) in zip(ref, dev):
        for o, b, a, g in zip(objs, rr, rd, gpu(objs)):
            modes.add((o["mode"], b["status"]))
            assert_same(g, b, tol_scale=16.0)          # one step from the reference's inputs
            assert_same(a, b, tol_scale=1e3)           # the device's own trajectory
    assert {(SR.NEW, SR.OK), (SR.CONTINUE, SR.OK), (SR.RESET, SR.OK)} <= modes


def test_cases_match_reference():
    from test_srif import CASES
    for name, (obj, prm) in CASES.items():
        assert_same(gpu([obj], **prm)[0], SR.reference_batch([obj], **prm)[0])


def test_two_runs_are_bit_identical():
    objs = SS.random_frame(10, 200, seed=3)
    _ = [_same_bits(a, b) for a, b in zip(gpu(objs), gpu(objs))]


def test_batch_equals_objects_one_by_one():
    objs = SS.random_frame(400, 50, seed=4)
    rng = np.random.default_rng(0)
    for i, o in enumerate(objs):               # mixed sizes and modes: a stepped filter continues, some start over
        n = int(rng.integers(0, 50))
        for k in ("stereo", "valid", "points", "m_L", "has_point"):
            o[k] = o[k][:n]
    first = gpu(objs)
    for i, (o, r) in enumerate(zip(objs, first)):
        if r["status"] == SR.OK and i % 3:
            o.update(mode=SR.CONTINUE if i % 3 == 1 else SR.RESET, state=r["state"], m_L=r["m_L"], has_point=r["has_point"])
    batch = gpu(objs)
    for o, r in zip(objs, batch):
        _same_bits(r, gpu([o])[0])
    assert {r["status"] for r in batch} >= {SR.OK, SR.TOO_FEW}


def test_empty_batch():
    assert gpu([]) == []
    o = SS.random_frame(1, 8)[0]
    empty = o | dict(stereo=np.zeros((0, 6)), valid=np.zeros((0, 2), bool), points=np.zeros((0, 6)), m_L=np.zeros((0, 3)),
                     has_point=np.zeros(0, bool))
    r = gpu([empty | dict(mode=SR.CONTINUE, state=SR.step(o)["state"]), empty])
    assert r[0]["status"] == SR.OK and r[1]["status"] == SR.TOO_FEW


def test_pnp_hand_off():
    """dynoba_pnp_ransac_batch's inliers and statuses go straight into the filter step"""
    objs = SS.random_frame(8, 150, seed=9)
    fx, fy, s, u0, v0, _ = SS.CALIB6
    problems = []
    for o in objs:
        Xp = SR.T4(o["pose_prev"])
        pw = (Xp[:3, :3] @ o["points"][:, :3].T).T + Xp[:3, 3]
        problems.append(dict(calib=[fx, fy, s, u0, v0], points=pw, kp=np.stack([o["stereo"][:, 3], o["stereo"][:, 5]], 1)))
    pnp = B.pnp_ransac_batch(problems, device=0, threshold_px=2.0)
    fed = []
    for o, p in zip(objs, pnp):
        sel = np.nonzero(p["inlier"])[0]
        fed.append(o | dict(pnp_status=p["status"], stereo=o["stereo"][sel], valid=o["valid"][sel], points=o["points"][sel],
                            m_L=o["m_L"][sel], has_point=o["has_point"][sel]))
    assert any(p["status"] == B.TRACK_VALID for p in pnp)
    for o, g, r in zip(fed, gpu(fed), SR.reference_batch(fed)):
        assert_same(g, r)
        assert g["solved"] == (o["pnp_status"] == B.TRACK_VALID and g["status"] == SR.OK)


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals_before_any_device_work(name):
    """BAD_ARG even for a device that does not exist: the checks come before the device is touched"""
    objs, prm = REFUSALS[name]
    for dev in (0, 63):
        with pytest.raises(B.DynobaError) as e:
            B.object_srif_batch(objs, device=dev, **prm)
        assert e.value.status == B.ERR_BAD_ARG
