"""dynoba_triangulate_batch on the H100: bit for bit the host build of triangulate.cuh (so every status equals it), the
50-digit reference within the a-priori bound, results independent of the batch around a problem, camera counts across
warp boundaries, C5-shaped full tracks, the empty batch and the refusals."""
import numpy as np
import pytest

import triangulation_reference as TR
from dynosam_b200 import binding as B
from dynosam_b200 import synth_stereo
from test_triangulate import K5, build_shim, camera, check, host, problem, stereo_cams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(tmp_path_factory.mktemp("trig"))


def same(a, d):
    for k in ("status", "point", "reproj", "sv"):
        assert np.array_equal(a[k], d[k], equal_nan=True), k


def sized_problems(seed=0):
    rng = np.random.default_rng(seed)
    probs = []
    for m in (1, 2, 15, 16, 17, 32, 33, 64, 65, 100):
        p = np.array([rng.uniform(-5, 5), rng.uniform(-2, 2), rng.uniform(5, 80)])
        cams = stereo_cams((m + 1)//2, 0.5, int(rng.integers(1 << 20)))[:m]
        probs.append(problem(cams, p, rng.uniform(0.02, 0.2), int(rng.integers(1 << 20))))
    return probs


def test_device_equals_host_build_and_reference(shim):
    probs = sized_problems()
    d = B.triangulate_batch(probs, device=0)
    same(host(shim, probs), d)
    a, refs = check(shim, probs)                     # the host build (= the device) against the reference
    near = [i for i, r in enumerate(refs) if abs(r["reproj"] - 3.0) < 1e-9 or (np.isfinite(r["sv"][2]) and abs(r["sv"][2] - 1.0) < 1e-9)]
    assert near == [], near                          # nothing within 1e-9 of a threshold in these cases
    assert [r["status"] for r in refs][0] == TR.DEGENERATE and sum(r["status"] == TR.OK for r in refs) >= 7


def test_full_tracks_c5_shaped(shim):
    p, st = synth_stereo.make_scene(n_frames=200, n_static=20000, seed=2, far_fraction=0.05, nan_right=0.05, outlier_fraction=0.01)
    off, poses, kp, cal = synth_stereo.full_track_problems(p.pose, st)
    a = dict(off=off, poses=poses, kp=kp, calib=cal)
    n = off.size - 1
    for dev in (False, True):
        r = dict(a, point=np.zeros((n, 3)), status=np.zeros(n, np.int32), reproj=np.zeros(n), sv=np.zeros((n, 4)))
        if dev:
            assert B.triangulate_call(B.load().dynoba_triangulate_batch, r, 1.0, 3.0, 0) == 0
            same(h, r)
        else:
            B.triangulate_call(shim.host_triangulate_batch, r, 1.0, 3.0); h = r
    assert len(set(h["status"].tolist())) >= 3


def test_batch_independence():
    probs = sized_problems(1)
    whole = B.triangulate_batch(probs, device=0)
    rev = B.triangulate_batch(probs[::-1], device=0)
    for i in range(len(probs)):
        alone = B.triangulate_batch([probs[i]], device=0)
        for k in ("status", "point", "reproj", "sv"):
            assert np.array_equal(alone[k][0], whole[k][i], equal_nan=True)
            assert np.array_equal(rev[k][len(probs) - 1 - i], whole[k][i], equal_nan=True)
    again = B.triangulate_batch(probs, device=0)
    same(whole, again)


def test_empty_batch_and_refusals():
    L = B.load()
    assert B.triangulate_batch([], device=0)["status"].size == 0
    good = [problem([camera(), camera(0.0, (1.0, 0.0, 0.0))], np.array([0.0, 0.0, 10.0]))]

    def call(a, rank_tol=1.0, thr=3.0):
        return B.triangulate_call(L.dynoba_triangulate_batch, a, rank_tol, thr, 0)
    assert call(B.triangulate_arrays(good)) == B.OK
    bad = []
    a = B.triangulate_arrays(good); a["off"][1] = -1; bad.append((a, 1.0, 3.0))
    a = B.triangulate_arrays(good); a["off"][0] = 1; bad.append((a, 1.0, 3.0))
    a = B.triangulate_arrays(good); a["poses"][0, 9] = np.nan; bad.append((a, 1.0, 3.0))
    a = B.triangulate_arrays(good); a["kp"][1, 0] = np.inf; bad.append((a, 1.0, 3.0))
    a = B.triangulate_arrays(good); a["calib"][0, 0] = 0.0; bad.append((a, 1.0, 3.0))
    a = B.triangulate_arrays(good); a["calib"][0, 1] = -1.0; bad.append((a, 1.0, 3.0))
    bad += [(B.triangulate_arrays(good), -1.0, 3.0), (B.triangulate_arrays(good), np.nan, 3.0), (B.triangulate_arrays(good), 1.0, np.nan),
            (B.triangulate_arrays(good), 1.0, -1.0)]
    for a, rt, th in bad:
        st = a["status"].copy()
        assert call(a, rt, th) == B.ERR_BAD_ARG and np.array_equal(a["status"], st)
    a = B.triangulate_arrays(good)
    assert B.triangulate_call(L.dynoba_triangulate_batch, dict(a, status=np.zeros(0, np.int32)), 1.0, 3.0, 0) == B.ERR_BAD_ARG
    assert call(B.triangulate_arrays(good), 1.0, np.inf) == B.OK                 # +inf turns the reprojection test off
