"""STEREO_PROJECTION static landmarks with the triangulations on the H100: the builder decides exactly as with the host
build, and dynoba_optimize on the emitted stereo graph runs the oracle's LM (equal iteration counts, chi^2 and values
within the parity bars of tests/test_gpu_parity.py)."""
import numpy as np
import pytest

from dynosam_b200 import synth_stereo
from dynosam_b200.binding import Solver
from dynosam_b200.builder import GraphBuilder
from test_builder_stereo import feed

pytestmark = pytest.mark.gpu


def test_device_decisions_equal_host():
    p, st = synth_stereo.make_scene(n_frames=60, n_static=3000, seed=5, far_fraction=0.1, nan_right=0.1, outlier_fraction=0.02)
    out = []
    for dev in (-1, 0):
        b = GraphBuilder(); feed(b, p, st, device=dev)
        out.append((b.problem(), b.static_stereo_stats())); b.close()
    (q, s), (r, t) = out
    assert s == t and s["added"] > 1000
    assert np.array_equal(q.point, r.point) and np.array_equal(q.point_keys, r.point_keys)
    for x, y in zip(q.blocks, r.blocks):
        assert x.type == y.type and np.array_equal(x.idx, y.idx) and np.array_equal(x.meas, y.meas, equal_nan=True)


def test_optimize_the_stereo_graph_like_the_oracle():
    from oracle import oracle as O
    p, st = synth_stereo.make_scene(n_frames=20, n_static=700, seed=9, nan_right=0.05)
    b = GraphBuilder(); feed(b, p, st, device=0)
    q = b.problem()
    s = Solver(); b.emit(s); s.problem = q
    o = O.OracleProblem(q)
    assert abs(s.error() - o.error()) <= 1e-6*o.error()
    st_ = s.optimize(); so = o.optimize()
    assert st_["iterations"] == so["iterations"] and st_["inner_iterations"] == so["inner_iterations"]
    assert abs(st_["error_final"] - so["error_final"]) <= 1e-6*so["error_final"]
    pose, point, _ = s.values()
    assert np.abs(pose - o.pose).max() < 1e-6 and np.abs(point - o.point).max() < 1e-5
    s.close(); b.close()
