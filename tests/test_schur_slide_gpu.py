"""Landmark elimination on the sliding-window path against the dense fp64 reference (schur_reference.py), on the graphs
of slide_plan.py: slot reuse over hundreds of chunks and many runs, tracklets at the chunk cap (NLOC 42..48), a
sequence break inside one object, objects interleaved in time and one object's chunk sequence split across two time
shards.  Same units and tolerance as test_schur_routes_gpu.py; the library's census (Solver.info()) must equal the
plan mirror's."""
import numpy as np
import pytest

import schur_reference as SR
import slide_plan as SP
from dynosam_b200.binding import Solver

pytestmark = pytest.mark.gpu

TOL = 1e-11
LAMBDAS = (1e-4, 1e-1)


@pytest.mark.parametrize("name", sorted(SP.SLIDE_GRAPHS))
def test_sliding_elimination_matches_reference(name):
    p = SP.SLIDE_GRAPHS[name]()
    P = SP.plan(p, SP.hybrid_block(p))
    s = Solver(p)
    info = s.info()
    assert info["window_accum_ctas"][1] == P.ctas and info["window_blocks_flushed"][1] == P.flushed, (info, P.ctas, P.flushed)
    npz = 6*p.n_pose
    for lam in LAMBDAS:
        s.linearize()
        R = SR.Reference(p, s.linearization, lam)
        S, g = s.reduced_system(lam)
        es, eg = R.s_err(S), R.g_err(g)
        d = s.solve(lam)
        el = R.l_err(d[npz:], d[:npz])
        print(f"{name} lambda {lam:g}: S {es:.2e} g_S {eg:.2e} dl {el:.2e}; {len(P.chunks)} chunks, {len(P.runs)} runs")
        assert es <= TOL and eg <= TOL and el <= TOL, (es, eg, el)
    s.close()


def test_c5_census():
    """the flagship graph: the dynamic accumulate runs in a few hundred runs instead of one CTA pair per chunk"""
    from dynosam_b200 import synth
    s = Solver(synth.make_config("C5"))
    s.finalize()
    info = s.info()
    print("C5 window census:", info["window_accum_ctas"], info["window_blocks_flushed"])
    assert info["window_accum_ctas"][1] <= 2000 and info["window_blocks_flushed"][1] <= 5_000_000, info
    assert np.all(np.array(info["window_accum_ctas"]) > 0)
    s.close()
