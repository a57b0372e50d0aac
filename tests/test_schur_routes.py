"""The dense fp64 elimination reference (schur_reference.py) against the CPU oracle, the power of its scaled comparator,
and the route graphs against the route mirror: every graph takes the cases it is built for."""
import dataclasses

import numpy as np
import pytest

import schur_reference as SR
from dynosam_b200 import synth
from dynosam_b200.problem import FLOWPROJ2, HYBRID3, POSE2POINT3, STEREO3, TERNARY3, MOTIONPOSE3


def _oracle(p):
    from oracle import oracle as O
    return O.OracleProblem(p)


GRAPHS = dict(SR.ROUTE_GRAPHS, c1_hybrid=lambda: synth.make_config("C1"), c1_wcme=lambda: synth.make_config("C1", formulation="wcme"))
# A stereo landmark seen once or twice has V = B^T B with condition ~(depth/baseline)^2 ~ 3e3: two fp64 inverses of it
# differ by that times the rounding unit.
REF_TOL = dict(window_np1=1e-12)


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_reference_matches_oracle(name):
    p = GRAPHS[name]()
    o = _oracle(p)
    for lam in (1e-4, 1e-1):
        R = SR.Reference(p, o.linearize_block, lam)
        So, go = SR.oracle_in_user_order(o, lam)
        tol = REF_TOL.get(name, 1e-13)
        assert R.s_err(So) <= tol and R.g_err(go) <= tol, (R.s_err(So), R.g_err(go))
        rc, d = o.schur_solve(lam)
        assert rc == 0
        npz = 6*p.n_pose
        assert R.l_err(d[npz:], d[:npz]) <= tol
        if R.H.shape[0] <= 4000:         # the oracle's dense normal equations (n x n)
            H, g = o.dense_normal()
            sc = np.sqrt(R.Hdiag)
            assert (np.abs(R.H.toarray() - H)/np.outer(sc, sc)).max() <= 1e-14
            assert (np.abs(R.g - g)/(sc*R.r)).max() <= 1e-14


def test_comparator_has_power():
    """A whole landmark removed, or one off-diagonal 6x6 block of S off by 1e-8 relative: both far above 1e-11."""
    p = synth.make_config("C1")
    o = _oracle(p)
    lam = 1e-4
    R = SR.Reference(p, o.linearize_block, lam)
    So, _ = SR.oracle_in_user_order(o, lam)
    assert R.s_err(So) <= 1e-13
    # one 15-observation static landmark removed
    b0 = p.blocks[0]
    assert b0.type == POSE2POINT3
    cnt = np.bincount(b0.idx[:, 1])
    l = int(np.flatnonzero(cnt == 15)[0])
    keep = b0.idx[:, 1] != l
    q = dataclasses.replace(p, blocks=[dataclasses.replace(b0, idx=b0.idx[keep], meas=b0.meas[keep])] + list(p.blocks[1:]))
    Sq, _ = SR.oracle_in_user_order(_oracle(q), lam)
    assert R.s_err(Sq) > 1e-6, R.s_err(Sq)
    # the off-diagonal block with the largest scaled entry, times (1 + 1e-8)
    d = np.sqrt(R.Hdiag[:R.npz])
    sc = np.abs(R.S)/np.outer(d, d)
    n = p.n_pose
    blk = sc.reshape(n, 6, n, 6).max(axis=(1, 3)); np.fill_diagonal(blk, 0)
    a, b = np.unravel_index(blk.argmax(), blk.shape)
    Sm = So.copy()
    Sm[6*a:6*a + 6, 6*b:6*b + 6] *= 1 + 1e-8; Sm[6*b:6*b + 6, 6*a:6*a + 6] *= 1 + 1e-8
    assert R.s_err(Sm) > 1e-11, R.s_err(Sm)


def test_mirror_constants():
    """The route mirror's constants as read from the CUDA sources, and the relations between them the routes rely on."""
    assert SR.GEN_REFUSE_ABOVE == SR.GG_MAXL                 # finalize refuses exactly what schur_general_kernel cannot hold
    assert SR.WIN_TMAX <= 32 and SR.STAGE_HALF_T == 16       # the stage kernel: one landmark per warp, two per warp at <= 16
    assert SR.WIN_TMAX < SR.SIMPLE_STAGED_T <= 32            # the simple kernel stages one factor per lane
    assert SR.CHUNK_CAP[0] >= SR.WIN_TMAX                    # NP = 1: a window landmark always fits one chunk
    assert SR.CHUNK_CAP[1] < 2*SR.WIN_TMAX <= SR.WIN_NLOC_MAX  # NP = 2: the widest landmarks get chunks of their own
    assert SR.win_ntiles(24) == 12 and SR.win_ntiles(40) == 30 and SR.win_ntiles(SR.WIN_NLOC_MAX) == 42
    assert -(-SR.win_ntiles(SR.CHUNK_CAP[1]) // SR.WIN_ACC_WARPS) == 2
    assert -(-SR.win_ntiles(2*SR.WIN_TMAX) // SR.WIN_ACC_WARPS) == 3


def _by(rs, route, *types):
    return [g for g in rs if g.route == route and (not types or g.ftype in types)]


def test_window_np1_graph_cases():
    p = SR.window_np1_graph()
    rs = SR.routes(p)
    assert {g.route for g in rs} == {"window"}
    cases = {1, 2, SR.STAGE_HALF_T - 1, SR.STAGE_HALF_T, SR.STAGE_HALF_T + 1, SR.WIN_TMAX}
    for t in (POSE2POINT3, STEREO3):
        Ts = np.array([g.T for g in rs if g.ftype == t])
        for T in cases:
            assert (Ts == T).sum() >= (100 if t == POSE2POINT3 else 20), (t, T)
    bi = next(i for i, b in enumerate(p.blocks) if b.type == POSE2POINT3)
    ng = sum(g.block == bi for g in rs)
    assert ng > 3*SR.HOST_SEGMENT_GROUPS and ng % 2 == 1
    ch = SR.chunk_stats(p, bi)
    assert max(c[1] for c in ch) > SR.WIN_BATCH_LMK and max(c[2] for c in ch) > SR.WIN_BATCH_SLOTS
    assert p.n_pose >= 440


def test_window_np2_graph_cases():
    p = SR.window_np2_graph()
    rs = SR.routes(p)
    hyb = _by(rs, "window", HYBRID3)
    Ts = {g.T for g in hyb}
    assert set(range(SR.STAGE_HALF_T + 1, SR.WIN_TMAX + 1)) <= Ts
    bi = next(i for i, b in enumerate(p.blocks) if b.type == HYBRID3)
    nl = [c[0] for c in SR.chunk_stats(p, bi)]
    assert {2*T for T in range(SR.CHUNK_CAP[1]//2 + 1, SR.WIN_TMAX + 1)} <= set(nl)       # NLOC 42..48: own chunks, 3 stripes
    assert any(SR.CHUNK_CAP[1] - 8 < x <= SR.CHUNK_CAP[1] for x in nl)                  # and shared chunks up to the cap


def test_simple_graph_cases():
    p = SR.simple_graph()
    rs = SR.routes(p)
    for t in (POSE2POINT3, HYBRID3):
        s = _by(rs, "simple", t)
        Ts = {g.T for g in s if not g.repeated}
        assert {SR.WIN_TMAX + 1, SR.SIMPLE_STAGED_T, SR.SIMPLE_STAGED_T + 1, 64, 65} <= Ts, (t, Ts)
        rep = [g.T for g in s if g.repeated]
        assert any(T <= SR.WIN_TMAX for T in rep) and any(T > SR.SIMPLE_STAGED_T for T in rep), (t, rep)
        assert len(_by(rs, "window", t)) > 100                  # the same block holds window landmarks: grp_win filters
        assert len({g.block for g in rs if g.ftype == t}) == 1
    assert len(_by(rs, "simple", FLOWPROJ2)) > 0


def test_general_graph_cases():
    rs = SR.routes(SR.general_wcme_graph())
    pts = {g.points for g in _by(rs, "general", TERNARY3)}
    assert {10, 11, 12, SR.GG_MAXL - 1, SR.GG_MAXL} <= pts
    assert not _by(rs, "unsupported")
    assert any(g.points == SR.GG_MAXL and g.T + g2.T > 32 for g in _by(rs, "general", POSE2POINT3)
               for g2 in _by(rs, "general", TERNARY3) if g2.root == g.root)
    # a static point with POSE2POINT3 and STEREO3 factors from the same frame: one general group over two blocks
    st = {g.root for g in _by(rs, "general", STEREO3)}
    assert st and all(g.points == 1 for g in _by(rs, "general", STEREO3))
    assert any(g.root in st for g in _by(rs, "general", POSE2POINT3))
    rs = SR.routes(SR.general_wcpe_graph())
    assert SR.GG_MAXL in {g.points for g in _by(rs, "general", MOTIONPOSE3)} and not _by(rs, "unsupported")


def test_refused_chain_graph_cases():
    rs = SR.routes(SR.refused_chain_graph())
    assert max(g.points for g in rs) == SR.GG_MAXL + 1
    assert {g.points for g in _by(rs, "unsupported")} == {SR.GG_MAXL + 1}
