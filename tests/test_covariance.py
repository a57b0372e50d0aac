"""CPU checks of dynoba_marginal_covariance's references: the tile recurrence of the band selected inversion
(selinv_reference.py) against numpy.linalg.inv on every plain band layout of band_reference, the dense reference on
closed-form graphs, and the reach of the GPU tests' graphs over the landmark routes."""
import numpy as np
import pytest

import band_reference as BR
import schur_reference as SR
import selinv_reference as SI
from dynosam_b200 import lie
from dynosam_b200.problem import BETWEEN6, MOTIONPOSE3, POSE2POINT3, PRIOR6, STEREO3, TERNARY3, FactorBlock, Problem

# selinv_reference against the equilibrated dense inverse, units sqrt(Sigma_aa Sigma_bb): the error follows
# kappa(D^-1/2 S D^-1/2), <= 100 in the dominant / graded families, ~1e10 in nearsing.  Measured worst: 1.4e-15
# (dominant, graded), 1.4e-7 (nearsing)
TOL_SELINV = {"dominant": 2e-14, "graded": 2e-14, "nearsing": 2e-6}


@pytest.mark.parametrize("name", [c.name for c in BR.PLAIN])
def test_selinv_reference_matches_inverse(name):
    case = BR.CASES[name]
    sysm = BR.build(case)
    ab, _ = sysm.band(0.0)
    S = BR.dense(ab)
    L = BR.layout(sysm.n, case.bw, -1)
    T = SI.selinv(SI.factor_tiles(S, L.WB))
    ref = SI.equilibrated_inverse(S)
    n = sysm.n
    i, j = np.tril_indices(n)
    keep = (i//BR.TILE - j//BR.TILE) <= L.WB
    i, j = i[keep], j[keep]
    got = np.array([SI.tiles_entry(T, a, b) for a, b in zip(i, j)])
    d = np.sqrt(np.abs(np.diag(ref)))
    err = float((np.abs(got - ref[i, j])/d[i]/d[j]).max())
    print(f"SELINV {case.family} {name}: {err:.2e}")
    assert err <= TOL_SELINV[case.family], err


def _dense_cov(p, kind, idx=None):
    from oracle.oracle import OracleProblem
    H, _ = OracleProblem(p).dense_normal()
    return SI.marginal_blocks(SI.equilibrated_inverse(H), (p.n_pose, p.n_point, p.n_flow, 0, 0), kind, idx)


IDENT = np.array([1.0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0])


def test_dense_reference_isotropic_prior():
    sigma = 0.3
    p = Problem(IDENT[None].copy(), np.zeros((0, 3)), blocks=[FactorBlock(PRIOR6, np.array([[0]]), IDENT[None], np.array([sigma]))])
    assert np.abs(_dense_cov(p, 0)[0] - sigma**2*np.eye(6)).max() <= 1e-15


@pytest.mark.parametrize("k", [1, 4, 9])
def test_dense_reference_between_chain(k):
    """prior on pose 0, k identity BetweenFactors of the same sigma at identity poses: Sigma_k = (k + 1) sigma^2 I"""
    sigma = 0.2
    poses = np.tile(IDENT, (k + 1, 1))
    blocks = [FactorBlock(PRIOR6, np.array([[0]]), IDENT[None], np.array([sigma])),
              FactorBlock(BETWEEN6, np.stack([np.arange(k), np.arange(1, k + 1)], 1), np.tile(IDENT, (k, 1)), np.array([sigma]))]
    C = _dense_cov(Problem(poses, np.zeros((0, 3)), blocks=blocks), 0)
    for j in range(k + 1):
        assert np.abs(C[j] - (j + 1)*sigma**2*np.eye(6)).max() <= 1e-13*(j + 1), j


def test_dense_reference_point_seen_once():
    """a point seen once through PoseToPointFactor from a pose held by a 1e-6 prior: sigma_z^2 I to rounding"""
    sz = 0.5
    rng = np.random.default_rng(3)
    X = lie.se3_exp(rng.normal(0, 0.3, (1, 6)))
    pw = np.array([[1.0, -2.0, 8.0]])
    z = lie.transform_to(X, pw)
    blocks = [FactorBlock(PRIOR6, np.array([[0]]), X, np.array([1e-6])),
              FactorBlock(POSE2POINT3, np.array([[0, 0]]), z, np.array([sz]))]
    C = _dense_cov(Problem(X, pw, blocks=blocks), 1)
    assert np.abs(C[0] - sz**2*np.eye(3)).max() <= 1e-9*sz**2


def test_gpu_graphs_reach_every_route():
    """the graphs of test_covariance_gpu.py take every landmark route: window NP = 1 and 2, simple (T > WIN_TMAX, a
    repeated pose, the flow type), general WCME and WCPE chains"""
    seen = set()
    for name, make in SI.cov_graphs().items():
        if name == "imu":            # velocities and biases: no landmark route of their own (routes() covers poses only)
            continue
        for g in SR.routes(make()):
            assert g.route != "unsupported", (name, g)
            if g.route == "window":
                seen.add("window NP = 1" if g.ftype in (POSE2POINT3, STEREO3) else "window NP = 2")
            elif g.route == "simple":
                if g.flow:
                    seen.add("simple flow")
                if g.T > SR.WIN_TMAX:
                    seen.add("simple T > WIN_TMAX")
                if g.repeated:
                    seen.add("simple repeated pose")
            elif g.route == "general":
                seen.add({TERNARY3: "general WCME", MOTIONPOSE3: "general WCPE"}.get(g.ftype, "general other"))
    want = {"window NP = 1", "window NP = 2", "simple flow", "simple T > WIN_TMAX", "simple repeated pose", "general WCME",
            "general WCPE"}
    assert want <= seen, want - seen
