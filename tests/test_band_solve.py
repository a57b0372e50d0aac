"""CPU checks of band_reference.py: the reference solves its systems, the comparators see a dropped band tile and a
1e-10 perturbation, the layout mirror equals the library's own partition, and the case list reaches every boundary."""
import numpy as np
import pytest

import band_reference as BR


def _small(name):
    s = BR.build(BR.CASES[name])
    ab, g = s.band(s.lam_abs(1e-3))
    return s, ab, g


@pytest.mark.parametrize("name", ["nt2_wb1", "wb3", "wb9_permuted", "wb4_graded", "c4_wb3_minimal"])
def test_reference_solves_the_dense_system(name):
    s, ab, g = _small(name)
    x = BR.solve(ab, g)
    S = BR.dense(ab)
    d = np.sqrt(ab[0])                                          # dense LU on the equilibrated system: graded rows too
    xd = np.linalg.solve(S/d[:, None]/d[None, :], g/d)/d
    assert BR.forward_error(ab[0], x, xd) <= 1e-14
    assert BR.backward_error(ab, x, g) <= 1e-15
    assert np.abs(BR.matvec(ab, x) - S @ x).max() <= 1e-12*np.abs(S @ x).max()
    assert BR.certified_kappa(ab) <= 100


def test_backward_error_is_scale_invariant():
    """the same system scaled by 10^U(-6, 6) per pose: the errors, in units of diag S, do not change"""
    s, ab, g = _small("wb3")
    x = BR.solve(ab, g)
    rng = np.random.default_rng(3)
    d = np.repeat(10.0**rng.uniform(-6, 6, s.case.n_pose), 6)
    abs_ = ab.copy()
    for k in range(ab.shape[0]):
        abs_[k, :s.n - k] *= d[:s.n - k]*d[k:]
    y = x/d
    assert abs(BR.backward_error(abs_, y, g*d) - BR.backward_error(ab, x, g)) <= 1e-15
    xp = x*(1 + 1e-9*rng.standard_normal(x.size))
    assert abs(BR.forward_error(abs_[0], xp/d, y) - BR.forward_error(ab[0], xp, x)) <= 1e-15


@pytest.mark.parametrize("name", ["wb3", "wb9_permuted", "c2_wb9"])
def test_comparators_reject_a_dropped_far_tile(name):
    """the solution of S with one tile of the outermost band offset zeroed fails both comparators by orders of
    magnitude over the GPU tolerances"""
    s, ab, g = _small(name)
    WB = s.fill_WB
    bad = ab.copy()
    K = _far_columns(ab, WB)
    K = K[K.size//2]                                            # a filled column tile in the middle
    for d in range(ab.shape[0]):
        j = np.arange(K*BR.TILE, min((K + 1)*BR.TILE, s.n - d))
        j = j[(j + d)//BR.TILE - K == WB]
        bad[d, j] = 0.0
    assert (bad != ab).any()
    x, xb = BR.solve(ab, g), BR.solve(bad, g)
    fwd, bwd = BR.forward_error(ab[0], xb, x), BR.backward_error(ab, xb, g)
    tf, tb = BR.TOL[s.case.family]
    assert fwd >= 1e4*tf and bwd >= 1e4*tb, (fwd, bwd)


def _far_columns(ab, WB):
    """column tiles with a non-zero entry in the outermost tile offset WB"""
    n = ab.shape[1]
    K = set()
    for d in range(ab.shape[0]):
        j = np.flatnonzero(ab[d, :n - d] != 0)
        K.update((j[(j + d)//BR.TILE - j//BR.TILE == WB]//BR.TILE).tolist())
    return np.array(sorted(K))


@pytest.mark.parametrize("name", ["wb3", "wb17_graded", "c4_wb3_minimal"])
def test_comparators_reject_a_small_perturbation_of_the_last_tile(name):
    """one entry of the outermost band tile off by 1e-10 of sqrt(S_ii S_jj) (the entry that meets the largest scaled
    solution component): both comparators notice"""
    s, ab, g = _small(name)
    x = BR.solve(ab, g)
    xs = np.abs(np.sqrt(ab[0])*x)
    n, best = s.n, (-1.0, 0, 0)
    for d in range(ab.shape[0]):
        j = np.flatnonzero(ab[d, :n - d] != 0)
        j = j[(j + d)//BR.TILE - j//BR.TILE == s.fill_WB]
        if j.size:
            k = j[np.argmax(np.maximum(xs[j], xs[j + d]))]
            best = max(best, (max(xs[k], xs[k + d]), d, int(k)))
    _, d, j = best
    bad = ab.copy()
    bad[d, j] += 1e-10*np.sqrt(ab[0, j]*ab[0, j + d])
    xb = BR.solve(bad, g)
    fwd, bwd = BR.forward_error(ab[0], xb, x), BR.backward_error(ab, xb, g)
    tf, tb = BR.TOL[s.case.family]
    assert fwd >= 10*tf and bwd >= 10*tb, (fwd, bwd)


def test_mirror_equals_plan_partition():
    """the mirror's multi-rank branch against dynoba_plan_partition, a pure host function of the library"""
    from dynosam_b200.binding import plan_partition
    for n_poses in (5, 60, 301, 2000, 6007, 22000):
        for bw in (0, 5, 31, 33, 95, 200, 959):
            for world in (1, 2, 3, 4, 8, 16):
                assert np.array_equal(BR.plan_partition(n_poses, bw, world), plan_partition(n_poses, bw, world)), (n_poses, bw, world)


def test_mirror_is_consistent():
    """chains tile the system, spiked chains sit next to boundary separators, no chain is shorter than max(WB, 2)"""
    for c in BR.CASES.values():
        L = c.layout()
        if L.C == 0:
            assert [(ch.NT, ch.Kend) for ch in L.chains] == [(L.NT, L.NT)]
            continue
        assert sum(ch.Kend for ch in L.chains) + (2*L.C - 1)*L.WB == L.NT
        assert all(ch.Kend >= max(L.WB, 2) for ch in L.chains)
        for k, g in enumerate(L.cells):
            assert L.chains[2*k].spiked == (k > 0) and L.chains[2*k + 1].spiked == (k < L.C - 1)
            assert g.m0 - g.a0 == BR.TILE*L.chains[2*k].Kend and g.b1 - g.m0 - L.WB*BR.TILE == BR.TILE*L.chains[2*k + 1].Kend


def test_cases_reach_every_boundary():
    """every case reaches the boundaries it names (by the mirror), and together they reach every listed boundary; a
    spike-chunk boundary counts only for the cases that name it, whose chunks test_spiked_cases_see_their_last_chunks
    shows to be visible"""
    seen = set()
    for c in BR.CASES.values():
        h = BR.boundaries(c.layout(), c.min_bandwidth)
        assert set(c.hits) <= h, (c.name, set(c.hits) - h)
        seen |= {b for b in h if b not in BR.SPIKE_BOUNDARIES or b in c.hits}
    missing = set(BR.REQUIRED) - seen
    assert not missing, missing
    assert all(h in BR.REQUIRED for c in BR.CASES.values() for h in c.hits)


@pytest.mark.parametrize("name", [c.name for c in BR.CASES.values() if set(c.hits) & set(BR.SPIKE_BOUNDARIES)])
def test_spiked_cases_see_their_last_chunks(name):
    """the solve with the last FF chunk, or the last spike-forward chunk, of a spiked chain left out misses the case's
    backward tolerance by more than 100x, while the exact solve meets it: a skipped or shortened last chunk fails"""
    s = BR.build(BR.CASES[name])
    ff, sf, exact = BR.dropped_chunk_errors(s)
    tol = BR.TOL[s.case.family][1]
    assert ff >= 100*tol and sf >= 100*tol and exact <= tol, (ff, sf, exact)


def test_marginal_cases_reach_their_boundaries():
    got = set()
    for label, case, k in BR.MARGINALS:
        L = case.layout()
        p0 = 6*(case.n_pose - k)
        K0 = p0//BR.TILE
        assert L.C == 0 and L.NT - K0 <= L.WB + 1, label
        got.add(p0 % BR.TILE)
        if k == case.n_pose:
            assert K0 == 0 and L.WB == L.NT - 1
        if L.NT - K0 == L.WB + 1:
            got.add("WB + 1")
    assert {0, 2, 30, "WB + 1"} <= got
    base = BR.MARGINAL_BASE.layout()
    assert base.NT - 6*(BR.MARGINAL_BASE.n_pose - 13)//BR.TILE == base.WB + 2     # the refused width


def test_families():
    """dominant and graded are certified (kappa <= 100 in diag units), near-singular is not, the negative prior makes S
    indefinite and lambda = 1.5 c positive definite again"""
    for name in ("wb7", "wb17_graded", "c2_kend15"):
        s = BR.build(BR.CASES[name])
        for rel in BR.CASES[name].lambdas:
            ab, _ = s.band(s.lam_abs(rel))
            assert BR.certified_kappa(ab) <= 100, (name, rel)
    s = BR.build(BR.CASES["nearsing_wb3"])
    ab, _ = s.band(0.0)
    ev = np.linalg.eigvalsh(BR.dense(ab))
    dg = np.sqrt(ab[0])
    evs = np.linalg.eigvalsh(BR.dense(ab)/dg[:, None]/dg[None, :])
    assert ev.min() > 0 and 1e8 <= evs.max()/evs.min() <= 1e12, evs.max()/evs.min()
    s = BR.build(BR.CASES["wb3"])
    neg, c = BR.negative_prior(s, 40)
    ab, _ = s.band(0.0, extra=[neg])
    assert np.linalg.eigvalsh(BR.dense(ab)).min() < 0
    ab, _ = s.band(1.5*c, extra=[neg])
    assert np.linalg.eigvalsh(BR.dense(ab)).min() > 0 and BR.certified_kappa(ab) <= 100
