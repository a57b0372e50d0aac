"""The reduced solve (csrc/kernels_band.cu: the dataflow band Cholesky, the cell scheme, the backward sweep) and
dynoba_marginal against LAPACK's band Cholesky, on the banded systems of band_reference.py: dense priors only, so the
device's S is bit-for-bit the banded assembly and the factorisation is tested alone.  Errors are in the units of
D = diag S (band_reference's comparators).

Tolerances (band_reference.TOL, per family): forward only where kappa(D^-1/2 S D^-1/2) is certified <= 100, backward
everywhere; the marginal TOL_MARG = 5e-14 in units of sqrt(S_aa S_bb).  Each is 13x to 63x the worst value measured over
every case, lambda and layout, identical on an H100 80GB HBM3 at 700 W and at 400 W:

    family        forward: worst / tol            backward: worst / tol
    dominant      3.4e-15 (c2_wb9) / 2e-13        2.0e-15 (wb16) / 1e-13
    graded        5.2e-15 (c4_wb17) / 2e-13       2.4e-15 (c4_wb17) / 1e-13
    indefinite    2.1e-15 (c2_kend17) / 1e-13     8.4e-16 (c2_kend17) / 5e-14
    nearsing      -                               3.3e-16 (nearsing_c2) / 1e-14
    laplacian     -                               7.9e-16 (laplacian_kend33) / 1e-14
    marginal      G 1.2e-15, g 3.0e-15 / 5e-14

The device's S equals the banded assembly bit for bit (dynoba_get_reduced_system), and repeated solves and other worker
splits (band_ctas_per_chain) return bit-identical steps.
"""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import band_reference as BR

pytestmark = pytest.mark.gpu

TOL_MARG = BR.TOL_MARG
_cache = {}


def _system(case):
    if case.name not in _cache:
        _cache[case.name] = BR.build(case)
    return _cache[case.name]


def _solver(sysm, extra=()):
    from dynosam_b200.binding import Solver
    c = sysm.case
    s = Solver(sysm.problem(extra))
    s.set_partition(c.cells)
    if c.outer_weight:
        s.set_tuning("outer_weight", c.outer_weight)
    if c.min_bandwidth:
        s.set_shard(0, 1, lambda *a: None, c.min_bandwidth)
    return s


def _step(s, sysm, lam):
    """dynoba_solve's pose step in solver order"""
    return s.solve(lam)[sysm.user_perm()]


def _errors(sysm, x, lam, extra=()):
    ab, g = sysm.band(lam, extra)
    bwd = BR.backward_error(ab, x, g)
    fwd = None if BR.TOL[sysm.case.family][0] is None else BR.forward_error(ab[0], x, BR.solve(ab, g))
    return fwd, bwd


def _check(family, fwd, bwd):
    tf, tb = BR.TOL[family]
    assert bwd <= tb and (tf is None or fwd <= tf), (family, fwd, bwd)


@pytest.mark.parametrize("name", [c.name for c in BR.PLAIN + BR.CELLS])
def test_solve_matches_lapack(name):
    """every case of the list at each of its lambdas: the plain band (WB 0..35, NT = 2, dense, the bandwidth clamp) and
    the cell layouts (1..16 cells, spiked chains around FF_CH, the outer weights, a clamped request)"""
    case = BR.CASES[name]
    sysm = _system(case)
    s = _solver(sysm)
    L = case.layout()
    info = s.info()
    assert info["reduced_dim"] == sysm.n and info["bandwidth"] == L.bw
    for rel in case.lambdas:
        lam = sysm.lam_abs(rel)
        fwd, bwd = _errors(sysm, _step(s, sysm, lam), lam)
        print(f"BAND {case.family} {name} lambda {rel:g}: forward {fwd if fwd is None else f'{fwd:.2e}'} backward {bwd:.2e}")
        _check(case.family, fwd, bwd)
    s.close()


@pytest.mark.parametrize("name", ["nt2_wb1", "wb9_permuted", "wb4_graded", "c2_wb9", "c4_wb3_minimal", "c4_wb3_graded_permuted"])
def test_reduced_system_is_the_banded_assembly(name):
    """dynoba_get_reduced_system equals the banded assembly bit for bit: the priors land in chain tiles, spike tiles and
    FF blocks through band_at, in user order after a permutation"""
    sysm = _system(BR.CASES[name])
    s = _solver(sysm)
    lam = sysm.lam_abs(1e-3)
    ab, g = sysm.band(lam)
    S, gS = s.reduced_system(lam)
    up = sysm.user_perm()
    Sr = np.zeros_like(S); Sr[np.ix_(up, up)] = BR.dense(ab)
    gr = np.zeros_like(gS); gr[up] = g
    assert np.array_equal(S, Sr), np.abs(S - Sr).max()
    assert np.array_equal(gS, gr), np.abs(gS - gr).max()
    s.close()


@pytest.mark.parametrize("name", ["c2_kend17", "c4_wb17"])
def test_spiked_solves_are_bit_identical(name):
    """the order of operations is fixed per tile: two solves on one handle, and other splits of the worker CTAs between
    the band and spike pools, return the same bits"""
    sysm = _system(BR.CASES[name])
    s = _solver(sysm)
    lam = sysm.lam_abs(1e-3)
    x0 = s.solve(lam)
    assert np.array_equal(s.solve(lam), x0)
    try:
        for k in (1, 3):
            s.set_tuning("band_ctas_per_chain", k)
            assert np.array_equal(s.solve(lam), x0), k
    finally:
        s.set_tuning("band_ctas_per_chain", 0)
    s.close()


# where the negative pose sits: (case, label, solver pose position from the layout)
INDEFINITE = [
    ("wb3", "tile 0", lambda L, n: 0),
    ("wb3", "last tile", lambda L, n: n - 1),
    ("c2_kend17", "tile 0", lambda L, n: 0),
    ("c2_kend17", "last tile", lambda L, n: n - 1),
    ("c2_kend17", "chain interior", lambda L, n: (L.cells[0].a0 + L.cells[0].m0)//12),
    ("c2_kend17", "middle separator M", lambda L, n: (L.cells[1].m0 + L.WB*BR.TILE//2)//6),
    ("c2_kend17", "boundary separator Q", lambda L, n: (L.cells[1].q0 + L.WB*BR.TILE//2)//6),
    ("c2_kend17", "last column of spiked chain A", lambda L, n: (L.cells[1].m0 - BR.TILE//2)//6),
    ("c2_kend17", "last column of spiked chain B", lambda L, n: (L.cells[0].m0 + L.WB*BR.TILE + BR.TILE//2)//6),
]


@pytest.mark.parametrize("name,label,where", INDEFINITE, ids=[f"{a}-{b}" for a, b, _ in INDEFINITE])
def test_indefinite_system_is_reported_then_solved(name, label, where):
    """a single-pose prior -c I makes S indefinite: DYNOBA_ERR_INDETERMINATE at lambda = 0, then the same handle solves
    at lambda = 1.5 c (positive definite) and matches LAPACK -- the fail flag is reset per call"""
    from dynosam_b200.binding import DynobaError, ERR_INDETERMINATE
    case = BR.CASES[name]
    sysm = _system(case)
    neg, c = BR.negative_prior(sysm, where(case.layout(), case.n_pose))
    s = _solver(sysm, extra=[neg])
    with pytest.raises(DynobaError) as ei:
        s.solve(0.0)
    assert ei.value.status == ERR_INDETERMINATE
    lam = 1.5*c
    fwd, bwd = _errors(sysm, _step(s, sysm, lam), lam, [neg])
    print(f"BAND indefinite {name} {label}: forward {fwd:.2e} backward {bwd:.2e}")
    _check("indefinite", fwd, bwd)
    s.close()


@pytest.mark.parametrize("label,case,k", BR.MARGINALS, ids=[m[0] for m in BR.MARGINALS])
def test_marginal_matches_dense_schur_complement(label, case, k):
    """dynoba_marginal of the last k poses (listed in another order) against S_kk - S_kr S_rr^-1 S_rk and its g"""
    sysm = _system(case)
    s = _solver(sysm)
    n_pose = case.n_pose
    ab, g = sysm.band(0.0)
    S = BR.dense(ab)
    p0 = 6*(n_pose - k)
    Gk, gk = BR.schur_marginal(S, g, p0)
    listed = np.random.default_rng(k).permutation(np.arange(n_pose - k, n_pose))
    G, gm = s.marginal(sysm.s2u[listed])
    perm = (6*(listed[:, None] - (n_pose - k)) + np.arange(6)[None, :]).reshape(-1)
    d = np.sqrt(ab[0, p0:])[perm]
    eG = float((np.abs(G - Gk[np.ix_(perm, perm)])/d[:, None]/d[None, :]).max())
    eg = float((np.abs(gm - gk[perm])/d).max()/(np.abs(gk)[perm]/d).max())
    print(f"BAND marginal {label}: G {eG:.2e} g {eg:.2e}")
    assert eG <= TOL_MARG and eg <= TOL_MARG, (eG, eg)
    s.close()


def test_marginal_refusals():
    """a kept block one tile wider than WB + 1 is refused; an indefinite eliminated block is reported"""
    from dynosam_b200.binding import DynobaError, ERR_INDETERMINATE, ERR_UNSUPPORTED
    sysm = _system(BR.MARGINAL_BASE)
    n_pose = BR.MARGINAL_BASE.n_pose
    s = _solver(sysm)
    with pytest.raises(DynobaError) as ei:
        s.marginal(sysm.s2u[np.arange(n_pose - 13, n_pose)])
    assert ei.value.status == ERR_UNSUPPORTED
    s.close()
    neg, _ = BR.negative_prior(sysm, 5)
    s = _solver(sysm, extra=[neg])
    with pytest.raises(DynobaError) as ei:
        s.marginal(sysm.s2u[np.arange(n_pose - 7, n_pose)])
    assert ei.value.status == ERR_INDETERMINATE
    s.close()


PROFILE_CASES = ["one_pose", "wb35", "c1_wb1", "c2_wb1_gq1", "c2_kend17", "c3_wb2_clamped", "c4_wb3_minimal", "c16_wb1"]
_PROFILE_SCRIPT = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import band_reference as BR
from dynosam_b200.binding import Solver
for name in sys.argv[1:]:
    case = BR.CASES[name]
    sysm = BR.build(case)
    s = Solver(sysm.problem())
    s.set_partition(case.cells)
    if case.outer_weight:
        s.set_tuning("outer_weight", case.outer_weight)
    s.set_tuning("band_profile", 1)
    print("CASE", name, file=sys.stderr, flush=True)
    s.solve(sysm.lam_abs(1e-3))
    s.close()
"""


def test_mirror_matches_the_device_layout(tmp_path):
    """the band profile (process-wide once on, hence a subprocess) prints every factorisation launch with the WB and the
    columns / spike of each of its problems: chains, cell separator systems and boundary system equal the mirror's"""
    tests = os.path.dirname(os.path.abspath(__file__))
    script = tmp_path / "profile.py"
    script.write_text(_PROFILE_SCRIPT.format(root=os.path.dirname(tests), tests=tests))
    r = subprocess.run([sys.executable, str(script), *PROFILE_CASES], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got, cur = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("CASE "):
            cur = got.setdefault(line.split()[1], [])
        elif m := re.match(r"\[band\]\s+launch: (\d+) problems, WB (\d+),", line):
            cur.append((int(m.group(2)), int(m.group(1)), []))
        elif m := re.match(r"\[band\]\s+spine \d+ \((\d+) columns(, spiked)?\)", line):
            cur[-1][2].append((int(m.group(1)), m.group(2) is not None))
    assert sorted(got) == sorted(PROFILE_CASES)
    for name in PROFILE_CASES:
        want = [(wb, len(p), p) for wb, p in BR.launches(BR.CASES[name].layout())]
        assert got[name] == want, (name, got[name], want)
