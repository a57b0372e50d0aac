"""The visual-inertial kernels on the device, case by case (tests/imu_cases.py) against the 50-digit reference
(tests/imu_lie_reference.py), through dynosam_b200.binding.Solver only: imu_kernel (J, b, per-factor error, chi^2),
vec_prior_kernel<3/6> (b and J bit for bit), nav_factors_kernel's scatter into the reduced system at every store
branch, the inert velocity scalars and nav_retract_kernel.

Errors are in units of the a-priori bound of imu_cases' docstring, so a tolerance of 16 means 16 x that bound's unit.
Each case prints `IMU H100 <case>: ...`.

Worst measured / tolerance, NVIDIA H100 80GB HBM3, power limit 700 W:

    family                                   b            A            factor error   chi^2 (relative)
    theta (bias-correction angle)            0.68 / 16    0.67 / 16    0.036 / 8      2.4e-11
    phi (every Logmap branch, straddles)     0.60 / 16    0.86 / 16    0.030 / 8      1.0e-5 (phi = pi - 1e-5)
    res (residual rotation)                  0.40 / 16    0.48 / 16    0.070 / 8      7.0e-11
    dt, g, |t| = 1e3                         0.46 / 16    0.99 / 16    0.066 / 8      8.3e-13
    R kinds and scales                       0.08 / 16    0.19 / 16    0.007 / 8      1.6e-15
    priors                                   0 (bits)     0 (bits)     0.22 / 8       2.2e-16
    blocks, big (4096 / 4097), shuffled      0.18 / 16    0.17 / 16    0.22 / 8       1.9e-15
    scatter (S, g_S vs dense, 16 layouts)    4.7e-16 of sqrt(S_aa S_bb) / 1e-14
    inert scalars (step vs dense solve)      2.0e-15 / 1e-8

chi^2 is held to n_partials eps plus the summed per-factor differences (which the factor-error column bounds); the
large relative chi^2 of a few cases is that sum, at their small chi^2.
"""
import numpy as np
import pytest

import imu_cases as IC
from dynosam_b200.problem import COMBINED_IMU15, PRIOR6, PRIOR_BIAS6, PRIOR_VEL3, SLOT_CLASS, FactorBlock, Problem

pytestmark = pytest.mark.gpu

CASES = IC.cases()
EPS = 2.0**-52


def _solver(p):
    from dynosam_b200.binding import Solver
    return Solver(p)


def _warp_sum_of_halves(b):
    """imu_kernel's warp_sum_d(0.5 rw^2) for lane 0, in its butterfly order: lanes 0..14 hold 0.5 rw^2, the rest 0"""
    v = np.zeros(32); v[:15] = 0.5*b*b
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[lanes ^ o]
    return v[0]


@pytest.mark.parametrize("name", list(CASES))
def test_linearization_and_errors(name):
    c = CASES[name]
    s = _solver(c.problem)
    s.linearize()
    e = [s.error() for _ in range(3)]
    assert e[0] == e[1] == e[2], e                               # the reduction order is fixed: same bits call to call
    IC.check_problem(c, s.linearization, s.factor_errors, e[0], "H100")
    for bi, blk in enumerate(c.problem.blocks):
        if blk.type != COMBINED_IMU15:
            continue
        # the WJ = true (linearize) and WJ = false (error) instantiations form r_w alike: the error sweep's per-factor
        # error is the warp sum of the linearisation's b, bit for bit
        _, b = s.linearization(bi); ef = s.factor_errors(bi)
        want = np.array([_warp_sum_of_halves(b[f]) for f in range(blk.n)])
        assert np.array_equal(ef, want), (name, np.abs(ef - want).max())
    s.close()


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith(("blocks_imu", "big_", "blocks_shuffled"))])
def test_copies_equal_the_factor_alone(name):
    """a factor's outputs do not depend on its slot: every tiled copy equals that factor evaluated alone (n = 1), bits"""
    c = CASES[name]; p = c.problem
    s = _solver(p); s.linearize()
    for bi, blk in enumerate(p.blocks):
        if blk.type != COMBINED_IMU15:
            continue
        A, b = s.linearization(bi); e = s.factor_errors(bi)
        pick = c.pick[bi]
        for d in sorted(set(int(x) for x in pick)):
            f = int(np.flatnonzero(pick == d)[0])
            sig = blk.sigma if blk.sigma_bcast else blk.sigma[f:f + 1]
            one = FactorBlock(blk.type, blk.idx[f:f + 1], blk.meas[f:f + 1], sig)
            q = Problem(p.pose, p.point, blocks=[one], vel=p.vel, bias=p.bias)
            t = _solver(q); t.linearize()
            A1, b1 = t.linearization(0); e1 = t.factor_errors(0)
            same = np.flatnonzero(pick == d)
            assert np.array_equal(A[same], np.broadcast_to(A1, A[same].shape)), (name, bi, d)
            assert np.array_equal(b[same], np.broadcast_to(b1, b[same].shape)), (name, bi, d)
            assert np.array_equal(e[same], np.broadcast_to(e1, e[same].shape)), (name, bi, d)
            t.close()
    s.close()


# ---------------------------------------------------------------------------------------------- scatter, inert, retract
def _graph(n_frames, seed=31, same_pose=True):
    """an IMU chain over n_frames frames, a velocity and a bias prior on every frame, one factor with the same pose in
    both pose slots and b_i == b_j (nav_factors_kernel's a == b store, with its c == c2 doubling)"""
    ch = IC.Chain(seed)
    j = None
    for k in range(n_frames - 1):
        j = ch.factor(j, theta=("1e-4", "0.3", "2e-5")[k % 3], phi="0.2", res="1e-2")
    R = IC.sqrt_info("cholesky", np.random.default_rng(seed))
    facs = list(ch.fac)
    if same_pose:
        k = n_frames//2
        facs.append(([k, k, k, k + 1, k, k], facs[0][1]))
    n = len(ch.pose)
    rng = np.random.default_rng(seed + 1)
    blocks = [ch.block(R, facs),
              FactorBlock(PRIOR_VEL3, np.arange(n)[:, None], np.array(ch.vel) + rng.normal(0, 0.1, (n, 3)), np.array([0.5])),
              FactorBlock(PRIOR_BIAS6, np.arange(n)[:, None], np.array(ch.bias) + rng.normal(0, 0.01, (n, 6)), np.array([0.1]*3 + [0.02]*3))]
    return ch.problem(blocks)


def _dense(p, s, lam):
    """J^T J + lam I and J^T b over [poses 6 | velocities 3 | biases 6] from the device's own J and b"""
    base = {0: 0, 3: 6*p.n_pose, 4: 6*p.n_pose + 3*p.n_vel}
    dim = {0: 6, 3: 3, 4: 6}
    n = 6*p.n_pose + 3*p.n_vel + 6*p.n_bias
    H = np.zeros((n, n)); g = np.zeros(n)
    for bi, blk in enumerate(p.blocks):
        A, b = s.linearization(bi)
        for f in range(blk.n):
            cols = []
            for k, c in enumerate(SLOT_CLASS[blk.type]):
                o = base[c] + dim[c]*blk.idx[f, k]
                cols.extend(range(o, o + dim[c]))
            np.add.at(H, np.ix_(cols, cols), A[f].T@A[f])
            np.add.at(g, cols, A[f].T@b[f])
    return H + lam*np.eye(n), g


ORDERS = {
    "frame": lambda n: (np.arange(n), np.arange(n), np.arange(n)),
    "poses_reversed": lambda n: (n - 1 - np.arange(n), np.arange(n), np.arange(n)),        # X_j before X_i: a < b
    "bias_reversed": lambda n: (np.arange(n), np.arange(n), n - 1 - np.arange(n)),         # b_j before b_i
    "kinds_apart": lambda n: (np.arange(n), np.arange(n) + n, 2*n - 1 - np.arange(n)),     # V after every X
}


@pytest.mark.parametrize("ncells", [-1, 0, 2, 4])
@pytest.mark.parametrize("order", list(ORDERS))
def test_scatter_reaches_every_store_branch(order, ncells):
    """reduced_system(lam)'s S and g_S against a dense assembly of the device's own J and b, in units of
    sqrt(S_aa S_bb) (a tolerance, not bits: the order of the fp64 RED atomics changes from run to run)"""
    p = _graph(24)
    p.pose_order, p.vel_order, p.bias_order = (x.astype(np.int32) for x in ORDERS[order](p.n_pose))
    s = _solver(p)
    s.set_partition(ncells)
    s.linearize()
    worst = 0.0
    for lam in (0.0, 1e-3, 1e4):
        H, g = _dense(p, s, lam)
        S, gS = s.reduced_system(lam)
        d = np.sqrt(np.diag(H))
        errS = (np.abs(S - H)/np.outer(d, d)).max(); errg = (np.abs(gS - g)/d).max()/max(1.0, (np.abs(g)/d).max())
        worst = max(worst, errS, errg)
        assert errS <= 1e-14 and errg <= 1e-14, (order, ncells, lam, errS, errg)
    print(f"IMU H100 scatter {order} cells={ncells}: {worst:.2g} of sqrt(S_aa S_bb)")
    s.close()


@pytest.mark.parametrize("n_vel", [42, 43])
def test_inert_scalars_neither_couple_nor_damp(n_vel):
    """the three inert scalars of each velocity block hold a unit diagonal, zero coupling and zero rhs at every lambda:
    the step equals the dense solve over the used scalars, λ = 0 included (a missing unit diagonal is a zero pivot);
    3 n_vel = 126 / 129 threads straddle nav_inert_kernel's 128-thread grid"""
    p = _graph(n_vel, same_pose=False)
    assert p.n_vel == n_vel
    p.blocks.append(FactorBlock(PRIOR6, np.arange(p.n_pose)[:, None], p.pose, np.array([1.0])))     # (fixes the gauge)
    s = _solver(p)
    s.set_partition(-1)
    s.linearize()
    for lam in (0.0, 1e-3, 1e4):
        H, g = _dense(p, s, lam)
        ref = np.linalg.solve(H, g)
        d = s.solve(lam)
        np_, nv = 6*p.n_pose, 3*p.n_vel
        got = np.concatenate([d[:np_], d[np_:np_ + nv], d[np_ + nv:]])
        dd = np.sqrt(np.diag(H))
        err = (np.abs(got - ref)*dd).max()/(np.abs(ref)*dd).max()
        print(f"IMU H100 inert n_vel={n_vel} lambda={lam:g}: step {err:.2g}")
        assert np.isfinite(got).all() and err <= 1e-8, (lam, err)
    s.close()


@pytest.mark.parametrize("n_nav", [127, 128, 129])
def test_retract_adds_bit_for_bit(n_nav):
    """after retract(delta), velocities and biases are numpy's x + delta bit for bit (n_vel + n_bias straddles
    nav_retract_kernel's 128-thread grid) and the poses are untouched by the navigation step"""
    nv = (n_nav + 1)//2; nb = n_nav - nv
    p = _graph(max(nv, nb))
    p.vel = p.vel[:nv]; p.bias = p.bias[:nb]
    p.blocks = [FactorBlock(PRIOR_VEL3, np.arange(nv)[:, None], p.vel + 0.1, np.array([0.5])),
                FactorBlock(PRIOR_BIAS6, np.arange(nb)[:, None], p.bias + 0.01, np.array([0.1]))]
    s = _solver(p)
    rng = np.random.default_rng(n_nav)
    delta = np.zeros(6*p.n_pose + 3*nv + 6*nb)
    delta[6*p.n_pose:] = rng.normal(0, 1, 3*nv + 6*nb)*np.exp(rng.uniform(-20, 5, 3*nv + 6*nb))
    s.retract(delta)
    vel, bias = s.nav_values(); pose, _, _ = s.values()
    assert np.array_equal(vel, p.vel + delta[6*p.n_pose:6*p.n_pose + 3*nv].reshape(nv, 3))
    assert np.array_equal(bias, p.bias + delta[6*p.n_pose + 3*nv:].reshape(nb, 6))
    assert np.array_equal(pose, p.pose)
    s.close()
