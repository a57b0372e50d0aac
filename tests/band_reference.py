"""Banded fp64 reference of the reduced solve (csrc/kernels_band.cu), a mirror of its layout, and seeded banded SPD systems
that reach every boundary of that layout.

Systems.  No landmarks and no factor blocks: n_pose poses at the identity and a list of dense priors
(dynoba_add_linear_prior).  A prior is a window of `span` consecutive solver positions with a dense symmetric G; windows
start every `stride` poses, so the filled band reaches bw = 6 (span - 1) + 5, the bandwidth the layout is cut for.  Each
prior is linearised at its poses' current values, so its right-hand side is g itself.  The device adds the priors to the
band in stream order, each entry at most once per launch, after writing lambda on the diagonal: S is bit-for-bit the
banded assembly below, and the tests see the factorisation alone.  Families:
    dominant     zero-diagonal random G; each scalar's first prior carries a diagonal t = 1.0205 max_i sum_j!=i |S_ij|, so
                 the Gershgorin discs of D^-1/2 S D^-1/2 (D = diag S) certify kappa <= 99 for every lambda >= 0
    graded       the same with every pose scaled by 10^U(-6, 6): S -> D S D, as 1e-6-sigma priors make it
    nearsing     G = A A^T of rank 0.4 of its size (the sum stays singular) plus eps on the diagonal: kappa_s ~ 1e10
    laplacian    G = a weighted graph Laplacian over the window's poses plus eps on the diagonal: its near-null mode is
                 constant along the time axis, so the spike of a chain next to a boundary separator does not decay with
                 the chain's length (in the other families it falls below rounding within about 16 columns)
    indefinite   dominant, plus one single-pose prior -c I (c = 2 lambda_max of that pose's diagonal block)

Comparators, in units of D = diag S (invariant under diagonal scaling):
    forward    max_a sqrt(S_aa) |x_a - x_ref,a| / max_a sqrt(S_aa) |x_ref,a|
    backward   ||D^-1/2 (S x - g)||_inf / (||D^-1/2 S D^-1/2||_inf ||D^1/2 x||_inf + ||D^-1/2 g||_inf)

Layout mirror.  ``layout`` restates band_plan_layout (chains, cell separator systems, boundary system) and
``plan_partition`` dynoba_plan_partition; the constants are read from the CUDA sources, so the boundary cases move with
them.  ``boundaries`` names what a layout exercises in the kernels.
"""
from __future__ import annotations

import dataclasses

import numpy as np
import scipy.linalg as sla

from schur_reference import _const

TILE = _const("internal.cuh", r"constexpr int TILE = (\d+);")
MAX_CELLS = _const("internal.cuh", r"constexpr int MAX_CELLS = (\d+);")
FF_CH = _const("kernels_band.cu", r"constexpr int FF_CH = (\d+);")
SPK_ROWS = _const("kernels_band.cu", r"constexpr int SPK_ROWS = (\d+);")
SF_CH = _const("kernels_band.cu", r"constexpr int SF_CH = (\d+);")
BW_CL, BW_TW = _const("kernels_band.cu", r"constexpr int BW_CL = (\d+), BW_TW = (\d+);", 2)
MAX_PRIOR_POSES = _const("api.cu", r"ARG\(h, \"null handle\"\); ARG\(n > 0 && n <= (\d+) && pose_idx")

# tolerances of test_band_solve_gpu.py per family, (forward, backward) in the units above; forward only where kappa is
# certified <= 100.  Its docstring has the measured values they come from.
TOL = {"dominant": (2e-13, 1e-13), "graded": (2e-13, 1e-13), "indefinite": (1e-13, 5e-14), "nearsing": (None, 1e-14),
       "laplacian": (None, 1e-14)}
TOL_MARG = 5e-14         # dynoba_marginal, units sqrt(S_aa S_bb)

IDENTITY = np.array([1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0, 0, 0, 0])


# ------------------------------------------------------------------------------------------------------------ layout mirror
@dataclasses.dataclass
class Chain:
    NT: int
    Kend: int
    spiked: bool
    TPC: int


@dataclasses.dataclass
class Cell:
    q0: int
    a0: int
    m0: int
    b1: int
    has_qa: bool
    has_qb: bool


@dataclasses.dataclass
class Layout:
    n: int
    bw: int
    NT: int
    WB: int
    n_pad: int
    cmax_raw: int          # feasible cells before the MAX_CELLS clamp
    cmax: int
    request: int
    C: int
    chains: list
    cells: list
    cs: list
    gq: list
    WBcs: int = 0
    TPCcs: int = 0
    NTgq: int = 0
    WBgq: int = 0
    TPCgq: int = 0
    outer_weight: float = 0.0


def layout(n, bw, ncell_request=-1, outer_weight=0.0, world=1):
    """band_plan_layout for one rank's view (every cell; chains 2c = A, 2c + 1 = B of cell c)"""
    bw = max(0, min(bw, max(n - 1, 0)))
    NT = max(-(-n//TILE), 1)
    WB = -(-bw//TILE)
    if NT > 1 and WB < 1:
        WB = 1
    WB = min(WB, NT - 1)
    minlen = max(WB, 2)
    raw = (NT + WB)//(2*WB + 2*minlen) if WB >= 1 else 0
    cmax = min(raw, MAX_CELLS)
    if ncell_request > 0:
        C = min(ncell_request, cmax)
    elif ncell_request < 0:
        C = 0
    else:
        C = min(world, cmax) if world > 1 else (2 if NT >= 4096 and cmax >= 2 else 1)
        if NT < max(8, 4*WB + 4):
            C = 0
        C = min(C, cmax)
    L = Layout(n, bw, NT, WB, NT*TILE, raw, cmax, ncell_request, C, [], [], [], [], outer_weight=outer_weight)
    if C == 0:
        L.chains.append(Chain(NT, NT, False, WB + 1))
        return L
    free = NT - (2*C - 1)*WB
    wgt = [1.0]*(2*C)
    if outer_weight > 0 or world == 1 or C != world:
        wgt[0] = wgt[-1] = outer_weight if outer_weight > 0 else (4.5 if C >= 2 else 1.0)
    else:
        wgt = [0.5]*(2*C)
        wgt[0] = wgt[-1] = 1.24
        wgt[1] = wgt[-2] = 0.6
    wsum = 0.0
    for x in wgt:
        wsum += x
    ln = [max(minlen, int(float(free)*w/wsum)) for w in wgt]
    used, k = sum(ln), 0
    while used < free:
        ln[k] += 1; used += 1; k = (k + 1) % (2*C)
    k = 0
    while used > free:
        if ln[k] > minlen:
            ln[k] -= 1; used -= 1
        k = (k + 1) % (2*C)
    t = 0
    for c in range(C):
        qa, qb = c > 0, c < C - 1
        q0 = t*TILE
        if c > 0:
            t += WB
        a0 = t*TILE; t += ln[2*c]
        m0 = t*TILE; t += WB + ln[2*c + 1]
        L.cells.append(Cell(q0, a0, m0, t*TILE, qa, qb))
        L.chains.append(Chain(ln[2*c] + WB, ln[2*c], qa, WB + 1 + (WB if qa else 0)))
        L.chains.append(Chain(ln[2*c + 1] + WB, ln[2*c + 1], qb, WB + 1 + (WB if qb else 0)))
    if t != NT:
        raise ValueError("band layout failed")
    L.WBcs = max(1, (3 if C >= 2 else 1)*WB - 1); L.TPCcs = L.WBcs + 1
    L.cs = [Chain(WB*(1 + g.has_qa + g.has_qb), WB, False, L.TPCcs) for g in L.cells]
    L.NTgq = (C - 1)*WB
    if C >= 2:
        L.WBgq = max(1, min(2*WB - 1, L.NTgq - 1)); L.TPCgq = L.WBgq + 1
        L.gq = [Chain(L.NTgq, L.NTgq, False, L.TPCgq)]
    else:
        L.WBgq, L.TPCgq = 0, 1
    return L


def plan_partition(n_poses, bw, world):
    """dynoba_plan_partition: first pose position of every rank's cells, [world + 1]"""
    L = layout(6*n_poses, bw, 0, 0.0, world)
    b = [L.n_pad]*(world + 1)
    b[0] = 0
    for c in range(L.C - 1, -1, -1):
        b[c*world//L.C] = 0 if c == 0 else L.cells[c].q0
    for r in range(world - 1, 0, -1):
        b[r] = min(b[r], b[r + 1])
    out = [min(x//6, n_poses) for x in b]
    out[world] = n_poses
    return np.array(out, np.int32)


def launches(L):
    """the factorisation launches of one damped solve: [(WB, [(Kend, spiked) per problem])]"""
    out = [(L.WB, [(c.Kend, c.spiked) for c in L.chains])]
    if L.C:
        out.append((L.WBcs, [(c.Kend, c.spiked) for c in L.cs]))
    if L.C >= 2:
        out.append((L.WBgq, [(c.Kend, c.spiked) for c in L.gq]))
    return out


def boundaries(L, min_bandwidth=0):
    """the named boundaries of the band kernels this layout reaches"""
    h = set()
    if L.WB == 0:
        h.add("one tile (WB = 0)")
    if L.NT == 2:
        h.add("NT = 2")
    if L.WB == 2:
        h.add("WB = 2 (spine owns dd <= 2)")
    if L.WB > BW_CL*BW_TW:
        h.add("WB > 32 (backward q loop)")
    if L.C == 0 and L.NT >= 2 and L.WB == L.NT - 1:
        h.add("dense band (WB = NT - 1)")
    if min_bandwidth > L.n - 1:
        h.add("min_bandwidth above n - 1")
    if L.C == MAX_CELLS:
        h.add("16 cells")
    if L.cmax_raw > MAX_CELLS and L.C:
        h.add("cmax clamped to MAX_CELLS")
    if L.C >= 2 and L.WB <= 3:
        h.add("cells with WB <= 3")
    if L.C == 1:
        h.add("1 cell")
    for c in (2, 3, 4, 8):
        if L.C == c:
            h.add(f"{c} cells")
    if L.NTgq == 1:
        h.add("one-tile boundary system")
    if L.request > L.cmax and L.C:
        h.add("request above cmax")
    if L.C and L.C == L.cmax and all(c.Kend == max(L.WB, 2) for c in L.chains):
        h.add("cmax with minimal chains")
    for c in L.chains:
        if c.spiked:
            for k, name in ((FF_CH - 1, "< 16"), (FF_CH, "16"), (FF_CH + 1, "17"), (2*FF_CH, "32"), (2*FF_CH + 1, "33")):
                if (c.Kend < FF_CH if name == "< 16" else c.Kend == k):
                    h.add(f"spiked Kend {name}")
            if L.WB % SPK_ROWS:
                h.add("spiked, WB % SPK_ROWS != 0")
            if c.Kend % SF_CH:
                h.add("spiked, partial spike-forward chunk")
        # the backward sweep solves two columns per cluster barrier: a chain's sweep covers its Kend factored columns
        # (Kend = NT for the plain band), so an odd count leaves one column for the last barrier
        h.add("backward sweep, odd column count" if c.Kend % 2 else "backward sweep, even column count")
    if L.C >= 2:
        ow = L.outer_weight
        h.add("outer_weight default" if ow <= 0 else f"outer_weight {ow:g}")
    return h


REQUIRED = [
    "one tile (WB = 0)", "NT = 2", "WB = 2 (spine owns dd <= 2)", "WB > 32 (backward q loop)", "dense band (WB = NT - 1)",
    "min_bandwidth above n - 1", "1 cell", "2 cells", "3 cells", "4 cells", "8 cells", "16 cells",
    "cmax clamped to MAX_CELLS", "cells with WB <= 3", "one-tile boundary system", "request above cmax",
    "cmax with minimal chains", "spiked Kend < 16", "spiked Kend 16", "spiked Kend 17", "spiked Kend 32",
    "spiked Kend 33", "spiked, WB % SPK_ROWS != 0", "spiked, partial spike-forward chunk",
    "backward sweep, odd column count", "backward sweep, even column count",
    "outer_weight default", "outer_weight 1", "outer_weight 12",
]


# ------------------------------------------------------------------------------------------------------------ systems
@dataclasses.dataclass
class Case:
    name: str
    family: str                 # dominant | graded | nearsing | indefinite
    n_pose: int
    span: int
    cells: int = -1             # dynoba_set_partition
    outer_weight: float = 0.0   # dynoba_set_tuning("outer_weight"), 0 = default
    lambdas: tuple = (0.0, 1e-3, 1e2)   # relative to the median diagonal of S at lambda = 0
    min_bandwidth: int = 0
    permute: bool = False
    seed: int = 0
    hits: tuple = ()            # boundaries the case is meant to reach (checked against the mirror)

    @property
    def bw(self):
        return max(6*(min(self.span, self.n_pose) - 1) + 5, self.min_bandwidth)

    def layout(self):
        return layout(6*self.n_pose, self.bw, self.cells, self.outer_weight)


def _n_pose(NT):
    """the most poses whose system has NT tiles, one fewer when that fills the last tile exactly"""
    n = 32*NT//6
    return n - 1 if (6*n) % TILE == 0 else n


def _span(WB):
    """the widest prior window whose band has WB tiles: bw = 6 span - 1 <= 32 WB"""
    return (TILE*WB + 1)//6


def _windows(n_pose, span):
    span = min(span, n_pose)
    stride = max(1, span//2)
    starts = list(range(0, n_pose - span + 1, stride))
    if starts[-1] != n_pose - span:
        starts.append(n_pose - span)
    return [np.arange(s, s + span) for s in starts]


@dataclasses.dataclass
class System:
    case: Case
    n: int
    s2u: np.ndarray             # user pose index of each solver position
    pose_order: np.ndarray      # hint for set_pose_order (None: identity)
    priors: list                # dicts: pos (solver pose positions, listing order), G, g
    fill_WB: int                # tile offsets the priors fill
    med: float = 1.0            # median diagonal of S at lambda = 0 (the unit of Case.lambdas)

    def problem(self, extra=()):
        from dynosam_b200.problem import Problem
        n_pose = self.case.n_pose
        lp = [dict(idx=self.s2u[pr["pos"]].astype(np.int32), lin=np.tile(IDENTITY, (pr["pos"].size, 1)), G=pr["G"], g=pr["g"],
                   f=0.0) for pr in list(self.priors) + list(extra)]
        return Problem(np.tile(IDENTITY, (n_pose, 1)), np.zeros((0, 3)), pose_order=self.pose_order, linear_priors=lp)

    # banded assembly in the device's order: lambda on the diagonal, then the priors as they were added
    def band(self, lam, extra=()):
        ab = np.zeros((self.bw_store + 1, self.n))
        ab[0] = lam
        gS = np.zeros(self.n)
        for pr in list(self.priors) + list(extra):
            P = (6*pr["pos"][:, None] + np.arange(6)[None, :]).reshape(-1)
            I, J = np.meshgrid(P, P, indexing="ij")
            m = I >= J
            ab[I[m] - J[m], J[m]] += pr["G"][m]
            gS[P] += pr["g"]
        return ab, gS

    @property
    def bw_store(self):
        return min(6*(min(self.case.span, self.case.n_pose) - 1) + 5, self.n - 1)

    def user_perm(self):
        """solver scalar -> user scalar"""
        return (6*self.s2u[:, None] + np.arange(6)[None, :]).reshape(-1)

    def lam_abs(self, rel):
        return rel*self.med


def build(case: Case) -> System:
    rng = np.random.default_rng(case.seed)
    n_pose, n = case.n_pose, 6*case.n_pose
    assert min(case.span, n_pose) <= MAX_PRIOR_POSES
    s2u = rng.permutation(n_pose) if case.permute else np.arange(n_pose)
    order = np.argsort(s2u).astype(np.int32) if case.permute else None     # solver position of each user pose
    wins = _windows(n_pose, case.span)
    priors = []
    for w in wins:
        pos = rng.permutation(w)
        m = 6*pos.size
        if case.family == "nearsing":
            A = rng.standard_normal((m, max(1, int(0.4*m))))
            G = A @ A.T
            G = np.tril(G) + np.tril(G, -1).T
        elif case.family == "laplacian":
            # weighted graph Laplacian of the window's poses: sum over pose pairs (e_a - e_b)(e_a - e_b)^T (x) W_ab, W_ab SPD
            k = pos.size
            G = np.zeros((m, m))
            for a_ in range(k):
                for b_ in range(a_ + 1, k):
                    M = rng.standard_normal((6, 6))
                    W = M @ M.T/6
                    ia, ib = slice(6*a_, 6*a_ + 6), slice(6*b_, 6*b_ + 6)
                    G[ia, ia] += W; G[ib, ib] += W; G[ia, ib] -= W; G[ib, ia] -= W
            G = np.tril(G) + np.tril(G, -1).T
        else:
            A = rng.standard_normal((m, m))
            G = (A + A.T)*0.5
            np.fill_diagonal(G, 0.0)
        priors.append(dict(pos=pos, G=G, g=rng.standard_normal(m)))
    sysm = System(case, n, s2u, order, priors, 0)
    # diagonal: dominant / graded: t = 1.02 max off-diagonal row sum; nearsing: eps = 1e-10 of the largest row sum
    ab, _ = sysm.band(0.0)
    R = _abs_rowsum(ab) - np.abs(ab[0])
    t = 1.0205*R.max() if case.family not in ("nearsing", "laplacian") else 1e-10*(R + np.abs(ab[0])).max()
    first = np.full(n, True)
    for pr in priors:
        P = (6*pr["pos"][:, None] + np.arange(6)[None, :]).reshape(-1)
        d = np.diag(pr["G"]).copy()
        d[first[P]] += t
        first[P] = False
        np.fill_diagonal(pr["G"], d)
    if case.family == "graded":
        D = 10.0**rng.uniform(-6, 6, n_pose)
        for pr in priors:
            dp = np.repeat(D[pr["pos"]], 6)
            G = dp[:, None]*pr["G"]*dp[None, :]
            pr["G"] = np.tril(G) + np.tril(G, -1).T
            pr["g"] = dp*pr["g"]
    ab, _ = sysm.band(0.0)
    sysm.fill_WB = _fill_check(ab)
    sysm.med = float(np.median(ab[0]))
    return sysm


def _fill_check(ab):
    """every tile offset dd = 0..WB of the assembled band has entries in several tile columns -> WB"""
    n = ab.shape[1]
    NT = -(-n//TILE)
    WB = min(-(-(ab.shape[0] - 1)//TILE), NT - 1)
    cols = [set() for _ in range(WB + 1)]
    for d in range(ab.shape[0]):
        j = np.flatnonzero(ab[d, :n - d] != 0)
        dd = (j + d)//TILE - j//TILE
        for k in np.unique(dd):
            cols[k].update((j[dd == k]//TILE).tolist())
    for dd in range(WB + 1):
        assert len(cols[dd]) >= min(2, NT - dd), (dd, len(cols[dd]))
    return WB


def negative_prior(sysm: System, pose_pos: int):
    """single-pose prior -c I at solver position pose_pos, c = 2 lambda_max of that pose's 6x6 block of S (lambda = 0)"""
    ab, _ = sysm.band(0.0)
    p0 = 6*pose_pos
    B = np.zeros((6, 6))
    for d in range(6):
        for j in range(6 - d):
            B[j + d, j] = B[j, j + d] = ab[d, p0 + j]
    c = 2.0*np.linalg.eigvalsh(B).max()
    return dict(pos=np.array([pose_pos]), G=-c*np.eye(6), g=np.zeros(6)), c


# ------------------------------------------------------------------------------------------------------------ reference
def dense(ab):
    n = ab.shape[1]
    S = np.zeros((n, n))
    for d in range(ab.shape[0]):
        i = np.arange(n - d)
        S[i + d, i] = ab[d, :n - d]
        S[i, i + d] = ab[d, :n - d]
    return S


def solve(ab, g):
    """LAPACK band Cholesky (dpbtrf / dpbtrs)"""
    return sla.cho_solve_banded((sla.cholesky_banded(ab, lower=True), True), g)


def matvec(ab, x):
    n = x.size
    y = ab[0]*x
    for d in range(1, ab.shape[0]):
        v = ab[d, :n - d]
        y[d:] += v*x[:n - d]
        y[:n - d] += v*x[d:]
    return y


def _abs_rowsum(ab, s=None):
    """sum_j |S_ij| s_j (s = 1 by default)"""
    n = ab.shape[1]
    s = np.ones(n) if s is None else s
    y = np.abs(ab[0])*s
    for d in range(1, ab.shape[0]):
        v = np.abs(ab[d, :n - d])
        y[d:] += v*s[:n - d]
        y[:n - d] += v*s[d:]
    return y


def certified_kappa(ab):
    """Gershgorin bound on kappa(D^-1/2 S D^-1/2); inf when the discs do not exclude 0"""
    dg = ab[0]
    if (dg <= 0).any():
        return np.inf
    r = (_abs_rowsum(ab, 1/np.sqrt(dg)) - np.abs(dg)/np.sqrt(dg))/np.sqrt(dg)
    rm = r.max()
    return (1 + rm)/(1 - rm) if rm < 1 else np.inf


def forward_error(d, x, xref):
    """d = diag S"""
    s = np.sqrt(d)
    return float(np.abs(s*(x - xref)).max()/np.abs(s*xref).max())


def backward_error(ab, x, g):
    s = np.sqrt(ab[0])
    r = (matvec(ab, x) - g)/s
    norm = (_abs_rowsum(ab, 1/s)/s).max()
    return float(np.abs(r).max()/(norm*np.abs(s*x).max() + np.abs(g/s).max()))


SPIKE_BOUNDARIES = ("spiked Kend < 16", "spiked Kend 16", "spiked Kend 17", "spiked Kend 32", "spiked Kend 33",
                    "spiked, partial spike-forward chunk")


def dropped_chunk_errors(sysm, lam=0.0):
    """Backward errors of the solves a skipped last chunk of cell 1's spiked chain A would return: (the last FF_CH chunk of
    FF -= sum_J Z(J) Z(J)^T missing, i.e. S_QQ too large by its terms; the last SF_CH chunk of g_Q -= sum_J Z(J) y_J
    missing, i.e. g_Q too large by its terms; the exact solve), Z = S_QA L_AA^-T and y = L_AA^-1 g_A over the chain's
    factored columns.  Dense, equilibrated solves."""
    L = sysm.case.layout()
    c, K = L.cells[1], L.chains[2].Kend
    ab, g = sysm.band(lam)
    S = dense(ab)
    A, Q = np.arange(c.a0, c.m0), np.arange(c.q0, c.a0)
    LA = np.linalg.cholesky(S[np.ix_(A, A)])
    Z = sla.solve_triangular(LA, S[np.ix_(A, Q)], lower=True).T
    y = sla.solve_triangular(LA, g[A], lower=True)
    d = np.sqrt(ab[0])

    def solve_eq(M, b):
        return np.linalg.solve(M/d[:, None]/d[None, :], b/d)/d
    f0, s0 = TILE*FF_CH*((K - 1)//FF_CH), TILE*SF_CH*((K - 1)//SF_CH)
    Sf = S.copy()
    Sf[np.ix_(Q, Q)] += Z[:, f0:] @ Z[:, f0:].T
    gs = g.copy()
    gs[Q] += Z[:, s0:] @ y[s0:]
    return tuple(backward_error(ab, x, g) for x in (solve_eq(Sf, g), solve_eq(S, gs), solve_eq(S, g)))


def schur_marginal(S, g, p0):
    """marginal of the trailing block [p0, n): S_kk - S_kr S_rr^-1 S_rk, g_k - S_kr S_rr^-1 g_r"""
    if p0 == 0:
        return S.copy(), g.copy()
    Srr, Skr = S[:p0, :p0], S[p0:, :p0]
    X = np.linalg.solve(Srr, np.concatenate([Skr.T, g[:p0, None]], 1))
    return S[p0:, p0:] - Skr @ X[:, :-1], g[p0:] - Skr @ X[:, -1]


# ------------------------------------------------------------------------------------------------------------ cases
PLAIN = [
    Case("one_pose", "dominant", 1, 1, hits=("one tile (WB = 0)",)),
    Case("one_tile", "dominant", 5, 5, hits=("one tile (WB = 0)",)),
    Case("nt2_dense", "dominant", 6, 6, hits=("NT = 2", "dense band (WB = NT - 1)")),
    Case("nt2_wb1", "graded", 10, 3, hits=("NT = 2",)),
    Case("wb1", "dominant", _n_pose(40), _span(1)),
    Case("wb2", "dominant", 150, _span(2), hits=("WB = 2 (spine owns dd <= 2)",)),
    Case("wb3", "dominant", 101, _span(3)),
    Case("wb4_graded", "graded", 133, _span(4)),
    Case("wb7", "dominant", 177, _span(7)),
    Case("wb8", "dominant", 201, _span(8)),
    Case("wb9_permuted", "dominant", 255, _span(9), permute=True),
    Case("wb16", "dominant", 333, _span(16)),
    Case("wb17_graded", "graded", 350, _span(17)),
    Case("wb32_n32", "dominant", 416, _span(32)),                          # n % 32 == 0 on purpose
    Case("wb33", "dominant", 420, _span(33), hits=("WB > 32 (backward q loop)",)),
    Case("wb35", "graded", 530, _span(35), hits=("WB > 32 (backward q loop)",)),
    Case("dense", "dominant", 40, 40, hits=("dense band (WB = NT - 1)",)),
    Case("bw_clamp", "dominant", 30, 4, min_bandwidth=100000, hits=("min_bandwidth above n - 1", "dense band (WB = NT - 1)")),
    Case("nearsing_wb3", "nearsing", 120, _span(3), lambdas=(0.0,)),
    Case("nearsing_wb9", "nearsing", 211, _span(9), lambdas=(0.0,)),
]

CELLS = [
    Case("c1_wb1", "dominant", _n_pose(30), _span(1), cells=1, hits=("1 cell",)),
    Case("c_default", "dominant", _n_pose(50), _span(2), cells=0, hits=("1 cell",)),
    Case("c2_wb1_gq1", "dominant", _n_pose(40), _span(1), cells=2, hits=("one-tile boundary system", "cells with WB <= 3")),
    Case("c16_wb1", "dominant", _n_pose(113), _span(1), cells=16, hits=("16 cells", "cmax clamped to MAX_CELLS")),
    Case("c16_wb2", "graded", _n_pose(130), _span(2), cells=16, hits=("16 cells", "cells with WB <= 3")),
    Case("c3_wb2", "dominant", _n_pose(60), _span(2), cells=3, hits=("3 cells",)),
    Case("c3_wb2_clamped", "dominant", _n_pose(26), _span(2), cells=8, hits=("request above cmax", "3 cells")),
    Case("c4_wb3_minimal", "dominant", _n_pose(45), _span(3), cells=4, hits=("cmax with minimal chains", "4 cells")),
    Case("c4_wb3_graded_permuted", "graded", _n_pose(75), _span(3), cells=4, permute=True),
    Case("c8_wb7", "dominant", _n_pose(230), _span(7), cells=8, hits=("8 cells",)),
    Case("c8_wb8", "dominant", _n_pose(260), _span(8), cells=8, hits=("8 cells",)),
    Case("c2_wb9", "dominant", _n_pose(80), _span(9), cells=2, hits=("spiked, WB % SPK_ROWS != 0",)),
    Case("c4_wb17", "graded", _n_pose(270), _span(17), cells=4, hits=("spiked, WB % SPK_ROWS != 0",)),
    # spiked chains around the FF chunk (FF_CH columns): outer_weight 1 makes all four chains of two cells equally long
    # (in these two families the spike decays: the last chunk of a long chain is below rounding, see the laplacian cases)
    Case("c2_kend15", "dominant", _n_pose(4*15 + 9), _span(3), cells=2, outer_weight=1, hits=("outer_weight 1",)),
    Case("c2_kend16", "dominant", _n_pose(4*16 + 9), _span(3), cells=2, outer_weight=1),
    Case("c2_kend17", "dominant", _n_pose(4*17 + 9), _span(3), cells=2, outer_weight=1),
    Case("c2_kend32", "dominant", _n_pose(4*32 + 9), _span(3), cells=2, outer_weight=1),
    Case("c2_kend33", "graded", _n_pose(4*33 + 9), _span(3), cells=2, outer_weight=1),
    Case("c2_ow12", "dominant", _n_pose(60), _span(2), cells=2, outer_weight=12, hits=("outer_weight 12",)),
    Case("c2_default_weight", "dominant", _n_pose(60), _span(2), cells=2, hits=("outer_weight default",)),
    Case("nearsing_c2", "nearsing", _n_pose(80), _span(3), cells=2, lambdas=(0.0,)),
    # spiked chains around the FF chunk whose last FF chunk and last spike-forward chunk are visible in the backward
    # error (test_band_solve.py checks this on the CPU): only these claim the spike-chunk boundaries
    Case("laplacian_kend15", "laplacian", _n_pose(4*15 + 9), _span(3), cells=2, outer_weight=1, lambdas=(0.0,),
         hits=("spiked Kend < 16", "spiked, partial spike-forward chunk")),
    Case("laplacian_kend16", "laplacian", _n_pose(4*16 + 9), _span(3), cells=2, outer_weight=1, lambdas=(0.0,),
         hits=("spiked Kend 16",)),
    Case("laplacian_kend17", "laplacian", _n_pose(4*17 + 9), _span(3), cells=2, outer_weight=1, lambdas=(0.0,),
         hits=("spiked Kend 17", "spiked, partial spike-forward chunk")),
    Case("laplacian_kend32", "laplacian", _n_pose(4*32 + 9), _span(3), cells=2, outer_weight=1, lambdas=(0.0,),
         hits=("spiked Kend 32",)),
    Case("laplacian_kend33", "laplacian", _n_pose(4*33 + 9), _span(3), cells=2, outer_weight=1, lambdas=(0.0,),
         hits=("spiked Kend 33", "spiked, partial spike-forward chunk")),
]

CASES = {c.name: c for c in PLAIN + CELLS}

# the kept blocks of dynoba_marginal: (case, n_keep, expected).  n_pose 60 with WB = 2 has NT = 12; the kept block starts at
# p0 = 6 (n_pose - n_keep), in tile K0 = p0 // 32, and must satisfy NT - K0 <= WB + 1
MARGINAL_BASE = Case("marginal_wb2", "dominant", 60, _span(2), lambdas=(0.0,))
MARGINAL_DENSE = Case("marginal_dense", "graded", 20, 20, lambdas=(0.0,))     # WB = NT - 1 = 3: every variable may be kept
MARGINALS = [
    ("p0 % 32 == 0, NT - K0 = WB + 1", MARGINAL_BASE, 12),       # p0 = 288
    ("p0 % 32 == 30", MARGINAL_BASE, 7),                         # p0 = 318
    ("p0 % 32 == 2", MARGINAL_BASE, 1),                          # p0 = 354
    ("p0 % 32 == 12", MARGINAL_BASE, 10),                        # p0 = 300
    ("p0 % 32 == 16", MARGINAL_BASE, 4),                         # p0 = 336
    ("n_keep = n_pose (Kend = 0)", MARGINAL_DENSE, 20),
    ("p0 % 32 == 16, dense", MARGINAL_DENSE, 12),                # p0 = 48
]
