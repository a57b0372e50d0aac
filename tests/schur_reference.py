"""Dense fp64 reference of the landmark elimination, the routes the symbolic phase sends landmark groups down, and
seeded graphs that take every route and every boundary inside one.

Reference.  Given a problem, the damping lambda and a function returning each factor block's whitened Jacobians and
rhs (the device's own, ``Solver.linearization``, so the elimination is tested apart from linearization rounding):

    J  stacked whitened Jacobians, columns [poses 6 | points 3 | flows 2] in user order (problem.SLOT_CLASS / CLASS_DIM)
    H  = J^T J,   g = J^T b
    S  = H_pp + lambda I - H_pl (H_ll + lambda I)^-1 H_lp,     g_S = g_p - H_pl (H_ll + lambda I)^-1 g_l
    dl = (H_ll + lambda I)^-1 (g_l - H_lp dp)                  (landmark and flow back-substitution for a given dp)

H_ll is block diagonal over the landmark groups, so its inverse is formed group by group in dense fp64.

Comparator.  Entries are compared in the units of the undamped-plus-lambda normal equations, so that a 1e-6-sigma
prior (H_aa ~ 1e12) loosens only its own rows:

    S:    |S_ab - S_ref,ab| / sqrt(H_aa H_bb)                    H_aa = diag(J^T J)_a + lambda, before elimination
    g_S:  |g_a - g_ref,a| / (sqrt(H_aa) r)                       r = max |b|, the largest whitened residual
    dl:   |dl_j - dl_ref,j| sqrt(H_jj) / (r + max |J_p dp|)      H_jj over the landmark columns

By Cauchy-Schwarz every term summed into S_ab is at most sqrt(H_aa H_bb) (and into g_a at most sqrt(H_aa) r), so
fp64 reassociation stays near 1e-16 times the number of terms in these units.

Route mirror.  ``routes(p)`` restates the symbolic phase (``finalize`` in csrc/api.cu, which leaves the window / simple
split to ``plan_windows`` in csrc/window_plan.cuh): union-find over factors that touch two landmarks, then per factor
block and group
    window   3-dof landmark type, the group's only block, one landmark, T <= WIN_TMAX, no pose repeated in the group
    simple   one landmark in one block otherwise (T > WIN_TMAX, a repeated pose, the flow type)
    general  several landmarks (chains), or a landmark with factors in several blocks; refused above GG_MAXL points
             or when a flow variable is in such a group
The constants are read from the CUDA sources, so the boundary cases below move with them.
"""
from __future__ import annotations

import dataclasses
import os
import re

import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from dynosam_b200 import lie, synth
from dynosam_b200.problem import (CLASS_DIM, DIM, FLOWPROJ2, HYBRID3, HYBRID_STEREO3, POSE2POINT3, PRIOR6, SLOT_CLASS,
                                  STEREO3, FactorBlock, Problem)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")


def _const(fname, pattern, n=1):
    with open(os.path.join(CSRC, fname)) as f:
        m = re.search(pattern, f.read())
    if m is None:
        raise RuntimeError(f"{fname}: no match for {pattern!r}; the route mirror must be updated with the source")
    v = tuple(int(x) for x in m.groups())
    return v[0] if n == 1 else v


WIN_TMAX = _const("internal.cuh", r"constexpr int WIN_TMAX = (\d+);")
WIN_NLOC_MAX = _const("internal.cuh", r"constexpr int WIN_NLOC_MAX = (\d+);")
WIN_BATCH_SLOTS = _const("internal.cuh", r"constexpr int WIN_BATCH_SLOTS = (\d+);")
WIN_BATCH_LMK = _const("internal.cuh", r"constexpr int WIN_BATCH_LMK = (\d+);")
WIN_ACC_WARPS = _const("internal.cuh", r"constexpr int WIN_ACC_WARPS = (\d+);")
GG_MAXL = _const("kernels_chain.cu", r"constexpr int GG_MAXL = (\d+);")
CHUNK_CAP = _const("api.cu", r"int cap = NPs == 1 \? (\d+) : (\d+);", 2)          # (static NP = 1, dynamic NP = 2)
GEN_REFUSE_ABOVE = _const("api.cu", r"if \(gcount\[r\] > (\d+) \|\| r >= npt\) h->supported = false;")
STAGE_HALF_T = _const("kernels_window.cu", r"two && T0 <= (\d+) && T1 <= \d+")   # two landmarks per warp at or below
SIMPLE_STAGED_T = _const("kernels_schur.cu", r"const bool staged = T <= (\d+);")
HOST_SEGMENT_GROUPS = _const("api.cu", r"ng/(\d+) \+ 1\)")                       # window chunking: one host segment per this many groups

WINDOW_TYPES = (POSE2POINT3, STEREO3, HYBRID3, HYBRID_STEREO3)


def win_ntiles(nloc):
    """internal.cuh win_ntiles: 8x4 tiles of the lower triangle of an nloc x nloc window"""
    n, tr = 0, 0
    while tr*8 < nloc:
        n += min(8*tr + 7, nloc - 1)//4 + 1
        tr += 1
    return n


# ------------------------------------------------------------------------------------------------------------ reference
class Reference:
    def __init__(self, p: Problem, jac, lam: float):
        npz, npt, nfl = 6*p.n_pose, 3*p.n_point, 2*p.n_flow
        off = [0, npz, npz + npt]
        n = npz + npt + nfl
        rows, cols, vals, rhs = [], [], [], []
        r0 = 0
        for bi, b in enumerate(p.blocks):
            A, bv = jac(bi)
            d = DIM[b.type]
            c0 = 0
            r = r0 + np.arange(b.n)[:, None]*d + np.arange(d)[None, :]          # [n, d]
            for k, cls in enumerate(SLOT_CLASS[b.type]):
                w = CLASS_DIM[cls]
                var = off[cls] + w*b.idx[:, k].astype(np.int64)
                for c in range(w):
                    rows.append(r.reshape(-1)); cols.append(np.repeat(var + c, d)); vals.append(A[:, :, c0 + c].reshape(-1))
                c0 += w
            rhs.append(bv.reshape(-1))
            r0 += b.n*d
        J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(r0, n))
        bb = np.concatenate(rhs) if rhs else np.zeros(0)
        H = (J.T @ J).tocsr()
        g = J.T @ bb
        self.H, self.g = H, g
        self.npz, self.lam = npz, lam
        self.Jp = J[:, :npz]
        self.Hdiag = H.diagonal() + lam
        self.r = max(np.abs(bb).max(initial=0.0), 1e-300)
        Hpp = H[:npz, :npz]
        self.Hpl = H[:npz, npz:].tocsr()
        self.Hll_inv = _block_inverse(H[npz:, npz:] + lam*sp.identity(n - npz, format="csr"))
        X = self.Hll_inv @ self.Hpl.T                          # (H_ll + lambda I)^-1 H_lp, sparse
        self.S = Hpp.toarray() + lam*np.eye(npz) - (self.Hpl @ X).toarray()
        self.g_l = g[npz:]
        self.gS = g[:npz] - self.Hpl @ (self.Hll_inv @ self.g_l)

    def back_substitute(self, dp):
        return self.Hll_inv @ (self.g_l - self.Hpl.T @ dp)

    def pose_step(self):
        d = np.sqrt(np.diag(self.S))          # equilibrated: rows of a 1e-6-sigma prior keep their digits
        return np.linalg.solve(self.S/d[:, None]/d[None, :], self.gS/d)/d

    def kappa_s(self):
        """condition number of D^-1/2 S D^-1/2, D = diag S: what the pose step's forward error scales with"""
        d = np.sqrt(np.diag(self.S))
        ev = np.linalg.eigvalsh(self.S/d[:, None]/d[None, :])
        return float(ev.max()/ev.min())

    # comparator (module docstring)
    def s_err(self, S):
        d = np.sqrt(self.Hdiag[:self.npz])
        return float((np.abs(S - self.S)/d[:, None]/d[None, :]).max())

    def g_err(self, g):
        return float((np.abs(g - self.gS)/(np.sqrt(self.Hdiag[:self.npz])*self.r)).max())

    def l_err(self, dl, dp):
        if dl.size == 0:
            return 0.0
        scale = self.r + np.abs(self.Jp @ dp).max(initial=0.0)
        return float((np.abs(dl - self.back_substitute(dp))*np.sqrt(self.Hdiag[self.npz:])/scale).max())


def _block_inverse(M):
    """inverse of a block-diagonal SPD sparse matrix, one dense fp64 inverse per connected block"""
    n = M.shape[0]
    if n == 0:
        return sp.csr_matrix((0, 0))
    ncomp, lab = connected_components(M, directed=False)
    order = np.argsort(lab, kind="stable")
    cnt = np.bincount(lab, minlength=ncomp)
    start = np.concatenate([[0], np.cumsum(cnt)])
    loc = np.empty(n, np.int64); loc[order] = np.arange(n) - start[lab[order]]     # position inside its block
    C = M.tocoo()
    rows, cols, vals = [], [], []
    for size in np.unique(cnt):
        comps = np.flatnonzero(cnt == size)
        slot = np.full(ncomp, -1); slot[comps] = np.arange(comps.size)
        dense = np.zeros((comps.size, size, size))
        k = slot[lab[C.row]] >= 0
        dense[slot[lab[C.row[k]]], loc[C.row[k]], loc[C.col[k]]] = C.data[k]
        inv = np.linalg.inv(dense)
        idx = order[start[comps][:, None] + np.arange(size)[None, :]]      # [k, size] variables of each block
        rows.append(np.repeat(idx, size, axis=1).reshape(-1)); cols.append(np.tile(idx, (1, size)).reshape(-1))
        vals.append(inv.reshape(-1))
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def oracle_in_user_order(o, lam):
    """OracleProblem.reduced_dense permuted from solver order to user pose order"""
    S, g, pos = o.reduced_dense(lam)
    perm = (6*pos.astype(np.int64)[:, None] + np.arange(6)[None, :]).reshape(-1)
    return S[np.ix_(perm, perm)], g[perm]


# ------------------------------------------------------------------------------------------------------------ route mirror
@dataclasses.dataclass
class Group:
    block: int                 # factor block (general groups: one entry per block they touch)
    ftype: int
    route: str                 # window | simple | general | unsupported
    T: int                     # factors of the group in this block
    nloc: int                  # distinct pose-like variables of the group in this block
    points: int                # landmarks in the group (chain length)
    repeated: bool             # a pose-like variable repeated among the group's factors in this block
    flow: bool
    root: int                  # union-find root: the landmark's own index for one-landmark groups (flows after points)


def landmark_roots(p: Problem):
    """union-find root of every landmark (points, then flows) over the factors that touch two landmarks"""
    npt, nfl = p.n_point, p.n_flow
    nl = npt + nfl
    uf = np.arange(nl)

    def find(x):
        while uf[x] != x:
            uf[x] = uf[uf[x]]
            x = uf[x]
        return x

    def lmk(cls, ix):
        return ix if cls == 1 else npt + ix

    for b in p.blocks:
        lcols = [k for k, c in enumerate(SLOT_CLASS[b.type]) if c != 0]
        if len(lcols) < 2:
            continue
        for row in b.idx:
            a = find(lmk(SLOT_CLASS[b.type][lcols[0]], row[lcols[0]]))
            for k in lcols[1:]:
                c = find(lmk(SLOT_CLASS[b.type][k], row[k]))
                if a != c:
                    uf[c] = a
    return np.array([find(i) for i in range(nl)], dtype=np.int64)


def routes(p: Problem):
    """every (block, landmark group) of p with the route the symbolic phase gives it"""
    npt, nl = p.n_point, p.n_point + p.n_flow
    root = landmark_roots(p)
    gcount = np.bincount(root, minlength=nl)
    blocks_of = {}
    per_block = []
    for bi, b in enumerate(p.blocks):
        sc = SLOT_CLASS[b.type]
        lcols = [k for k, c in enumerate(sc) if c != 0]
        if not lcols:
            per_block.append(None)
            continue
        k0 = lcols[0]
        g = root[b.idx[:, k0] + (0 if sc[k0] == 1 else npt)]
        per_block.append(g)
        for r in np.unique(g):
            blocks_of.setdefault(int(r), set()).add(bi)
    out = []
    for bi, b in enumerate(p.blocks):
        g = per_block[bi]
        if g is None:
            continue
        sc = SLOT_CLASS[b.type]
        pcols = [k for k, c in enumerate(sc) if c == 0]
        nlmk = sum(1 for c in sc if c != 0)
        order = np.argsort(g, kind="stable")
        gs = g[order]
        starts = np.flatnonzero(np.r_[True, gs[1:] != gs[:-1]])
        for s0, s1 in zip(starts, np.r_[starts[1:], gs.size]):
            r = int(gs[s0]); f = order[s0:s1]
            poses = b.idx[f][:, pcols].reshape(-1)
            T, nloc = int(f.size), int(np.unique(poses).size)
            rep = nloc < poses.size
            flow = r >= npt
            one = nlmk == 1 and len(blocks_of[r]) == 1 and gcount[r] == 1
            if not one:
                route = "unsupported" if (gcount[r] > GEN_REFUSE_ABOVE or flow) else "general"
            elif b.type in WINDOW_TYPES and T <= WIN_TMAX and not rep:
                route = "window"
            else:
                route = "simple"
            out.append(Group(bi, b.type, route, T, nloc, int(gcount[r]), bool(rep), bool(flow), r))
    return out


def chunk_stats(p: Problem, bi: int):
    """the window chunks of block bi as one host segment builds them: [(nloc, landmarks, slots)].  Single-block groups
    are ordered by their smallest last-slot pose index (two pose slots) or first pose position (one), then by id."""
    b = p.blocks[bi]
    sc = SLOT_CLASS[b.type]
    pcols = [k for k, c in enumerate(sc) if c == 0]
    lcol = [k for k, c in enumerate(sc) if c != 0][0]
    NP = len(pcols)
    cap = CHUNK_CAP[0] if NP == 1 else CHUNK_CAP[1]
    pos = np.empty(p.n_pose, np.int64)
    pos[np.argsort(p.pose_order if p.pose_order is not None else np.arange(p.n_pose), kind="stable")] = np.arange(p.n_pose)
    win = {g.root for g in routes(p) if g.block == bi and g.route == "window"}
    fac = {}
    for i, l in enumerate(b.idx[:, lcol]):
        fac.setdefault(int(l), []).append(i)
    keys = []
    for l in win:
        pp = b.idx[fac[l]][:, pcols]
        keys.append((int(pp[:, -1].min()) if NP >= 2 else int(pos[pp[:, 0]].min()), l))
    chunks, cur, lm, slots = [], set(), 0, 0
    for _, l in sorted(keys):
        vs = set(b.idx[fac[l]][:, pcols].reshape(-1).tolist())
        if cur and len(cur) + len(vs - cur) > cap:
            chunks.append((len(cur), lm, slots)); cur, lm, slots = set(), 0, 0
        cur |= vs; lm += 1; slots += NP*len(fac[l])
    if cur:
        chunks.append((len(cur), lm, slots))
    return chunks


# ------------------------------------------------------------------------------------------------------------ route graphs
def _weak_priors(p: Problem, sigma=0.05):
    """the same graph with every PRIOR6 at sigma: no row of S dominated by a 1e-6-sigma prior"""
    blocks = [FactorBlock(b.type, b.idx, b.meas, np.full(6, sigma), b.robust_k, b.aux_idx) if b.type == PRIOR6 else b
              for b in p.blocks]
    return dataclasses.replace(p, blocks=blocks)


def _append(b: FactorBlock, idx, meas, aux=None):
    return FactorBlock(b.type, np.concatenate([b.idx, idx]), np.concatenate([b.meas, meas]), b.sigma, b.robust_k,
                       None if b.aux_idx is None else np.concatenate([b.aux_idx, aux]))


def _static_tracks(rng, X, n0, lengths, N, depth=(4.0, 40.0), noise=0.1, repeat=()):
    """explicit static tracks: track i has lengths[i] observations on consecutive frames; tracks listed in `repeat` see
    one of their frames twice (a duplicated factor with a perturbed measurement).  -> (idx [pose, point], z, p_init)"""
    L = np.asarray(lengths, dtype=np.int64)
    birth = rng.integers(0, N - L + 1)
    d = rng.uniform(*depth, L.size)
    pc = np.stack([rng.uniform(-0.4, 0.4, L.size)*d, rng.uniform(-0.15, 0.15, L.size)*d, d], 1)
    pw = lie.transform_from(X[birth], pc)
    fr, pid = [], []
    for i, (b0, l) in enumerate(zip(birth, L)):
        f = b0 + np.arange(l)
        if i in repeat:
            f = np.sort(np.r_[f, f[rng.integers(0, l)]])
        fr.append(f); pid.append(np.full(f.size, n0 + i))
    fr, pid = np.concatenate(fr), np.concatenate(pid)
    z = lie.transform_to(X[fr], pw[pid - n0]) + rng.normal(0, noise, (fr.size, 3))
    return np.stack([fr, pid], 1), z, pw + rng.normal(0, 0.05, pw.shape)


def window_np1_graph(seed=1):
    """Static landmarks on the window path (NP = 1), POSE2POINT3 and STEREO3: T = 1, 2, 15, 16, 17 and WIN_TMAX, hundreds
    of each in random order (half-warp and full-warp staging pairs), an odd group count, chunks holding more than
    WIN_BATCH_LMK landmarks and WIN_BATCH_SLOTS slots, and more than 3 host segments' worth of groups in one block.
    440 frames: long enough for four cells of the reduced solve."""
    rng = np.random.default_rng(seed)
    N = 440
    base = synth.make_problem(n_frames=N, n_objects=0, n_static=0, n_dynamic=0, seed=seed)
    X = base.meta["gt_camera"]
    cases = [1, 2, STAGE_HALF_T - 1, STAGE_HALF_T, STAGE_HALF_T + 1, WIN_TMAX]
    fill = 3*HOST_SEGMENT_GROUPS + 1 - 200*len(cases)
    lengths = rng.permutation(np.r_[np.repeat(cases, 200), rng.integers(1, 4, fill)])
    if lengths.size % 2 == 0:
        lengths = np.r_[lengths, 5]
    idx, z, pinit = _static_tracks(rng, X, 0, lengths, N)
    blocks = [FactorBlock(POSE2POINT3, idx, z, np.array([0.2]), 1e-4)]
    # stereo: points that stay in front of the camera over a WIN_TMAX-frame track at 1 m per frame, a block of their own
    sl = rng.permutation(np.repeat(cases, 40))
    sidx, _, spinit = _static_tracks(rng, X, lengths.size, sl, N, depth=(WIN_TMAX + 2.0, WIN_TMAX + 12.0))
    K = base.calib
    q = lie.transform_to(X[sidx[:, 0]], np.concatenate([pinit, spinit])[sidx[:, 1]])
    zs = np.stack([K[3] + K[0]*q[:, 0]/q[:, 2], K[3] + K[0]*(q[:, 0] - K[5])/q[:, 2], K[4] + K[1]*q[:, 1]/q[:, 2]], 1)
    blocks.append(FactorBlock(STEREO3, sidx, zs + rng.normal(0, 0.5, zs.shape), np.array([1.0, 1.0, 1.5]), 1.345))
    return _weak_priors(dataclasses.replace(base, point=np.concatenate([pinit, spinit]), blocks=blocks + base.blocks,
                                            point_keys=None))


def _hybrid_tracks(rng, p, obj, lengths, n0, repeat=()):
    """explicit HYBRID3 tracks on object `obj` of a hybrid make_problem graph (one motion variable per frame of the
    object): consecutive frames inside the object's span, optionally one frame seen twice"""
    hyb = next(b for b in p.blocks if b.type == HYBRID3)
    sel = hyb.aux_idx == obj
    f2h = dict(zip(hyb.idx[sel, 0].tolist(), hyb.idx[sel, 1].tolist()))
    frames = np.array(sorted(f2h))
    X = p.meta["gt_camera"]; Hgt = p.meta["gt_motion"]; N = p.meta["n_frames"]; Le = p.aux_pose[obj]
    rows, zs, m0 = [], [], []
    for i, l in enumerate(lengths):
        s0 = frames[rng.integers(0, frames.size - l + 1)]
        f = s0 + np.arange(l)
        if i in repeat:
            f = np.sort(np.r_[f, f[rng.integers(0, l)]])
        h = np.array([f2h[x] for x in f])
        m = rng.uniform(-1, 1, 3)*np.array([2.0, 1.0, 1.0])
        w = lie.transform_from(Hgt[h - N], np.tile(lie.transform_from(Le[None], m[None])[0], (f.size, 1)))
        zs.append(lie.transform_to(X[f], w) + rng.normal(0, 0.1, (f.size, 3)))
        rows.append(np.stack([f, h, np.full(f.size, n0 + i)], 1)); m0.append(m + rng.normal(0, 0.05, 3))
    return np.concatenate(rows), np.concatenate(zs), np.array(m0)


def window_np2_graph(seed=2):
    """Hybrid landmarks (NP = 2) with T up to WIN_TMAX: T = 21..24 have NLOC = 2T > 40, a chunk of their own with three
    stripes of the accumulate kernel, next to T <= 20 landmarks that share chunks."""
    p = synth.make_problem(n_frames=120, n_objects=2, n_static=1500, n_dynamic=700, formulation="hybrid", seed=seed,
                           object_span=(110, 120), max_dynamic_age=WIN_TMAX)
    return _weak_priors(p)


def simple_graph(seed=3):
    """The simple kernel: static (NP = 1) and hybrid (NP = 2) landmarks with T = WIN_TMAX + 1, SIMPLE_STAGED_T,
    SIMPLE_STAGED_T + 1, 64, 65 (staged and unstaged), landmarks that see one pose twice with T <= WIN_TMAX and with
    T > SIMPLE_STAGED_T (the M + M^T branch), all in the same blocks as window landmarks; plus a flow star."""
    rng = np.random.default_rng(seed)
    p = synth.make_problem(n_frames=150, n_objects=1, n_static=800, n_dynamic=250, formulation="hybrid", seed=seed,
                           object_span=(150, 150))
    X = p.meta["gt_camera"]; N = p.meta["n_frames"]
    cases = [WIN_TMAX + 1, SIMPLE_STAGED_T, SIMPLE_STAGED_T + 1, 64, 65]
    ls = np.r_[np.repeat(cases, 4), [10, 10, 40, 40]]
    rep = set(range(ls.size - 4, ls.size))
    idx, z, pi = _static_tracks(rng, X, p.n_point, ls, N, repeat=rep)
    blocks = list(p.blocks)
    bi = next(i for i, b in enumerate(blocks) if b.type == POSE2POINT3)
    blocks[bi] = _append(blocks[bi], idx, z)
    hidx, hz, hm = _hybrid_tracks(rng, p, 0, ls, p.n_point + ls.size, repeat=rep)
    hi = next(i for i, b in enumerate(blocks) if b.type == HYBRID3)
    blocks[hi] = _append(blocks[hi], hidx, hz, np.zeros(hidx.shape[0], np.int32))
    # flow star on camera 3 (Pose3FlowProjectionFactor: one flow variable per factor)
    nf = 40
    kp = np.stack([rng.uniform(100, 1100, nf), rng.uniform(50, 320, nf)], 1); depth = rng.uniform(4, 30, nf)
    meas = np.concatenate([kp, depth[:, None], np.tile(p.pose[2], (nf, 1))], 1)
    blocks.append(FactorBlock(FLOWPROJ2, np.stack([np.arange(nf), np.full(nf, 3)], 1), meas, np.array([0.5]), 0.0))
    return _weak_priors(dataclasses.replace(p, point=np.concatenate([p.point, pi, hm]), flow=rng.normal(0, 1.0, (nf, 2)),
                                            blocks=blocks, point_keys=None, pose_keys=None))


def general_wcme_graph(seed=4):
    """WCME chains of every length up to GG_MAXL points (10, 11, 12 cross the 32 warp lanes at n = 3*points; GG_MAXL is
    n = 63, with 2*GG_MAXL - 1 > 32 factors), and static points seen by POSE2POINT3 and STEREO3 from the same frame
    (a general group whose two blocks hit one pose: the M + M^T branch)."""
    rng = np.random.default_rng(seed)
    p = synth.make_problem(n_frames=60, n_objects=2, n_static=600, n_dynamic=400, formulation="wcme", seed=seed,
                           object_span=(60, 60), max_dynamic_age=GG_MAXL)
    ptp = p.blocks[0]
    first = np.flatnonzero(np.r_[True, ptp.idx[1:, 1] != ptp.idx[:-1, 1]])[:150]
    cam, pid = ptp.idx[first, 0], ptp.idx[first, 1]
    K = p.calib
    q = lie.transform_to(p.pose[cam], p.point[pid])
    q[:, 2] = np.abs(q[:, 2]) + 1.0
    zs = np.stack([K[3] + K[0]*q[:, 0]/q[:, 2], K[3] + K[0]*(q[:, 0] - K[5])/q[:, 2], K[4] + K[1]*q[:, 1]/q[:, 2]], 1)
    st = FactorBlock(STEREO3, np.stack([cam, pid], 1), zs + rng.normal(0, 1.0, zs.shape), np.array([1.5, 1.5, 2.0]), 1.345)
    return _weak_priors(dataclasses.replace(p, blocks=list(p.blocks) + [st]))


def general_wcpe_graph(seed=5):
    """WCPE chains (four-key LandmarkMotionPoseFactor) up to GG_MAXL points."""
    p = synth.make_problem(n_frames=40, n_objects=1, n_static=300, n_dynamic=200, formulation="wcpe", seed=seed,
                           object_span=(40, 40), max_dynamic_age=GG_MAXL)
    return _weak_priors(p)


def refused_chain_graph(seed=2):
    """a WCME chain of GG_MAXL + 1 points: one point past the general-group kernel"""
    return synth.make_problem(n_frames=40, n_objects=1, n_static=50, n_dynamic=40, formulation="wcme", seed=seed,
                              max_dynamic_age=GG_MAXL + 1, object_span=(40, 40))


ROUTE_GRAPHS = {
    "window_np1": window_np1_graph,
    "window_np2": window_np2_graph,
    "simple": simple_graph,
    "general_wcme": general_wcme_graph,
    "general_wcpe": general_wcpe_graph,
    "all_types": synth.make_all_types_problem,
}


def permuted(p, seed, landmark_runs):
    """The same graph with its factors listed in another order: whole landmark runs shuffled (the order DynOSAM's
    formulations produce up to the order of the landmarks -- the run-based sort of the symbolic phase) or every factor
    shuffled individually (the general stable sort)."""
    rng = np.random.default_rng(seed)
    blocks = []
    for b in p.blocks:
        n = b.idx.shape[0]
        if landmark_runs and b.type in (POSE2POINT3, HYBRID3):
            lm = b.idx[:, -1]
            starts = np.flatnonzero(np.r_[True, lm[1:] != lm[:-1]])
            runs = np.split(np.arange(n), starts[1:])
            perm = np.concatenate([runs[i] for i in rng.permutation(len(runs))])
        else:
            perm = rng.permutation(n)
        sig = b.sigma if b.sigma.ndim == 1 else b.sigma[perm]
        blocks.append(FactorBlock(b.type, b.idx[perm], None if b.meas is None else b.meas[perm], sig, b.robust_k,
                                  aux_idx=None if b.aux_idx is None else b.aux_idx[perm]))
    return dataclasses.replace(p, blocks=blocks)
