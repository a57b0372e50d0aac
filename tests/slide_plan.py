"""Mirror of the window plan (``plan_windows`` in csrc/window_plan.cuh) and graphs that reach its boundaries.

For one factor block, ``plan(p, bi)`` restates what the host builds for the accumulate kernel when the block's groups
form one host segment (fewer than schur_reference.HOST_SEGMENT_GROUPS groups); ``plan(p, bi, nseg)`` cuts the group list
into nseg segments as the host does with nseg threads (chunks, slots and runs restart in each):
    chunks   greedy, in the symbolic phase's landmark order, at most CHUNK_CAP variables (schur_reference.chunk_stats)
    slots    NP = 2: a variable keeps its window slot over consecutive chunks that contain it, an entering variable takes
             the lowest free slot; NP = 1: slots in ascending solver position, chunk by chunk
    runs     NP = 2: max(WIN_RUN_MIN_CHUNKS, ceil(chunks / WIN_RUNS)) consecutive chunks; NP = 1: one chunk each
    census   accumulate CTAs (one per run and stripe of its window's 8x4 tiles) and the 6x6 blocks flushed: a slot pair
             some landmark's clique touched, when either slot changes variable and at the run's end
"""
from __future__ import annotations

import dataclasses

import numpy as np

import schur_reference as SR
from dynosam_b200 import synth
from dynosam_b200.problem import HYBRID3, SLOT_CLASS, FactorBlock

WIN_RUNS = SR._const("internal.cuh", r"constexpr int WIN_RUNS = (\d+);")
WIN_RUN_MIN_CHUNKS = SR._const("internal.cuh", r"constexpr int WIN_RUN_MIN_CHUNKS = (\d+);")


@dataclasses.dataclass
class Plan:
    np_: int
    chunks: list          # [set of solver positions]
    cliques: list         # per chunk: [list of solver positions of each landmark]
    slots: list           # per chunk: [WIN_NLOC_MAX] solver position in each slot, -1 empty
    runs: list            # [(first chunk, end chunk)]
    ctas: int
    flushed: int

    def transitions(self):
        """(run, chunk) of every chunk that follows another in its run, with the slots that change variable there"""
        out = []
        for r, (c0, c1) in enumerate(self.runs):
            for c in range(c0 + 1, c1):
                out.append((r, c, [s for s in range(SR.WIN_NLOC_MAX) if self.slots[c - 1][s] != self.slots[c][s]]))
        return out

    def reused_slots(self):
        """slots that, inside a run, pass from one variable straight to another"""
        return sum(1 for _, c, ch in self.transitions() for s in ch if self.slots[c - 1][s] >= 0 and self.slots[c][s] >= 0)


def positions(p):
    """solver position of every pose (the stable order of the pose hint)"""
    pos = np.empty(p.n_pose, np.int64)
    pos[np.argsort(p.pose_order if p.pose_order is not None else np.arange(p.n_pose), kind="stable")] = np.arange(p.n_pose)
    return pos


def block_groups(p, bi):
    """the landmark groups of block bi in the symbolic phase's order, [(route, root, factors)]: by the smallest
    last-slot pose index (two pose slots) or first pose position (one), then by root, the general groups last; a
    group's factors by the position of the first pose slot"""
    b = p.blocks[bi]
    sc = SLOT_CLASS[b.type]
    pcols = [k for k, c in enumerate(sc) if c == 0]
    lcol = [k for k, c in enumerate(sc) if c != 0][0]
    pos = positions(p)
    route = {g.root: g.route for g in SR.routes(p) if g.block == bi}
    g = SR.landmark_roots(p)[b.idx[:, lcol] + (0 if sc[lcol] == 1 else p.n_point)]
    order = np.lexsort((pos[b.idx[:, pcols[0]]], g))
    starts = np.flatnonzero(np.r_[True, g[order][1:] != g[order][:-1]])
    out = []
    for f in np.split(order, starts[1:]):
        r = int(g[f[0]]); pp = b.idx[f][:, pcols]
        key = int(pp[:, -1].min()) if len(pcols) >= 2 else int(pos[pp[:, 0]].min())
        out.append(((route[r] in ("general", "unsupported"), key, r), route[r], r, f))
    return [x[1:] for x in sorted(out, key=lambda x: x[0])]


def plan(p, bi, nseg=None) -> Plan:
    b = p.blocks[bi]
    pcols = [k for k, c in enumerate(SLOT_CLASS[b.type]) if c == 0]
    NP = len(pcols)
    cap = SR.CHUNK_CAP[0] if NP == 1 else SR.CHUNK_CAP[1]
    pos = positions(p)
    groups = block_groups(p, bi)
    if nseg is None:
        assert len(groups) < SR.HOST_SEGMENT_GROUPS, "the mirror covers one host segment"
        nseg = 1
    ng = len(groups)
    chunks, cliques, seg = [], [], []
    for t in range(nseg):
        cur, cl = set(), []
        for route, _, f in groups[ng*t//nseg:ng*(t + 1)//nseg]:
            if route != "window":
                continue
            vs = set(pos[b.idx[f][:, pcols].reshape(-1)].tolist())
            if cur and len(cur) + len(vs - cur) > cap:
                chunks.append(cur); cliques.append(cl); seg.append(t); cur, cl = set(), []
            cur |= vs; cl.append(sorted(vs))
        if cur:
            chunks.append(cur); cliques.append(cl); seg.append(t)
    slots = []
    for c, ch in enumerate(chunks):
        if NP == 1:
            row = sorted(ch) + [-1]*(SR.WIN_NLOC_MAX - len(ch))
        else:
            if c == 0 or seg[c] != seg[c - 1]:
                occ, where = [-1]*SR.WIN_NLOC_MAX, {}
            occ = [v if v in ch else -1 for v in occ]
            for v in sorted(ch):
                if where.get(v, -1) >= 0 and occ[where[v]] == v:
                    continue
                s = occ.index(-1)
                occ[s] = v; where[v] = s
            row = list(occ)
        slots.append(row)
    L = max(WIN_RUN_MIN_CHUNKS, -(-len(chunks)//WIN_RUNS)) if NP == 2 else 1
    runs = []
    for t in sorted(set(seg)):
        c0, c1 = seg.index(t), len(seg) - seg[::-1].index(t)
        runs += [(c, min(c + L, c1)) for c in range(c0, c1, L)]
    ctas = flushed = 0
    for c0, c1 in runs:
        ext = max(max([s + 1 for s in range(SR.WIN_NLOC_MAX) if slots[c][s] >= 0], default=0) for c in range(c0, c1))
        ctas += -(-SR.win_ntiles(ext)//SR.WIN_ACC_WARPS)
        touched = set()
        for c in range(c0, c1 + 1):
            change = set(range(SR.WIN_NLOC_MAX)) if c == c1 else \
                {s for s in range(SR.WIN_NLOC_MAX) if c > c0 and slots[c - 1][s] != slots[c][s]}
            gone = {t for t in touched if t[0] in change or t[1] in change}
            flushed += len(gone); touched -= gone
            if c == c1:
                break
            slot_of = {v: s for s, v in enumerate(slots[c]) if v >= 0}
            for vs in cliques[c]:
                ss = [slot_of[v] for v in vs]
                touched |= {(max(x, y), min(x, y)) for x in ss for y in ss}
    return Plan(NP, chunks, cliques, slots, runs, ctas, flushed)


def hybrid_block(p):
    return next(i for i, b in enumerate(p.blocks) if b.type == HYBRID3)


# ------------------------------------------------------------------------------------------------------------ graphs
def long_object_graph(seed=11):
    """One object over 360 frames, ~9 tracklets born per frame: hundreds of consecutive chunks of one object, so window
    slots are reused over and over inside a run, and the chunks make many runs."""
    return SR._weak_priors(synth.make_problem(n_frames=360, n_objects=1, n_static=600, n_dynamic=3300, formulation="hybrid",
                                              seed=seed, object_span=(360, 360)))


def cap_graph(seed=12):
    """Tracklets living up to WIN_TMAX frames: NLOC 42..48 chunks (a landmark of their own, three stripes) inside runs
    with the shared chunks up to the cap."""
    return SR._weak_priors(synth.make_problem(n_frames=150, n_objects=1, n_static=400, n_dynamic=1500, formulation="hybrid",
                                              seed=seed, object_span=(150, 150), max_dynamic_age=SR.WIN_TMAX))


def drop_points(p, keep):
    """p without the landmarks whose mask entry is False (and their factors), points renumbered"""
    new = np.cumsum(keep) - 1
    blocks = []
    for b in p.blocks:
        ls = [k for k, c in enumerate(SLOT_CLASS[b.type]) if c == 1]
        if not ls:
            blocks.append(b)
            continue
        sel = keep[b.idx[:, ls[0]]]
        idx = b.idx[sel].copy()
        for k in ls:
            idx[:, k] = new[idx[:, k]]
        blocks.append(FactorBlock(b.type, idx, None if b.meas is None else b.meas[sel], b.sigma if b.sigma_bcast else b.sigma[sel],
                                  b.robust_k, None if b.aux_idx is None else b.aux_idx[sel]))
    return dataclasses.replace(p, point=p.point[keep], blocks=blocks, point_keys=None if p.point_keys is None else p.point_keys[keep])


def gap_graph(seed=13):
    """One object whose dynamic landmarks stop for 12 frames in the middle of its span (its motions there are held by
    the smoothing factors alone): two consecutive chunks of one object share no variable."""
    p = synth.make_problem(n_frames=160, n_objects=1, n_static=500, n_dynamic=1200, formulation="hybrid", seed=seed,
                           object_span=(160, 160))
    hb = p.blocks[hybrid_block(p)]
    keep = np.ones(p.n_point, bool)
    lo = np.full(p.n_point, 1 << 30); hi = np.full(p.n_point, -1)
    np.minimum.at(lo, hb.idx[:, 2], hb.idx[:, 0]); np.maximum.at(hi, hb.idx[:, 2], hb.idx[:, 0])
    keep[(hi >= 70) & (lo < 82)] = False
    return SR._weak_priors(drop_points(p, keep))


def interleaved_graph(seed=14):
    """Four objects whose spans overlap in time: runs that pass from one object's chunks to the next object's."""
    return SR._weak_priors(synth.make_problem(n_frames=140, n_objects=4, n_static=500, n_dynamic=2400, formulation="hybrid",
                                              seed=seed, object_span=(90, 120)))


def time_shards(p, split):
    """p cut in time like a 2-rank run: landmarks first seen before frame `split` on shard 0, the others on shard 1
    (poses replicated).  An object alive at `split` has its chunk sequence split between the two."""
    first = np.full(p.n_point, 1 << 30)
    for b in p.blocks:
        sc = SLOT_CLASS[b.type]
        if 1 in sc and 0 in sc:
            np.minimum.at(first, b.idx[:, sc.index(1)], b.idx[:, sc.index(0)])
    return [drop_points(p, first < split), drop_points(p, first >= split)]


def shard_graphs(seed=15):
    p = SR._weak_priors(synth.make_problem(n_frames=160, n_objects=1, n_static=500, n_dynamic=1600, formulation="hybrid",
                                           seed=seed, object_span=(160, 160)))
    return time_shards(p, 80)


SLIDE_GRAPHS = {
    "long_object": long_object_graph,
    "cap": cap_graph,
    "gap": gap_graph,
    "interleaved": interleaved_graph,
    "shard0": lambda: shard_graphs()[0],
    "shard1": lambda: shard_graphs()[1],
}
