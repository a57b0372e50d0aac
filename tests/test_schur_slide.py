"""The sliding window plan of the landmark elimination (slide_plan.py mirrors it): every graph of
test_schur_slide_gpu.py reaches the boundary it is built for, checked on the plan alone."""
import pytest

import schur_reference as SR
import slide_plan as SP


_cache = {}


def _plan(name):
    if name not in _cache:
        p = SP.SLIDE_GRAPHS[name]()
        _cache[name] = (p, SP.plan(p, SP.hybrid_block(p)))
    return _cache[name]


def test_run_constants():
    assert SP.WIN_RUN_MIN_CHUNKS >= 2 and SP.WIN_RUNS >= 132        # runs slide, and fill an H100 (132 SMs)
    assert SR.CHUNK_CAP[1] <= SR.WIN_NLOC_MAX                       # an entering variable always finds a free slot


@pytest.mark.parametrize("name", sorted(SP.SLIDE_GRAPHS))
def test_plan_is_consistent(name):
    """slots hold exactly each chunk's variables, a variable that stays keeps its slot, a landmark's clique is in one chunk"""
    _, P = _plan(name)
    assert P.np_ == 2
    for c, (ch, row) in enumerate(zip(P.chunks, P.slots)):
        assert {v for v in row if v >= 0} == ch and sum(v >= 0 for v in row) == len(ch)
        if c:
            prev = {v: s for s, v in enumerate(P.slots[c - 1]) if v >= 0}
            assert all(row[prev[v]] == v for v in ch if v in prev)
        assert all(set(vs) <= ch for vs in P.cliques[c])
    assert P.runs[0][0] == 0 and P.runs[-1][1] == len(P.chunks)
    assert all(a[1] == b[0] for a, b in zip(P.runs, P.runs[1:]))


def test_long_object_reuses_slots_over_many_runs():
    _, P = _plan("long_object")
    assert len(P.chunks) >= 150 and len(P.runs) >= 20
    assert P.reused_slots() >= 300
    # the point of the runs: far fewer flushes than one per touched block per chunk
    per_chunk = SP.Plan(2, P.chunks, P.cliques, P.slots, [(c, c + 1) for c in range(len(P.chunks))], 0, 0)
    assert P.flushed*3 < _flushes(per_chunk)


def _flushes(P):
    n = 0
    for c0, c1 in P.runs:
        for c in range(c0, c1):
            slot_of = {v: s for s, v in enumerate(P.slots[c]) if v >= 0}
            n += len({(max(slot_of[x], slot_of[y]), min(slot_of[x], slot_of[y])) for vs in P.cliques[c] for x in vs for y in vs})
    return n


def test_cap_graph_has_widest_chunks_inside_runs():
    _, P = _plan("cap")
    wide = [c for c, ch in enumerate(P.chunks) if len(ch) > SR.CHUNK_CAP[1]]
    assert {len(P.chunks[c]) for c in wide} >= {2*T for T in range(SR.CHUNK_CAP[1]//2 + 1, SR.WIN_TMAX + 1)}
    inner = [c for c in wide if any(c0 < c < c1 - 1 for c0, c1 in P.runs)]
    assert inner, "a 42..48-variable chunk between two others of its run"
    assert any(max(s for s in range(SR.WIN_NLOC_MAX) if P.slots[c][s] >= 0) == SR.WIN_NLOC_MAX - 1 for c in wide)


def test_gap_graph_breaks_the_sequence_inside_a_run():
    _, P = _plan("gap")
    full = [c for _, c, ch in P.transitions() if not (P.chunks[c] & P.chunks[c - 1])]
    assert full, "two consecutive chunks of a run with no variable in common"


def test_interleaved_graph_runs_cross_objects():
    p, P = _plan("interleaved")
    hb = p.blocks[SP.hybrid_block(p)]
    obj_of_motion = dict(zip(hb.idx[:, 1].tolist(), hb.aux_idx.tolist()))
    import numpy as np
    pos = np.empty(p.n_pose, np.int64)
    pos[np.argsort(p.pose_order, kind="stable")] = np.arange(p.n_pose)
    inv = {int(pos[m]): o for m, o in obj_of_motion.items()}
    objs = [{inv[v] for v in ch if v in inv} for ch in P.chunks]
    assert all(len(o) == 1 for o in objs)
    assert len({next(iter(o)) for o in objs}) == 4
    assert any(len({next(iter(objs[c])) for c in range(c0, c1)}) > 1 for c0, c1 in P.runs)


def test_shards_split_one_objects_chunk_sequence():
    p0, P0 = _plan("shard0")
    p1, P1 = _plan("shard1")
    assert len(P0.chunks) >= SP.WIN_RUN_MIN_CHUNKS and len(P1.chunks) >= SP.WIN_RUN_MIN_CHUNKS
    # both shards hold chunks of the one object, and the chunks next to the cut share motion variables across shards
    assert max(P0.chunks[-1]) >= min(P1.chunks[0])
