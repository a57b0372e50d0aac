"""The window plan and the factor order of the symbolic phase (csrc/window_plan.cuh), built for the host, against their
mirrors: slide_plan.plan and schur_reference.routes for the plan, the general stable sort for the factor order's
run-sorting fast path.  Mutations of a copy of the header, and a chunk cap one below finalize's, each fail the plan
comparison."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import schur_reference as SR
import slide_plan as SP
from dynosam_b200 import synth
from dynosam_b200.problem import SLOT_CLASS

ROOT = SR.ROOT
CSRC = SR.CSRC
GWIN = {"window": 1, "simple": 2, "general": 0, "unsupported": 0}


def _build(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [CSRC]
    if patch is not None:                      # a mutated copy of window_plan.cuh, seen only by this build
        src = open(os.path.join(CSRC, "window_plan.cuh")).read()
        assert src.count(patch[0]) == 1, patch
        d = str(tmp_path / "mut"); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "window_plan.cuh"), "w").write(src.replace(patch[0], patch[1]))
        inc = [d, CSRC]
    so = str(tmp_path / ("window_plan_host%s.so" % ("" if patch is None else "_mut")))
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC,-fopenmp", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "window_plan_host.cu"), "-o", so, "-lgomp"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("window_plan"))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------------------------------------------------- window plan
def _host_plan(lib, p, bi, nseg, cap=None):
    """the library's plan of block bi, fed the mirror's group order and (by default) finalize's chunk cap"""
    b = p.blocks[bi]
    pcols = [k for k, c in enumerate(SLOT_CLASS[b.type]) if c == 0]
    groups = SP.block_groups(p, bi)
    order = np.concatenate([f for _, _, f in groups])
    gp = np.r_[0, np.cumsum([f.size for _, _, f in groups])].astype(np.int32)
    gl = np.array([r if GWIN[route] else -1 for route, r, _ in groups], np.int32)
    n = b.idx.shape[0]; stride = -(-n//32)*32
    prow = np.zeros((2, stride), np.int32)
    for k, col in enumerate(pcols):
        prow[k, :n] = SP.positions(p)[b.idx[order, col]]
    if cap is None:
        cap = SR.CHUNK_CAP[len(pcols) - 1]
    sz = np.zeros(9, np.int64)
    lib.host_plan_windows(C.c_int(len(pcols)), C.c_int(stride), C.c_int64(p.n_pose), _ptr(prow[0]), _ptr(prow[1]), _ptr(gp), _ptr(gl),
                          C.c_int(len(groups)), C.c_int(cap), C.c_int(nseg), _ptr(sz))
    gwin = np.zeros(sz[0], np.uint8); lvar = np.zeros(sz[1], np.uint8)
    jobs = np.zeros((sz[2], 4), np.int32); bat = np.zeros((sz[3], 4), np.int32)
    cb = np.zeros(sz[4], np.int32); cv = np.zeros(sz[5], np.int32)
    lib.host_plan_copy(_ptr(gwin), _ptr(lvar), _ptr(jobs), _ptr(bat), _ptr(cb), _ptr(cv))
    return dict(groups=groups, prow=prow, gwin=gwin, lvar=lvar.reshape(len(pcols), stride), jobs=jobs, batches=bat,
                chunk_batch=cb, cvars=cv.reshape(-1, SR.WIN_NLOC_MAX), ctas=int(sz[6]), flushed=int(sz[7]), all_window=bool(sz[8]))


def _mismatches(H, P):
    """what of the library's plan H differs from the mirror's plan P"""
    bad = []
    cv = H["cvars"]
    if [set(r[r >= 0].tolist()) for r in cv] != P.chunks:
        bad.append("chunks")
    if cv.tolist() != P.slots:
        bad.append("cvars")
    if sorted({(int(j[0]), int(j[1])) for j in H["jobs"]}) != P.runs:
        bad.append("runs")
    if H["ctas"] != P.ctas or H["ctas"] != len(H["jobs"]):
        bad.append("ctas")
    if H["flushed"] != P.flushed:
        bad.append("flushed")
    if H["gwin"].tolist() != [GWIN[route] for route, _, _ in H["groups"]]:
        bad.append("gwin")
    if H["all_window"] != all(route != "simple" for route, _, _ in H["groups"]):
        bad.append("all_window")
    # every window factor's lvar names the window slot its chunk gave that pose slot's variable
    cb, bat = H["chunk_batch"], H["batches"]
    for c in range(len(cb) - 1):
        for g0, g1, f0, f1 in bat[cb[c]:cb[c + 1]]:
            if not all(H["gwin"][g0:g1] == 1):
                bad.append("batches")
            for k in range(H["lvar"].shape[0]):
                if not np.array_equal(cv[c][H["lvar"][k, f0:f1]], H["prow"][k, f0:f1]):
                    bad.append("lvar")
    return sorted(set(bad))


_graphs = {}


def _graph(name):
    if name not in _graphs:
        _graphs[name] = (SP.SLIDE_GRAPHS.get(name) or SR.ROUTE_GRAPHS.get(name) or SEGMENT_GRAPHS[name])()
    return _graphs[name]


def _window_blocks(p):
    return [bi for bi, b in enumerate(p.blocks) if b.type in SR.WINDOW_TYPES]


@pytest.mark.parametrize("name", sorted(SP.SLIDE_GRAPHS) + ["window_np1", "window_np2"])
def test_plan_equals_the_mirror(lib, name):
    p = _graph(name)
    for bi in _window_blocks(p):
        ng = len(SP.block_groups(p, bi))
        nseg = ng//SR.HOST_SEGMENT_GROUPS + 1            # the library's segments on at least that many threads
        H, P = _host_plan(lib, p, bi, nseg), SP.plan(p, bi, nseg)
        assert len(P.chunks) > 0
        assert not _mismatches(H, P), (name, bi, nseg, _mismatches(H, P))


def segment_graph(seed=16):
    """More than HOST_SEGMENT_GROUPS window-path landmarks of two objects in one HYBRID3 block: the host cuts the group
    list into segments, and chunks, slots and runs restart in each."""
    return SR._weak_priors(synth.make_problem(n_frames=200, n_objects=2, n_static=300, n_dynamic=5200, formulation="hybrid",
                                              seed=seed, object_span=(200, 200)))


SEGMENT_GRAPHS = {"segments": segment_graph}


def test_segments_pin_the_plan(lib):
    p = _graph("segments")
    bi = SP.hybrid_block(p)
    assert sum(route == "window" for route, _, _ in SP.block_groups(p, bi)) > SR.HOST_SEGMENT_GROUPS
    plans = {}
    for nseg in (1, 3):
        H, P = _host_plan(lib, p, bi, nseg), SP.plan(p, bi, nseg)
        assert not _mismatches(H, P), (nseg, _mismatches(H, P))
        plans[nseg] = P
    one, three = plans[1], plans[3]
    assert one.runs != three.runs and one.slots != three.slots       # the segments change the plan


MUTATIONS = {
    "entering variable takes the highest free slot":
        ("int fs = 0;\n        for (int32_t p_ : sorted) if (stamp[p_] == -2) { while (occ[fs] >= 0) fs++;",
         "int fs = WIN_NLOC_MAX - 1;\n        for (int32_t p_ : sorted) if (stamp[p_] == -2) { while (occ[fs] >= 0) fs--;", "long_object"),
    "run length": ("std::max<int>(WIN_RUN_MIN_CHUNKS, ", "std::max<int>(WIN_RUN_MIN_CHUNKS + 1, ", "long_object"),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_of_the_plan_fails(tmp_path, mutation):
    old, new, name = MUTATIONS[mutation]
    mut = _build(tmp_path, (old, new))
    p = _graph(name)
    bi = SP.hybrid_block(p)
    bad = _mismatches(_host_plan(mut, p, bi, 1), SP.plan(p, bi))
    print(f"window plan mutation '{mutation}' caught on {name}: {bad}")
    assert bad, mutation


def test_chunk_cap_one_below_fails(lib):
    """the mirror and finalize read the chunk cap from the same line of api.cu; a plan built with one less (NP = 2:
    40 -> 39) disagrees with the mirror"""
    p = _graph("cap")
    bi = SP.hybrid_block(p)
    bad = _mismatches(_host_plan(lib, p, bi, 1, cap=SR.CHUNK_CAP[1] - 1), SP.plan(p, bi))
    print(f"window plan with chunk cap {SR.CHUNK_CAP[1] - 1}: {bad}")
    assert "chunks" in bad


# ---------------------------------------------------------------------------------------------------------- factor order
def _order(lib, frank, key, ngroups, fast):
    perm = np.empty(frank.size, np.int32)
    lib.host_order_block_factors(_ptr(perm), _ptr(frank), _ptr(key), C.c_int64(frank.size), C.c_int64(ngroups), C.c_int(fast))
    return perm


def _runs(rng, nl, fmax, ascending=True, split=False):
    """factors of nl landmarks (ranks 0..nl-1 in shuffled order), each listed contiguously with up to fmax poses;
    split: one landmark's factors in two runs.  -> frank, key"""
    ranks = rng.permutation(nl)
    runs = [(r, np.sort(rng.choice(100000, rng.integers(1, fmax + 1), replace=False))) for r in ranks]
    if not ascending:
        runs[nl//2] = (runs[nl//2][0], np.array([7, 3]))
    if split:
        r, ps = runs[0]
        runs.append((r, ps + 100000))
    frank = np.concatenate([np.full(ps.size, r, np.int32) for r, ps in runs])
    pose = np.concatenate([ps for _, ps in runs]).astype(np.int64)
    return frank, (frank.astype(np.int64) << 32) | pose


@pytest.mark.parametrize("case", ["fast", "not ascending", "rank split", "more runs than groups"])
def test_factor_order_fast_path_equals_the_stable_sort(lib, case):
    rng = np.random.default_rng(7)
    nl = 40000                                        # > 65536 factors: the runs are found in several segments
    frank, key = _runs(rng, nl, 8, ascending=case != "not ascending", split=case == "rank split")
    ngroups = nl - 1 if case == "more runs than groups" else nl
    assert frank.size > 65536
    ref = np.argsort(key, kind="stable")
    fast, fallback = _order(lib, frank, key, ngroups, 1), _order(lib, frank, key, ngroups, 0)
    assert np.array_equal(fallback, ref)
    assert np.array_equal(fast, ref)
