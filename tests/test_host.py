"""CPU-only tests: C-ABI surface, host-side containers, oracle self-consistency, sharding logic (gloo)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from dynosam_b200 import synth  # noqa: E402
from dynosam_b200 import problem as P  # noqa: E402


def test_capi_exports_every_declared_symbol():
    """libdynoba.so loads without a GPU and exports every function include/dynoba.h declares."""
    import __graft_entry__ as g
    if not os.path.exists(os.path.join(ROOT, "dynosam_b200", "libdynoba.so")):
        g.build()
    from dynosam_b200 import binding
    lib = binding.load()
    hdr = open(os.path.join(ROOT, "include", "dynoba.h")).read()
    declared = set(re.findall(r"\b(dynoba_[a-z_0-9]+)\s*\(", hdr)) - {"dynoba_allreduce_fn", "dynoba_reduce_fn", "dynoba_status"}
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in dynoba.h but not exported"
    assert set(binding.EXPORTS) <= declared
    assert lib.dynoba_version() >= 100
    assert lib.dynoba_status_string(-4) == b"indeterminate linear system"


def test_no_cpu_fallback_without_device():
    """The product path must fail loudly when there is no CUDA device."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dynosam_b200 import binding
    with pytest.raises(binding.DynobaError) as ei:
        binding.Solver(synth.make_config("C1"))
    assert ei.value.status == binding.ERR_CUDA


def test_product_never_imports_oracle():
    """oracle/ is test infrastructure: nothing under dynosam_b200/ may import, link or dlopen it."""
    bad = re.compile(r"(from\s+oracle|import\s+oracle|libdynoba_oracle|dynoba_oracle\.h|oracle/)")
    for dirpath, _, files in os.walk(os.path.join(ROOT, "dynosam_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp", "Makefile")):
                src = open(os.path.join(dirpath, f)).read()
                assert not bad.search(src), f"{os.path.join(dirpath, f)} references the oracle"


def test_key_encoding_matches_reference_symbols():
    """dynosam_opt/include/dynosam_opt/Symbols.hpp:14-20,126-152 and src/Symbols.cc:160-175
    (reference tests: test_dynamic_point_symbol.cc:40-104)."""
    assert int(P.camera_pose_key(7)) == (ord('X') << 56) | 7
    assert int(P.static_landmark_key(123456)) == (ord('l') << 56) | 123456
    k = int(P.object_motion_key(3, 11))
    assert k >> 56 == ord('H') and (k >> 48) & 0xFF == ord('0') + 3 and k & 0xFFFFFFFFFFFF == 11
    # Cantor pairing round trip, incl. the reference's literal example pairs
    for a, b in [(0, 0), (1, 0), (0, 1), (47, 32), (12345, 678), (2_000_000, 9_999)]:
        z = P.cantor_pair(a, b)
        assert int(z) == (a + b)*(a + b + 1)//2 + b
        k1, k2 = P.cantor_depair(z)
        assert (int(k1), int(k2)) == (a, b)
    dk = int(P.dynamic_landmark_key(5, 77))
    assert dk >> 56 == ord('m') and dk & ((1 << 56) - 1) == int(P.cantor_pair(77, 5))


def test_generator_is_deterministic_and_follows_topology_rules():
    a = synth.make_config("C1"); b = synth.make_config("C1")
    assert np.array_equal(a.pose, b.pose) and np.array_equal(a.point, b.point)
    for x, y in zip(a.blocks, b.blocks):
        assert np.array_equal(x.idx, y.idx) and (x.meas is None or np.array_equal(x.meas, y.meas))
    ptp = a.blocks[0]
    assert ptp.type == P.POSE2POINT3
    cnt = np.bincount(ptp.idx[:, 1])
    assert cnt.min() >= 2 and cnt.max() <= 15                  # min_static_observations, max track age
    hyb = [x for x in a.blocks if x.type == P.HYBRID3][0]
    cnt = np.bincount(hyb.idx[:, 2])[a.meta["n_static"]:]
    assert cnt.min() >= 3 and cnt.max() <= 20                  # min_dynamic_observations, max dynamic age
    # algorithmic bytes per factor of the materialising linearize (SURVEY.md 8d)
    def per_factor(t, sigma_dim=1, aux=False):
        return 4*P.ARITY[t] + 8*P.MEAS_DIM[t] + 8*sigma_dim + (4 if aux else 0) + 8*P.DIM[t]*(P.JCOLS[t] + 1)
    assert per_factor(P.POSE2POINT3) == 280 and per_factor(P.STEREO3) == 280
    assert per_factor(P.TERNARY3) == 332 and per_factor(P.HYBRID3, aux=True) == 432
    expect = sum(x.n*per_factor(x.type, x.sigma_dim, x.aux_idx is not None) for x in a.blocks) + \
        96*(a.n_pose + a.aux_pose.shape[0]) + 24*a.n_point
    assert a.jacobian_bytes() == expect


@pytest.mark.parametrize("formulation", ["hybrid", "wcme"])
def test_oracle_schur_path_equals_dense_normal_equations(formulation):
    from oracle import oracle as O
    p = synth.make_problem(n_frames=10, n_objects=2, n_static=120, n_dynamic=60, formulation=formulation, seed=5)
    o = O.OracleProblem(p)
    H, g = o.dense_normal()
    for lam in (1e-5, 1e-1):
        d_ref = np.linalg.solve(H + lam*np.eye(H.shape[0]), g)
        rc, d = o.schur_solve(lam)
        assert rc == 0 and np.linalg.norm(d - d_ref) <= 1e-7*np.linalg.norm(d_ref)


def test_oracle_lm_reduces_error_and_is_deterministic():
    from oracle import oracle as O
    os.environ["OMP_NUM_THREADS"] = "1"
    p = synth.make_config("C1")
    r1 = O.OracleProblem(p).optimize(); r2 = O.OracleProblem(p).optimize()
    assert r1["error_final"] < 0.01*r1["error_initial"]
    assert r1["iterations"] == r2["iterations"] and abs(r1["error_final"] - r2["error_final"]) <= 1e-9*r1["error_final"]


@pytest.mark.parametrize("formulation,n_static", [("hybrid", 300), ("wcme", 300), ("wcme", 0)])
def test_bandwidth_rule_matches_oracle(formulation, n_static):
    """bench.problem_bandwidth (what the multi-GPU ranks pass as the common min_bandwidth) follows the symbolic phase's
    rule, incl. world-centric tracklet chains, whose points form ONE landmark group."""
    import bench
    from oracle import oracle as O
    p = synth.make_problem(n_frames=30, n_objects=3, n_static=n_static, n_dynamic=150, seed=9, formulation=formulation)
    st = O.OracleProblem(p).optimize(max_iterations=1)
    assert bench.problem_bandwidth(p) == st["bandwidth"]
    assert max(bench.problem_bandwidth(bench.shard_problem(p, r, 2)) for r in range(2)) <= st["bandwidth"]


@pytest.mark.parametrize("formulation", ["hybrid", "wcme"])
def test_landmark_sharding_partitions_the_graph(formulation):
    """Every factor lands on exactly one rank and a factor never refers to a landmark of another rank: the points of a
    world-centric tracklet chain (joined by ternary factors) stay together."""
    import bench
    p = synth.make_problem(n_frames=30, n_objects=3, n_static=300, n_dynamic=150, seed=9, formulation=formulation)
    shards = [bench.shard_problem(p, r, 4) for r in range(4)]
    assert sum(s.n_point for s in shards) == p.n_point
    for t in set(b.type for b in p.blocks):
        assert sum(b.n for s in shards for b in s.blocks if b.type == t) == sum(b.n for b in p.blocks if b.type == t)
    kept = np.stack([s.meta["kept_points"] for s in shards])
    assert (kept.sum(0) == 1).all()
    for s in shards:                       # remapped landmark indices stay inside the shard's own points
        for b in s.blocks:
            for k, c in enumerate(P.SLOT_CLASS[b.type]):
                if c == 1 and b.n:
                    assert b.idx[:, k].min() >= 0 and b.idx[:, k].max() < s.n_point
    # the shard of a rank is a slice in time: its landmarks' first frames do not interleave with the next rank's
    assert np.allclose(sum(s_.n_factors for s_ in shards), p.n_factors)


_GLOO_WORKER = r'''
import os, sys
sys.path.insert(0, {root!r})
import numpy as np, torch, torch.distributed as dist
from dynosam_b200 import synth
import bench
from oracle import oracle as O
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
p = synth.make_problem(n_frames=16, n_objects=2, n_static=200, n_dynamic=100, seed=11)
lam = 1e-4
full = O.OracleProblem(p)
S_full, g_full, pos = full.reduced_dense(lam)
shard = bench.shard_problem(p, rank, world)
S, g, pos_r = O.OracleProblem(shard).reduced_dense(lam)
assert np.array_equal(pos, pos_r)
if rank != 0:                       # damping lambda*I on the pose block is added once (rank 0)
    S -= lam*np.eye(S.shape[0])
t = torch.from_numpy(np.concatenate([S.reshape(-1), g]))
dist.all_reduce(t)                  # the single exchange step of the sharded solver
n = S.shape[0]
S_sum = t[:n*n].numpy().reshape(n, n); g_sum = t[n*n:].numpy()
assert np.abs(S_sum - S_full).max() <= 1e-9*np.abs(S_full).max(), np.abs(S_sum - S_full).max()
assert np.abs(g_sum - g_full).max() <= 1e-9*np.abs(g_full).max()
e = torch.tensor([O.OracleProblem(shard).error()], dtype=torch.float64); dist.all_reduce(e)
assert abs(float(e) - full.error()) <= 1e-9*full.error()
dist.destroy_process_group()
print("rank", rank, "ok")
'''


def test_sharded_reduced_system_allreduce_gloo(tmp_path):
    """world_size-2 gloo run of the multi-GPU exchange: per-rank partial reduced systems (oracle arithmetic)
    all-reduce to the unsharded one; chi^2 partial sums all-reduce to graph.error."""
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_WORKER.format(root=ROOT))
    env = dict(os.environ, OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29571", str(script)],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert r.stdout.count("ok") == 2


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm the driver runs next to ours) prints ONE JSON line with the contract's
    keys, on a tiny time-slice so that it finishes in seconds; it must not touch the CUDA library."""
    import json, subprocess, sys, os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--scale", "0.002",
                          "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip().startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["unit"] == "LM iterations/s"
    for k in ("metric", "value", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] in ("port", "reference") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_bench_own_arm_fails_loudly_without_gpu():
    """No CPU fallback: without a CUDA device the product arm of bench.py exits non-zero instead of printing a number."""
    import subprocess, sys, os
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--config", "C1", "--steps", "1", "--warmup", "0",
                          "--no-cpu-baseline", "--no-e2e"], capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode != 0
    assert not any(l.strip().startswith("{") for l in out.stdout.splitlines())


def test_bench_dump_outputs_names_dtypes_and_budget(tmp_path, monkeypatch):
    """bench.dump_outputs writes pose / point / chi2 (+ flow when present) as float64 .npy; above the byte budget it writes
    the same seeded row sample on every call and stays under the budget."""
    import bench
    rng = np.random.default_rng(3)
    pose, point, flow = rng.normal(size=(500, 12)), rng.normal(size=(20000, 3)), rng.normal(size=(300, 2))

    class Stub:
        def values(self):
            return pose, point, flow
    st = {"error_initial": 2.0, "error_final": 1.0}
    bench.dump_outputs(str(tmp_path / "full"), Stub(), st)
    full = {f: np.load(tmp_path / "full" / f) for f in os.listdir(tmp_path / "full")}
    assert sorted(full) == ["chi2.npy", "flow.npy", "point.npy", "pose.npy"]
    assert all(a.dtype == np.float64 for a in full.values())
    assert np.array_equal(full["point.npy"], point) and np.array_equal(full["chi2.npy"], [2.0, 1.0])
    monkeypatch.setattr(bench, "DUMP_BUDGET", 100_000)
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), Stub(), st)
    sizes = sum(os.path.getsize(tmp_path / "a" / f) for f in os.listdir(tmp_path / "a"))
    assert sizes <= 100_000 + 4*128                                # (+ one .npy header per file)
    for f in os.listdir(tmp_path / "a"):
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype == np.float64 and np.array_equal(a, b)
    p = np.load(tmp_path / "a" / "point.npy")
    assert 0 < p.shape[0] < point.shape[0] and (p[:, None, :] == point[None, :200, :]).all(2).any(1).sum() > 0


def test_gtsam_adapter_compiles_against_api_stubs():
    """include/dynoba_gtsam_adapter.hpp (the drop-in for RegularBackendModule.cc:405-428) is real code: it must compile,
    with every factor branch incl. stereo and flow projection, against declarations of the GTSAM 4.2 / DynOSAM API it
    touches (tests/stubs/; GTSAM itself is absent from the container)."""
    for extra in ([], ["-DDYNOBA_FLOWPROJ_ACCESSORS"]):
        r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Wno-pragma-once-outside-header", "-DDYNOBA_WITH_GTSAM", *extra,
                            "-I", os.path.join(ROOT, "tests", "stubs"), "-I", os.path.join(ROOT, "include"), "-x", "c++",
                            os.path.join(ROOT, "include", "dynoba_gtsam_adapter.hpp")], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-3000:]
    src = open(os.path.join(ROOT, "include", "dynoba_gtsam_adapter.hpp")).read()
    for t in ("DYNOBA_STEREO3", "DYNOBA_HYBRID_STEREO3", "DYNOBA_FLOWPROJ2", "dynoba_set_calibration"):
        assert t in src


def test_motion_solver_adapter_compiles_against_api_stubs():
    """include/dynoba_motion_solver_adapter.hpp (the binding of the batched per-object refinements, MotionSolver.cc:673-713) is
    real code over gtsam value types: it must compile against the same API stubs."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Wextra", "-Wno-pragma-once-outside-header", "-I", os.path.join(ROOT, "tests", "stubs"),
                        "-I", os.path.join(ROOT, "include"), "-x", "c++", os.path.join(ROOT, "include", "dynoba_motion_solver_adapter.hpp")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    src = open(os.path.join(ROOT, "include", "dynoba_motion_solver_adapter.hpp")).read()
    for t in ("dynoba_flow_pose_batch", "dynoba_motion_refine_batch", "OpticalFlowAndPoseBatch", "MotionOnlyRefinementBatch"):
        assert t in src


def _build_capi_smoke(tmp_path):
    exe = str(tmp_path / "capi_smoke")
    libdir = os.path.join(ROOT, "dynosam_b200")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "capi", "capi_smoke.c"),
                        "-o", exe, "-L", libdir, "-ldynoba", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def test_plain_c_program_links_the_abi(tmp_path):
    """dynoba.h is valid C99 and a C program links libdynoba.so directly (no ctypes).  Without a GPU the program must
    stop at dynoba_create with DYNOBA_ERR_CUDA (exit code 3): there is no CPU path to fall back to."""
    import torch
    exe = _build_capi_smoke(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    if torch.cuda.is_available():
        assert r.returncode == 0, r.stdout + r.stderr
    else:
        assert r.returncode == 3, (r.returncode, r.stdout, r.stderr)


_GLOO_CELL_WORKER = r'''
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tools"))
import numpy as np, torch, torch.distributed as dist
from dynosam_b200 import synth
import bench, cell_proto
from oracle import oracle as O
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
# a trajectory long enough for two cells: static + one object, short tracks -> narrow band
p = synth.make_problem(n_frames=90, n_objects=1, n_static=500, n_dynamic=80, seed=4, max_static_age=3, max_dynamic_age=3, object_span=(30, 40))
lam = 1e-3
full = O.OracleProblem(p)
S_full, g_full, pos = full.reduced_dense(lam)
shard = bench.shard_problem(p, rank, world)               # time shard: this rank's landmarks and pose-only factors
S, g, pos_r = O.OracleProblem(shard).reduced_dense(lam)
assert np.array_equal(pos, pos_r)
if rank != 0:
    S -= lam*np.eye(S.shape[0])                           # damping is added once
# (reduced_dense returns the system in SOLVER order -- the band); padding to whole model tiles
T = cell_proto.T
n = S.shape[0]; npad = (n + T - 1)//T*T
def ordered(M, v):
    Mo = np.eye(npad); Mo[:n, :n] = M
    vo = np.zeros(npad); vo[:n] = v
    if rank != 0: Mo[n:, n:] = 0.0                        # padding diagonal also only once
    return Mo, vo
So, go = ordered(S, g)
bw = bench.problem_bandwidth(p); WB = (bw + T - 1)//T
x = cell_proto.cell_solve(So, go, WB, 2, rank, world, dist)
ref = np.linalg.solve(S_full, g_full)
err = np.abs(x[:n] - ref).max()/np.abs(ref).max()
assert err < 1e-8, err
dist.destroy_process_group()
print("rank", rank, "cells ok", err)
'''


def test_distributed_cell_solve_gloo(tmp_path):
    """world_size-2 gloo run of the DISTRIBUTED reduced solve's exchange pattern on the executable specification
    (tools/cell_proto.py): per-rank partial reduced systems of the time-sharded graph (oracle arithmetic), a reduce per cell
    to its owner, all-reduce of the boundary-separator system and of the solution; the result equals the dense solve of
    the unsharded system."""
    script = tmp_path / "worker_cells.py"
    script.write_text(_GLOO_CELL_WORKER.format(root=ROOT))
    env = dict(os.environ, OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29573", str(script)],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.count("cells ok") == 2


def test_plan_partition_is_a_pure_host_function():
    """dynoba_plan_partition needs neither a handle nor a device: monotone bounds covering the pose axis; with one cell per
    rank the end ranks (plain chain + short spiked chain) get more of the axis than the middle ranks (two spiked chains)."""
    from dynosam_b200.binding import plan_partition
    for world in (1, 2, 4, 8):
        b = plan_partition(60027, 959, world)
        assert b[0] == 0 and b[-1] == 60027 and (np.diff(b) > 0).all(), (world, b)
    b = np.diff(plan_partition(60027, 959, 8))
    assert b[0] > 1.5*b[3] and b[-1] > 1.5*b[3] and abs(int(b[2]) - int(b[4])) <= 64
    # a system too short for eight cells still yields valid bounds (ranks without a cell own an empty slice)
    b = plan_partition(300, 959, 8)
    assert b[0] == 0 and b[-1] == 300 and (np.diff(b) >= 0).all()
