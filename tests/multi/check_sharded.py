"""torchrun worker (N GPUs): the time-sharded solver against the unsharded oracle.  Run on a machine with 2 GPUs
through `python -m torch.distributed.run --nproc-per-node 2 ... tests/multi/check_sharded.py`.

Covers both multi-GPU modes of libdynoba: the replicated reduced solve (one all-reduce of the whole reduced system) and
the distributed one (dynoba_set_reduce: cells of the band owned by ranks, a reduce per cell, all-reduce of the boundary
system and of the pose update)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np, torch, torch.distributed as dist
from dynosam_b200 import synth
from dynosam_b200.binding import Solver
import bench
from oracle import oracle as O

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
import datetime
dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(seconds=90))


def _tensor(dev, n):
    class _A:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (dev, False), "version": 3, "strides": None}
    return torch.as_tensor(_A(), device=f"cuda:{local}")


def allreduce(dev, n, stream):
    with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
        dist.all_reduce(_tensor(dev, n))


def reduce(dev, n, root, stream):
    with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
        dist.reduce(_tensor(dev, n), dst=root)


long_kw = dict(n_frames=1200, n_objects=3, n_static=6000, n_dynamic=1500, formulation="hybrid", seed=5,
               object_span=(200, 300), max_static_age=6, max_dynamic_age=6)
cases = [("C1 hybrid, replicated solve", synth.make_config("C1"), False, 0),
         ("C1 wcme, replicated solve", synth.make_config("C1", formulation="wcme"), False, 0),
         ("C3 x0.03, replicated solve", synth.make_config("C3", scale=0.03), False, 0),
         ("1200-frame graph, distributed solve, one cell per rank", synth.make_problem(**long_kw), True, 0),
         ("1200-frame graph, distributed solve, two cells per rank", synth.make_problem(**long_kw), True, 2*world)]
for name, p, distributed, cells in cases:
    print(f"[rank {rank}] case: {name}", file=sys.stderr, flush=True)
    bw = bench.problem_bandwidth(p)
    sh = bench.shard_problem(p, rank, world)
    s = Solver(sh, device=local); s.set_shard(rank, world, allreduce, bw)
    if distributed:
        s.set_reduce(reduce); s.set_partition(cells)
    o = O.OracleProblem(p)
    e = s.error(); eo = o.error()
    assert abs(e - eo) <= 1e-9*eo, (name, e, eo)
    lam = 1e-4
    d = s.solve(lam)
    rc, do = o.schur_solve(lam)
    # compare the pose part (replicated) and this rank's landmarks
    npose = p.n_pose
    keep = sh.meta["kept_points"]
    dl = do[6*npose:].reshape(-1, 3)[keep].reshape(-1)
    err_p = np.linalg.norm(d[:6*npose] - do[:6*npose])/np.linalg.norm(do[:6*npose])
    err_l = np.linalg.norm(d[6*npose:] - dl)/np.linalg.norm(dl)
    assert err_p < 1e-6 and err_l < 1e-6, (name, err_p, err_l)
    st = s.optimize(max_iterations=8); so = o.optimize(max_iterations=8)
    assert st["iterations"] == so["iterations"] and st["inner_iterations"] == so["inner_iterations"], (name, st, so)
    assert abs(st["error_final"] - so["error_final"]) <= (1e-5 if distributed else 1e-6)*so["error_final"], (name, st["error_final"], so["error_final"])
    if rank == 0:
        print(f"{name}: sharded x{world} ok  chi2 {st['error_final']:.9f} vs oracle {so['error_final']:.9f}  step err {err_p:.2e}/{err_l:.2e}", flush=True)
    s.close()
if rank == 0:
    print(f"all sharded x{world} cases ok", flush=True)
dist.destroy_process_group()
