"""Graphs on which the two scalars of each LM decision (oldLin and lin, lm_reference) are checked, each naming the
partial-sum producers and the edges it reaches.  ``tests/test_lm_cases.py`` checks on the CPU that every claim holds and
that the list together reaches every producer; ``tests/test_lm_model_gpu.py`` runs them on the device.

Producers of lin (csrc/api.cu solve_step): backsub_simple_kernel (landmark and flow blocks), backsub_general_kernel
(chains and points in several blocks), pose_model_kernel (pose-only blocks), nav_model_kernel (IMU and nav priors),
prior_model_kernel (dense priors; 256-thread stride: more than 42 poses), pose_delta_norm_kernel (1/2 lambda |dp|^2).
"""
from __future__ import annotations

import dataclasses
import os
import re

import numpy as np

import schur_reference as SR

from dynosam_b200 import synth
from dynosam_b200.problem import (SLOT_CLASS, BETWEEN6, COMBINED_IMU15, FLOWPROJ2, HYBRID3, HYBRID_STEREO3, POSE2POINT3, PRIOR6,
                                  PRIOR_BIAS6, PRIOR_VEL3, SMOOTH_HYBRID6, SMOOTH_POSE6, STEREO3, TERNARY3, MOTIONPOSE3)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")


def _const(fname, pattern):
    m = re.search(pattern, open(os.path.join(CSRC, fname)).read())
    assert m, (fname, pattern)
    return int(m.group(1))


NAV_THREADS = _const("kernels_imu.cu", r"constexpr int NAV_THREADS = (\d+);")
POSE_MODEL_THREADS = _const("kernels_schur.cu", r"pose_model_kernel<<<\(blk\.n \+ \d+\)/(\d+), ")
POSE_ONLY_GRID = _const("api.cu", r"b\.pose_only \? \(int\)\(\(n \+ \d+\)/(\d+)\)")     # what finalize reserves per pose-only block
PRIOR_THREADS = _const("kernels_prior.cu", r"prior_model_kernel<<<1, (\d+), ")
LIN_THREADS = _const("kernels_factor.cu", r"constexpr int LIN_THREADS = (\d+);")
IMU_WARPS = _const("kernels_imu.cu", r"constexpr int IMU_WARPS = (\d+);")
SCHUR_WARPS = _const("kernels_schur.cu", r"constexpr int SCHUR_WARPS = (\d+);")
SUM_THREADS = _const("kernels_factor.cu", r"sum_kernel<<<1, (\d+), ")
GENERAL_PER_CTA = _const("kernels_chain.cu", r"int general_grid\(int n_groups\) \{ return \(n_groups \+ \d+\)/(\d+); \}")
POSE_NORM_THREADS = _const("kernels_schur.cu", r"int pose_norm_grid\(int n\) \{ return \(n \+ \d+\)/(\d+); \}")
LAMBDAS = (1e-300, 1e-5, 1.0, 1e5)
REQUIRED_TYPES = {POSE2POINT3, STEREO3, HYBRID3, HYBRID_STEREO3, FLOWPROJ2, TERNARY3, MOTIONPOSE3, PRIOR6, BETWEEN6,
                  SMOOTH_HYBRID6, SMOOTH_POSE6, COMBINED_IMU15, PRIOR_VEL3, PRIOR_BIAS6}
REQUIRED_POSE_ONLY_N = {NAV_THREADS - 1, NAV_THREADS, NAV_THREADS + 1}


@dataclasses.dataclass
class Case:
    name: str
    problem: object
    partition: int = 0                # dynoba_set_partition: -1 one band, 0 automatic, 2 / 4 cells
    claims: tuple = ()                # boundaries it reaches (checked by test_lm_cases.py)
    lambdas: tuple = LAMBDAS


def prior_at_current(p, idx, seed, scale=30.0):
    """a dense prior over poses idx, linearised at their current values (so d = 0 at the first linearisation)"""
    rng = np.random.default_rng(seed)
    n = len(idx)
    A = rng.normal(0, 1, (6*n + 4, 6*n))
    G = A.T @ A*scale + 5.0*np.eye(6*n)
    return dict(idx=np.asarray(idx, np.int32), lin=p.pose[np.asarray(idx)].copy(), G=G, g=rng.normal(0, 3.0, 6*n), f=0.7)


def _with_priors(p, *priors):
    return dataclasses.replace(p, linear_priors=list(priors))


def pose_first(p):
    """the same graph with its pose-only and navigation blocks ahead of the landmark blocks: their solve partials then
    lie inside the range the linearize and error partials use, so a mis-sized range would sum a live, nonzero partial"""
    first = [b for b in p.blocks if all(c in (0, 3, 4) for c in SLOT_CLASS[b.type])]
    return dataclasses.replace(p, blocks=first + [b for b in p.blocks if b not in first])


def cases():
    out = []
    c1 = synth.make_config("C1")
    out.append(Case("hybrid_c1", c1, claims=("huber",)))
    out.append(Case("hybrid_c1_one_band", c1, partition=-1))
    out.append(Case("hybrid_c1_pose_first", pose_first(c1), claims=("stale_slot_pose",)))
    out.append(Case("all_types", synth.make_all_types_problem(), partition=2))
    out.append(Case("wcme", synth.make_problem(n_frames=12, n_objects=2, n_static=200, n_dynamic=120, formulation="wcme", seed=4),
                    claims=("general",)))
    out.append(Case("wcpe", synth.make_problem(n_frames=12, n_objects=1, n_static=200, n_dynamic=100, formulation="wcpe", seed=5),
                    claims=("general",), lambdas=(1e-5, 1.0, 1e5)))      # gauge freedom: singular up to lambda I
    for k in (1, 2, 3):                                              # one chain per dynamic tracklet
        out.append(Case(f"general_groups_{k}", synth.make_problem(n_frames=8, n_objects=1, n_static=40, n_dynamic=k,
                                                                  formulation="wcme", seed=30 + k), claims=("general",)))
    out.append(Case("imu", synth.make_problem(n_frames=10, n_objects=0, n_static=150, n_dynamic=0, seed=8, robust=False, imu=True)))
    out.append(Case("imu_4cells", synth.make_problem(n_frames=200, n_objects=0, n_static=600, n_dynamic=0, seed=9, robust=False,
                                                     imu=True, max_static_age=4), partition=4))
    for nf in (NAV_THREADS, NAV_THREADS + 1, NAV_THREADS + 2):      # nf - 1 odometry / IMU factors, ahead of the landmarks
        p = synth.make_problem(n_frames=nf, n_objects=0, n_static=300, n_dynamic=0, seed=nf, max_static_age=4)
        out.append(Case(f"pose_only_{nf - 1}", pose_first(p), claims=("stale_slot_pose",)))
        q = synth.make_problem(n_frames=nf, n_objects=0, n_static=200, n_dynamic=0, seed=nf, robust=False, imu=True, max_static_age=4)
        out.append(Case(f"imu_{nf - 1}", pose_first(q), claims=("stale_slot_nav",), lambdas=(1e-5, 1.0)))
    for nf in (42, 43, 85, 86):                                     # B.n = 6 nf either side of 256 and 512
        out.append(Case(f"band_n_{6*nf}", synth.make_problem(n_frames=nf, n_objects=0, n_static=200, n_dynamic=0, seed=nf,
                                                             max_static_age=4), lambdas=(1e-5, 1.0)))
    # sum_kernel's stride: 1023, 1024 and 1025 partials in all, and more than twice the stride
    for n_static, used in ((4077, 1023), (4081, 1024), (4085, 1025), (8385, 2100)):
        out.append(Case(f"used_{used}", synth.make_problem(n_frames=20, n_objects=0, n_static=n_static, n_dynamic=0,
                                                           max_static_age=4, seed=21), claims=(("used", used),),
                        lambdas=(1e-5, 1.0)))
    base = synth.make_problem(n_frames=50, n_objects=1, n_static=500, n_dynamic=100, seed=11, max_static_age=5)
    out.append(Case("one_prior", _with_priors(base, prior_at_current(base, [45, 46, 47, 48, 49], 1))))
    big = list(range(3, 3 + PRIOR_THREADS//6 + 1))                  # 43 poses: 258 rows, past the 256-thread stride
    out.append(Case("two_priors_strided", _with_priors(base, prior_at_current(base, big, 2, 1.0),
                                                       prior_at_current(base, [48, 49], 3)), claims=("prior_stride",)))
    out.append(Case("prior_after_pose_first", _with_priors(pose_first(base), prior_at_current(base, [48, 49], 4)),
                    claims=("stale_slot_pose",)))
    return out


def _ceil(a, b):
    return -(-a//b)


def partial_layout(p):
    """finalize's partial-sum layout (csrc/api.cu), restated: per factor block its linearize range [part_off, +lin) and
    its solve range [bs_off, +bs) with the kind of producer, then the priors, the general groups and 1/2 lambda |dp|^2.
    Returns (blocks [(type, kind, part_off, lin, bs_off, bs, n_groups)], n_lin_partials, used, general group count)."""
    nav = (PRIOR_VEL3, PRIOR_BIAS6, COMBINED_IMU15)
    lmk_blocks = [bi for bi, b in enumerate(p.blocks) if all(c in (0, 1, 2) for c in SLOT_CLASS[b.type])]
    sub = dataclasses.replace(p, blocks=[p.blocks[bi] for bi in lmk_blocks])
    groups, general = {}, set()
    for g in SR.routes(sub):
        groups[lmk_blocks[g.block]] = groups.get(lmk_blocks[g.block], 0) + 1
        if g.route == "general":
            general.add(g.root)
    out, part, bs = [], 0, 0
    for bi, b in enumerate(p.blocks):
        lin = (_ceil(b.n, IMU_WARPS) if b.type == COMBINED_IMU15 else _ceil(b.n, NAV_THREADS)) if b.type in nav else _ceil(b.n, LIN_THREADS)
        pose_only = all(c in (0, 3, 4) for c in SLOT_CLASS[b.type])
        ng = groups.get(bi, 0)
        nb = _ceil(b.n, POSE_ONLY_GRID) if pose_only else _ceil(ng, SCHUR_WARPS)
        kind = ("nav" if b.type in nav else "pose") if pose_only else "simple"
        out.append((b.type, kind, part, lin, bs, nb, ng))
        part += lin; bs += nb
    part += len(p.linear_priors); bs += len(p.linear_priors)
    bs += _ceil(len(general), GENERAL_PER_CTA)
    n_pose_like = p.n_pose + p.n_vel + p.n_bias
    used = bs + _ceil(6*n_pose_like, POSE_NORM_THREADS)
    return out, part, used, len(general)


def b_n(p, t):
    return max(b.n for b in p.blocks if b.type == t)


def claims_hold(case):
    """the claims of a case that its problem actually reaches; returns the set of boundaries it reaches"""
    p = case.problem
    reached = set()
    for b in p.blocks:
        if b.n:
            reached.add(("type", b.type))
    pose_only = {b.n for b in p.blocks if b.type in (PRIOR6, BETWEEN6, SMOOTH_HYBRID6, SMOOTH_POSE6, COMBINED_IMU15,
                                                       PRIOR_VEL3, PRIOR_BIAS6)}
    for n in pose_only:
        reached.add(("pose_only_n", n))
    reached.add(("priors", len(p.linear_priors)))
    for pr in p.linear_priors:
        if 6*len(pr["idx"]) > PRIOR_THREADS:
            reached.add(("prior_stride",))
    reached.add(("partition", case.partition))
    if any(b.robust_k > 0 for b in p.blocks):
        reached.add(("huber",))
    for lam in case.lambdas:
        reached.add(("lambda", lam))
    L, n_lin, used, n_general = partial_layout(p)
    reached.add(("used", used))
    if used > 2*SUM_THREADS:
        reached.add(("used_over_two_strides",))
    reached.add(("general_groups", n_general))
    reached.add(("band_n", 6*(p.n_pose + p.n_vel + p.n_bias)))
    bs_end = L[-1][4] + L[-1][5] if L else 0
    for t, kind, part_off, lin, bs_off, nb, ng in L:
        if kind == "simple" and ng:
            reached.add(("simple_groups_mod", ng % SCHUR_WARPS))
        if kind in ("pose", "nav"):
            # one extra partial reserved after this block would be left unwritten by the solve, and the sum would
            # pick up what the linearize / error partials left there: it lies inside their range and a later
            # producer extends the sum past it
            slot = bs_off + nb
            if slot < n_lin and (slot < bs_end or p.linear_priors or n_general):
                reached.add(("stale_slot_" + kind,))
            if kind == "nav" and t == COMBINED_IMU15:
                reached.add(("nav_n", b_n(p, t)))
    # the symbolic phase's landmark routes (mirror of graphs without navigation variables): window / simple ->
    # backsub_simple_kernel, general -> backsub_general_kernel
    for g in (SR.routes(p) if p.n_vel == 0 and p.n_bias == 0 else []):
        reached.add(("route", g.route))
        if g.route == "general":
            reached.add(("general",))
    return reached
