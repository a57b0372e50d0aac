"""CPU half of the star-problem cases (tests/star_cases.py): the 50-digit reference checks itself and an independent objective,
GenericProjectionFactor's Jacobian equals the oracle's restatement, every name of REQUIRED is reached and every claim is true,
and the batch entry points refuse LM parameters under which tryLambda cannot end."""
import numpy as np
import pytest
from mpmath import mp, mpf

import lie_reference as LR
import star_cases as SC
import star_reference as SR
from dynosam_b200 import lie


def test_every_required_name_is_reached():
    hits = set()
    for c in SC.all_cases():
        hits.update(c.hits)
    assert not set(SC.REQUIRED) - hits, sorted(set(SC.REQUIRED) - hits)
    assert SC.STAR_THREADS == 256 and SC.STAR_WARPS == 8 and SC.MR_SCR > 0
    assert np.gcd(SC.PERIOD, SC.STAR_THREADS) == 1 and np.gcd(SC.PERIOD, 32) == 1


def test_size_claims():
    """the block-size claims, derived from STAR_THREADS / STAR_WARPS as read from kernels_star.cu"""
    sizes = [c for c in SC.all_cases() if c.name == "flow:sizes"][0]
    ns = [len(q["depth"]) for q in sizes.problems]
    assert ns == SC.FLOW_N
    assert any(4*n == 6 + 2*n for n in ns)                                              # exact fit: residuals == unknowns
    last_warp = (SC.STAR_WARPS - 1)*32
    assert last_warp in ns and last_warp + 1 in ns                                      # N - 1 >= 7*32: a feature on the last warp
    assert SC.STAR_THREADS in ns and SC.STAR_THREADS + 1 in ns                          # N > STAR_THREADS: a thread holds two features
    assert 2*SC.STAR_THREADS + 1 in ns and max(ns) >= 16*SC.STAR_THREADS
    mixed = [c for c in SC.all_cases() if c.name == "motion:mixed"][0]
    ns = [len(q["kp_prev"]) for q in mixed.problems]
    assert {0, 1, SC.STAR_THREADS + 1, 4*SC.STAR_THREADS} <= set(ns) and any(a == 4*SC.STAR_THREADS and b == 0 for a, b in zip(ns, ns[1:]))


def test_trace_case_claims():
    """each termination / outlier-round case ends as it claims in star_oracle's run (for at least one of its problems; the
    capped cases with outliers left after the last allowed round, outlier_rounds 4 with none found before the cap), and the
    all-removing threshold leaves no flow-projection factor"""
    for c in SC.trace_cases():
        runs = [SC.oracle_run(c, q) for q in c.problems]
        want = c.exit["ended"]
        if want in ("relative", "absolute"):
            assert any(o.get("lm_ended", o["ended"]) == want for o in runs), (c.name, [o["ended"] for o in runs])
        elif want == "cap":
            assert any(o["ended"] == "cap" and o["rounds"] == c.params["outlier_rounds"] for o in runs), c.name
        elif want == "no_outliers":
            assert any(o["ended"] == "no_outliers" and 1 <= o["rounds"] < c.params["outlier_rounds"] for o in runs), c.name
        if c.params.get("outlier_threshold") == 1e-12:
            assert all(not o["inlier"].any() for o in runs)


def test_oracle_single_step_within_its_bound():
    """star_oracle's fp64 single damped step (the dense LM the trace tests compare with) is within the step bound of the 50-digit
    reference on every case small enough for its dense matrices (flow N <= 513, motion N <= 257), in the comparator's units.
    Not flow:cheirality: its depth-1e-12 feature puts 1e30 next to 1 in the dense matrix, whose Cholesky then fails at the
    first lambda (the device's per-feature elimination does not), so the oracle takes no single step there."""
    from oracle import star_oracle as SO
    worst = dict(step=0.0, error_initial=0.0, error_final=0.0)
    for c in SC.flow_cases() + SC.motion_cases():
        if c.name == "flow:cheirality":
            continue
        p = SC.binding_params(c)
        lm = {k: v for k, v in p.items() if k in SO.DEFAULTS}
        keep = [q for q in c.problems if len(q["depth" if c.kind == "flow" else "kp_prev"]) <= (513 if c.kind == "flow" else 257)]
        if not keep:
            continue
        outs = []
        for q in keep:
            if c.kind == "flow":
                outs.append(SO.flow_pose_lm(q["pose_init"], q["pose_prev"], q["calib"], q["kp_prev"], q["depth"], q["flow"], *c.sig, **lm))
            else:
                o = SO.motion_refine_lm(q["pose_prev"], q["pose_cur"], q["motion_init"], q["calib"], q["kp_prev"], q["kp_cur"], q["points_init"], *c.sig, **lm)
                outs.append(o)
        sub = SC.Case(c.name, c.kind, keep, c.hits, c.sig, c.lam)
        w, bad = SC.evaluate(sub, outs)
        assert not bad, bad
        for k in worst:
            worst[k] = max(worst[k], w[k])
    print("star_oracle single step, worst / bound", worst)
    assert worst["step"] <= 16 and worst["error_initial"] <= 4 and worst["error_final"] <= 4, worst


def test_calibration_and_cheirality_claims():
    for name in ("flow:calib_batch", "motion:calib_batch"):
        c = [c for c in SC.all_cases() if c.name == name][0]
        Ks = np.array([q["calib"] for q in c.problems])
        assert len({tuple(k) for k in Ks}) == len(Ks) and set(Ks[:, 2]) >= {0.0, -12.0}
        assert (Ks[:, 0] != Ks[:, 1]).all()
    c = [c for c in SC.all_cases() if c.name == "flow:cheirality"][0]
    q = c.problems[0]
    z = [LR.camera_point(LR.FLOWPROJ2, [LR.vec([0, 0]), LR.pose(q["pose_init"])], LR.vec(q["kp_prev"][j]) + LR.vec([q["depth"][j]]) + LR.vec(q["pose_prev"]),
                         None, LR.vec(q["calib"]))[2] for j in range(4)]
    assert z[0] < 0 and z[1] == 0 and z[2] == 0 and 0 < z[3] <= 1e-12
    assert np.signbit(q["depth"][1]) and not np.signbit(q["depth"][2])
    c = [c for c in SC.all_cases() if c.name == "flow:exit:failed_cholesky"][0]
    assert c.problems[0]["depth"][5] == 5e-324
    c = [c for c in SC.all_cases() if c.name == "motion:cheirality"][0]
    q = c.problems[0]
    qa = [LR.act_inv(LR.pose(q["pose_prev"]), LR.vec(q["points_init"][j, :3]))[2] for j in range(6)]
    qb = [LR.act_inv(LR.pose(q["pose_cur"]), LR.vec(q["points_init"][j, 3:]))[2] for j in range(6)]
    assert qa[0] < 0 < qb[0] and qb[1] < 0 < qa[1] and qa[2] < 0 and qb[2] < 0
    assert qa[3] == 0 and qa[4] == 0 and np.signbit(q["points_init"][4, 2]) and qa[5] > 0 and qb[5] > 0


def test_huber_claims():
    """the whitened norm of the factor a Huber case names is 5 exactly (in 50 digits and in fp64), and k sits at it or one
    ulp either side"""
    for c in SC.all_cases():
        if "huber" not in c.name or c.name.startswith("huber"):
            continue
        q = c.problems[0]; k = c.sig[2]
        if c.kind == "flow":
            r, _, _ = SR._flow_raw(q["pose_init"], q["pose_prev"], q["calib"], q["kp_prev"][0], q["depth"][0], q["flow"][0], jac=False)
            sig = c.sig[0]
        elif c.name.startswith("projection"):
            (r, _, _), _, _ = SR._motion_raw(q["pose_prev"], q["pose_cur"], q["motion_init"], q["calib"], q["kp_prev"][0], q["kp_cur"][0], q["points_init"][0], jac=False)
            sig = c.sig[1]
        else:
            _, _, (r, _, _) = SR._motion_raw(q["pose_prev"], q["pose_cur"], q["motion_init"], q["calib"], q["kp_prev"][0], q["kp_cur"][0], q["points_init"][0], jac=False)
            sig = c.sig[0]
        n = mp.sqrt(sum((x/mpf(sig))**2 for x in r))
        assert n == 5
        want = {"n=k": 5.0, "n=k+ulp": np.nextafter(5.0, 0.0), "n=k-ulp": np.nextafter(5.0, 10.0)}[c.name.split(":")[-1]]
        assert k == want


def _dense_step(blocks, mult, glob, ng, lam):
    """the same damped system assembled dense and solved at once (no elimination)"""
    nl = [b.nl for b in blocks]
    ncol = ng + sum(n*m for n, m in zip(nl, mult))
    rows, rhs = [], []
    c0 = ng
    for Bk, m in zip(blocks, mult):
        for _ in range(m):
            for i in range(len(Bk.b)):
                row = [mpf(0)]*ncol; row[:ng] = Bk.Ag[i]; row[c0:c0 + Bk.nl] = Bk.Al[i]; rows.append(row); rhs.append(Bk.b[i])
            c0 += Bk.nl
    for i in range(len(glob.b)):
        row = [mpf(0)]*ncol; row[:ng] = glob.Ag[i]; rows.append(row); rhs.append(glob.b[i])
    A = mp.matrix(rows); b = mp.matrix(rhs)
    return mp.lu_solve(A.T*A + mpf(lam)*mp.eye(ncol), A.T*b)


@pytest.mark.parametrize("kind", ["flow", "motion"])
def test_elimination_equals_a_dense_solve(kind):
    if kind == "flow":
        q = SC.flow_problem(SC.flow_geometry(31, period=3), 7)
        sig = (1.0, 0.5, 1.0)
        P, mult = SR._distinct(q)
        blocks = [SR._flow_rows(q, q["pose_init"], q["flow"], j, sig, np.ones(P, bool)) for j in range(P)]
        glob, ng = SR.Rows(6, 0), 6
    else:
        q = SC.motion_problem(SC.motion_geometry(32, period=3), 4)
        sig = (0.05, 2.0, 1.0, 1e-2)
        P, mult = SR._distinct_motion(q)
        poses = [q["pose_prev"], q["pose_cur"], q["motion_init"]]
        blocks = [SR._motion_rows(q, poses, q["points_init"], j, sig) for j in range(P)]
        glob, ng = SR._prior_rows(q, poses, sig), 18
    for lam in (1e-5, 1.0):
        e = SR.eliminate(blocks, mult, glob, ng, lam)
        d = _dense_step(blocks, mult, glob, ng, lam)
        assert max(abs(d[i] - e["dg"][i]) for i in range(ng)) < mpf("1e-35")*(1 + max(abs(x) for x in e["dg"]))
        c0 = ng
        for j, m in enumerate(mult):
            for _ in range(m):
                assert max(abs(d[c0 + c] - e["dl"][j][c]) for c in range(blocks[j].nl)) < mpf("1e-35")*(1 + max(abs(x) for x in e["dl"][j]))
                c0 += blocks[j].nl
        assert e["new_lin"] <= e["old_lin"] and e["kappa"] >= 1


def test_flow_objective_equals_the_independent_objective():
    """the reference's objective equals test_star.py's numpy / scipy statement at fp64 values (synth_star's calibration)"""
    import test_star as TS
    from dynosam_b200.synth_star import K5
    q = SC.flow_problem(SC.flow_geometry(33, K=K5, period=30), 30)
    for sig in ((1.0, 0.5, 1.0), (10.0, 3.33, 0.0)):
        e, s = SR.flow_objective(q, q["pose_init"], q["flow"], sig)
        f = TS._flow_pose_objective(q, q["pose_init"], q["flow"], sig)
        assert abs(float(e) - f) <= 1e-12*max(f, 1.0)


def test_projection_jacobian_equals_the_oracle():
    """GenericProjectionFactor: the 50-digit residual and Jacobian against oracle/star_oracle.projection_factor, skew included,
    and the behind-camera branch"""
    from oracle import star_oracle as SO
    rng = np.random.default_rng(5)
    for K in SC.K_BATCH + [SC.K_MAIN]:
        for _ in range(3):
            X = lie.se3_exp(rng.normal(0, 0.3, (1, 6)))[0]
            p = X[9:] + X[:9].reshape(3, 3) @ np.array([rng.uniform(-2, 2), rng.uniform(-1, 1), rng.uniform(4, 20)])
            z = rng.uniform(0, 500, 2)
            r0, Jx, Jp = SO.projection_factor(X, p, K, z)
            T = LR.pose(X)
            r = SR.projection_residual(T, LR.vec(p), LR.vec(K), LR.vec(z)); J = np.array(LR.to_float(SR.projection_jacobian(T, LR.vec(p), LR.vec(K), LR.vec(z))))
            assert np.abs(np.array(LR.to_float(r)) - r0).max() <= 1e-12*np.abs(z).max()
            assert np.abs(J[:, :6] - Jx).max() <= 1e-10*np.abs(Jx).max() and np.abs(J[:, 6:] - Jp).max() <= 1e-10*np.abs(Jp).max()
    X = SC._identity()
    r = SR.projection_residual(LR.pose(X), LR.vec([0.0, 0.0, -1.0]), LR.vec(SC.K_MAIN), LR.vec([0.0, 0.0]))
    J = SR.projection_jacobian(LR.pose(X), LR.vec([0.0, 0.0, -1.0]), LR.vec(SC.K_MAIN), LR.vec([0.0, 0.0]))
    assert r == [2*mpf(SC.K_MAIN[0])]*2 and all(x == 0 for row in J for x in row)


_BAD_LM = [dict(lambda_initial=0.0), dict(lambda_initial=-1e-5), dict(lambda_initial=float("nan")), dict(lambda_initial=float("inf")),
           dict(lambda_factor=1.0), dict(lambda_factor=0.9), dict(lambda_factor=float("nan")), dict(lambda_factor=float("inf")),
           dict(lambda_upper_bound=float("nan")), dict(lambda_factor=float(np.nextafter(1.0, 2.0))), dict(lambda_factor=1.05),
           # tolerances under which a give-up need not end the outer loop
           dict(relative_error_tol=0.0, absolute_error_tol=-1.0), dict(relative_error_tol=float("nan"), absolute_error_tol=float("nan")),
           dict(relative_error_tol=1e-5, absolute_error_tol=-1.0, error_tol=-1.0)]


@pytest.mark.parametrize("bad", _BAD_LM, ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_batches_refuse_lm_parameters_that_cannot_end(bad):
    """feature-free problems (error 0 at the initial values, so even without the check no LM loop could start): the parameters
    are refused with DYNOBA_ERR_BAD_ARG before any device work, on machines with or without a GPU"""
    from dynosam_b200 import binding
    import torch
    fq = dict(pose_init=SC._identity(), pose_prev=SC._identity(), calib=SC.K_MAIN, kp_prev=np.zeros((0, 2)), depth=np.zeros(0), flow=np.zeros((0, 2)))
    mq = dict(pose_prev=SC._identity(), pose_cur=SC._identity(), motion_init=SC._identity(), calib=SC.K_MAIN, kp_prev=np.zeros((0, 2)),
              kp_cur=np.zeros((0, 2)), points_init=np.zeros((0, 6)))
    for fn, q in ((binding.flow_pose_batch, fq), (binding.motion_refine_batch, mq)):
        with pytest.raises(binding.DynobaError) as e:
            fn([q, q], **bad)
        assert e.value.status == -1
        if torch.cuda.is_available():
            assert fn([q, q], lambda_lower_bound=0.0)[0]["iterations"] == 0
        else:
            with pytest.raises(binding.DynobaError) as e:
                fn([q, q], lambda_lower_bound=0.0)
            assert e.value.status == -3
