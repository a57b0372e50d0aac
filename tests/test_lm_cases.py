"""The case list of the LM model scalars (tests/lm_cases.py) reaches every partial-sum producer and the edges it names,
and the partial counts finalize reserves agree with the grids the model kernels launch."""
import lm_cases as LC


def test_reserved_partials_match_the_kernels():
    """finalize reserves (n + 127)/128 partials for every pose-only block; pose_model_kernel and nav_model_kernel write
    one per CTA of their own size.  A mismatch would leave a stale partial in lin or overwrite a neighbour's."""
    assert LC.POSE_ONLY_GRID == LC.POSE_MODEL_THREADS == LC.NAV_THREADS
    assert LC.PRIOR_THREADS == 256


def test_cases_reach_every_producer_and_edge():
    reached, names = set(), set()
    for c in LC.cases():
        r = LC.claims_hold(c)
        for claim in c.claims:
            assert (claim if isinstance(claim, tuple) else (claim,)) in r, (c.name, claim)
        reached |= r
        assert c.name not in names
        names.add(c.name)
    for t in LC.REQUIRED_TYPES:
        assert ("type", t) in reached, t
    for n in LC.REQUIRED_POSE_ONLY_N:
        assert ("pose_only_n", n) in reached, n
    for route in ("window", "simple", "general"):
        assert ("route", route) in reached, route
    for k in (0, 1, 2):
        assert ("priors", k) in reached
    assert ("prior_stride",) in reached and ("huber",) in reached
    for part in (-1, 2, 4):
        assert ("partition", part) in reached
    for lam in LC.LAMBDAS:
        assert ("lambda", lam) in reached
    # partial-sum layout edges (lm_cases.partial_layout restates finalize's layout)
    for n in (LC.SUM_THREADS - 1, LC.SUM_THREADS, LC.SUM_THREADS + 1):
        assert ("used", n) in reached, n
    assert ("used_over_two_strides",) in reached
    for k in (1, 2, 3):
        assert ("general_groups", k) in reached, k
    for r in (LC.SCHUR_WARPS - 1, 0, 1):
        assert ("simple_groups_mod", r) in reached, r
    for edge in (256, 512):
        assert any(("band_n", n) in reached for n in range(edge - 6, edge)), edge
        assert any(("band_n", n) in reached for n in range(edge + 1, edge + 7)), edge
    for n in LC.REQUIRED_POSE_ONLY_N:
        assert ("nav_n", n) in reached, n
    assert ("stale_slot_pose",) in reached and ("stale_slot_nav",) in reached
