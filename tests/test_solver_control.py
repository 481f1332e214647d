"""The solver control flow between evaluations -- the Lewis-Overton line search, the L-BFGS history ring and two-loop, the stopping
tests, the ALM dual update and its exits -- at solver settings the yaml never uses.  This file holds the case table and the
per-trajectory comparison that tests/test_gpu_solver_control.py runs both paths against, and checks on the CPU oracle alone that the
table still reaches what it is meant to force:

  * CASES: one parameter set per branch (history ring wraps, the accepted maxima mem_size 1024 / past 16, both delta tests off,
    LBFGSERR_MAXIMUMITERATION followed by more ALM iterations, max_iter 0 / 1, convergence at the first evaluation or the first
    dual update, rho capped at beta, a hard line-search error, LBFGS_STOP), each run on generated problems of two terrains and on
    three edge shapes (N1_M1, N64_M128, off_map of test_gpu_tp_shapes.CASES);
  * the bench's workload at the yaml parameters never fills the yaml's 256-slot ring, so without the table no test wraps it;
  * trajectory by trajectory, the throughput path can only be held to the oracle where the oracle's own outcome does not hinge on
    rounding: a trajectory is *decided* when three runs from inputs perturbed by a relative EPS agree with the unperturbed run.
    The decided fraction of every short-solve workload the GPU test compares stays above a floor, so that comparison cannot pass
    vacuously."""

import numpy as np
import pytest


from workloads import BUDGETS, DISCRETE, SOLVER_CASES, STRUCTURAL, bench_problems, case_budget, case_params, case_problems, decided, oracle




# ------------------------------------------------------------------ the guards (no GPU)
@pytest.fixture(scope="module")
def sets(bumps_map, hill_map):
    return case_problems(bumps_map, hill_map)


@pytest.mark.parametrize("case", list(SOLVER_CASES))
def test_case_reaches_its_branch(built, sets, case):
    """the oracle's own records show each case forcing what it is meant to force"""
    p = case_params(case)
    recs = [r for _, m, pb in sets for r, _, _ in oracle(p, m, pb)]
    assert SOLVER_CASES[case][1](recs), (case, [tuple(getattr(r, f) for f in DISCRETE) + (r.rho_final,) for r in recs])


def test_bench_workload_never_fills_the_yaml_ring(built, hill_map):
    """at the yaml parameters (mem_size 256) no problem of the bench's workload accepts 256 cautious updates in one inner solve: the
    ring's wrap, the full ring and (j + m - 1) % m across zero are reached only by the case table"""
    from uneven_planner_b200 import configs
    p = configs.params_for("hill")
    pb = bench_problems(hill_map, 1024)
    mb = np.array([r.max_bound for r, _, _ in oracle(p, hill_map, pb)])
    print("bench workload at the yaml parameters: max_bound %d (median %d) over %d problems, mem_size %d" %
          (mb.max(), int(np.median(mb)), pb.B, p.mem_size))
    assert mb.max() < p.mem_size


# decided fractions measured on the CPU oracle (x86-64, gcc -O3 -ffp-contract=off): the budgeted workload 0.84 (k = 34) .. 1.0 at
# precision 65, 0.86 at 32; the cases 0.6 (max_mem_past, past1, ... at 40 evaluations) .. 1.0.  The floors sit below with margin
FLOOR_BUDGET = {65: 0.7, 32: 0.7}
FLOOR_CASE = {65: 0.5, 32: 0.5}


@pytest.mark.parametrize("prec", [65, 32])
def test_decided_fraction_of_the_budgeted_workload(built, hill_map, prec):
    from uneven_planner_b200 import configs
    p = configs.params_for("hill")
    pb = bench_problems(hill_map, 128)
    fr = {k: float(decided(p, hill_map, pb, prec, k)[1].mean()) for k in BUDGETS[prec]}
    print("precision %d, decided fraction per budget: %s" % (prec, {k: round(v, 3) for k, v in fr.items()}))
    assert all(v >= FLOOR_BUDGET[prec] for v in fr.values()), fr


@pytest.mark.parametrize("prec", [65, 32])
def test_decided_fraction_of_the_cases(built, sets, prec):
    names = list(SOLVER_CASES) if prec == 65 else list(STRUCTURAL)
    fr = {}
    for c in names:
        p = case_params(c)
        masks = [decided(p, m, pb, prec, case_budget(c, prec))[1] for _, m, pb in sets]
        fr[c] = float(np.concatenate(masks).mean())
    print("precision %d, decided fraction per case: %s" % (prec, {k: round(v, 3) for k, v in fr.items()}))
    low = {c: v for c, v in fr.items() if v < FLOOR_CASE[prec]}
    assert not low, low
