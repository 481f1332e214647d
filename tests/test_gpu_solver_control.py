"""Both paths' L-BFGS and ALM control flow against the oracle, trajectory by trajectory, at the solver settings the yaml never uses
(the case table of tests/test_solver_control.py, which also checks that every case still reaches its branch):

  * parity path (precision 64): every case on generated bumps and hill problems and the N1_M1 / N64_M128 / off_map shapes, whole
    record and coefficients bit for bit against the oracle, unbudgeted and under set_budget(k) against budget_oracle;
  * throughput path: every case at precision 65 (under the case's evaluation budget, CASE_BUDGET) and the structural cases at
    precision 32, and set_budget(k) for k in BUDGETS on 128 problems of the bench's workload, against the same oracle runs.  Every
    decided trajectory (test_solver_control.decided: three runs from inputs perturbed by EPS agree with the unperturbed one) must
    have the oracle's discrete record fields and rho_final, and its continuous fields and coefficients within TOLC;
  * four environments on one grid that differ in mem_size (3, 17, 256, 1024), past (0, 3, 16), int_K and inner_max_iter, in one
    interleaved batch: on the parity path bit for bit the oracle and each environment alone, on the throughput path byte for byte
    each environment alone (history strides of the largest mem_size, rings wrapping at each environment's own), also submitted at
    depth 4 and as one ticket per environment in flight at once;
  * ualm_set_params' limits on mem_size, past and the throughput path's int_K.

Measured on one H100 80GB HBM3 at a 400 W power limit: the worst relative error of a decided trajectory's continuous fields and
coefficients is 2.0e-9 at precision 65 (the 40-evaluation cases; 1.2e-12 .. 5.0e-10 for the budgets 1 .. 34), so TOLC[65] = 1e-7,
and 3.4e-5 at precision 32, so TOLC[32] = 1e-3.  The file takes about 2.5 minutes there on 16 host cores, most of it oracle time."""

import numpy as np
import pytest

import workloads
from harness import ctx, gpu, same_values, solve_diff, split  # noqa: F401


pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sets(bumps_map, hill_map):
    return workloads.case_problems(bumps_map, hill_map)


def _solve(gpu, prec, params, mapdata, pb, budget=0):
    opt = gpu.BatchALMTrajOpt(precision=prec).init(params).set_environment(mapdata).set_budget(budget)
    out = split(pb, opt.optimize(pb))
    opt.close()
    return out


def _check_decided(got, ref, mask, prec, what):
    """every decided trajectory agrees with the oracle; returns (decided count, worst continuous error among them)"""
    worst = 0.0
    for i in np.nonzero(mask)[0]:
        same, err = workloads.trajectory_error(got[i], ref[i])
        g, w = got[i][0], ref[i][0]
        assert same, (what, int(i), [(f, getattr(g, f), getattr(w, f)) for f in workloads.DISCRETE + ("rho_final",) if getattr(g, f) != getattr(w, f)])
        assert err <= workloads.TOLC[prec], (what, int(i), err)
        worst = max(worst, err)
    return int(mask.sum()), worst


# ------------------------------------------------------------------ A: the parity path, bit for bit
@pytest.mark.parametrize("case", list(workloads.SOLVER_CASES))
def test_parity_case_bitwise(gpu, sets, case):
    """unbudgeted against the oracle, and under set_budget(k) against budget_oracle"""
    p = workloads.case_params(case)
    for label, m, pb in sets:
        for k in (0, 1, 5, 30):
            want = workloads.oracle(p, m, pb, k)
            got = _solve(gpu, 64, p, m, pb, k)
            for i in range(pb.B):
                assert not solve_diff(got[i], want[i]), ((case, label, k, i), solve_diff(got[i], want[i]))


# ------------------------------------------------------------------ C: the throughput path, trajectory by trajectory
@pytest.mark.parametrize("prec,case", [(65, c) for c in workloads.SOLVER_CASES] + [(32, c) for c in workloads.STRUCTURAL])
def test_throughput_case_against_oracle(gpu, sets, prec, case):
    p = workloads.case_params(case)
    k = workloads.case_budget(case, prec)
    tot, worst = 0, 0.0
    for label, m, pb in sets:
        ref, mask = workloads.decided(p, m, pb, prec, k)
        got = _solve(gpu, prec, p, m, pb, k)
        n, w = _check_decided(got, ref, mask, prec, (prec, case, label))
        tot += n; worst = max(worst, w)
    print("precision %d, %s (budget %d): %d decided trajectories, worst continuous error %.2e" % (prec, case, k, tot, worst))


@pytest.mark.parametrize("prec,k", [(65, k) for k in workloads.BUDGETS[65]] + [(32, k) for k in workloads.BUDGETS[32]])
def test_throughput_budget_against_oracle(gpu, hill_map, prec, k):
    from uneven_planner_b200 import configs
    p = configs.params_for("hill")
    pb = workloads.bench_problems(hill_map, 128)
    ref, mask = workloads.decided(p, hill_map, pb, prec, k)
    got = _solve(gpu, prec, p, hill_map, pb, k)
    n, w = _check_decided(got, ref, mask, prec, (prec, k))
    print("precision %d, budget %d: %d of %d decided, worst continuous error %.2e" % (prec, k, n, pb.B, w))


# ------------------------------------------------------------------ B: environments that differ in solver parameters
ENV_PARAMS = [dict(), dict(mem_size=3, past=0), dict(mem_size=1024, past=16), dict(mem_size=17, int_K=31, inner_max_iter=50)]


@pytest.fixture(scope="module")
def envs(hill_map):
    """four environments on the hill grid, and a batch of 8 bench problems per environment, interleaved (problem i in environment
    i % 4)"""
    from uneven_planner_b200 import problems
    params = [workloads._p(**kw) for kw in ENV_PARAMS]
    base = workloads.bench_problems(hill_map, 32)
    pbs = [base.select(np.arange(e, 32, 4)) for e in range(4)]
    mixed = problems.concat(pbs, [0, 1, 2, 3]).select(np.array([8 * (i % 4) + i // 4 for i in range(32)]))
    return params, pbs, mixed


@pytest.mark.parametrize("prec", [64, 65, 32])
def test_environments_differing_in_solver_parameters(gpu, hill_map, envs, prec):
    params, pbs, mixed = envs
    where = [(i % 4, i // 4) for i in range(mixed.B)]
    opt = ctx(gpu, prec, params, [hill_map] * 4)
    # first 30 evaluations per problem (the 3- and 17-slot rings wrap by then): a short check before the full solves
    short = [_solve(gpu, prec, params[e], hill_map, pbs[e], 30) for e in range(4)]
    got = split(mixed, opt.set_budget(30).optimize(mixed))
    opt.set_budget(0)
    for i, (e, j) in enumerate(where):
        assert same_values(got[i], short[e][j]), (prec, "budget 30", i, e, j)
    alone = [_solve(gpu, prec, params[e], hill_map, pbs[e]) for e in range(4)]
    runs = {"optimize": split(mixed, opt.optimize(mixed)), "depth 4": split(mixed, opt.wait(opt.submit(mixed, depth=4)))}
    # one ticket per environment in flight at once: lanes whose history strides and rings differ run side by side
    tickets = [opt.submit(pbs[e] if e == 0 else _in_env(pbs[e], e), depth=4) for e in range(4)]
    per_env = [split(pbs[e], opt.wait(t)) for e, t in enumerate(tickets)]
    opt.close()
    for what, got in runs.items():
        for i, (e, j) in enumerate(where):
            assert same_values(got[i], alone[e][j]), (prec, what, i, e, j)
    for e in range(4):
        for j in range(pbs[e].B):
            assert same_values(per_env[e][j], alone[e][j]), (prec, "ticket per environment", e, j)
    if prec == 64:
        for e in range(4):
            want = workloads.oracle(params[e], hill_map, pbs[e])
            for j in range(pbs[e].B):
                assert not solve_diff(alone[e][j], want[j]), ((e, j), solve_diff(alone[e][j], want[j]))
    elif prec == 65:
        # the full solves are chaotic (DESIGN section 2): the oracle comparison runs on the 30-evaluation solves, where the oracle
        # decides 30 of the 32 trajectories
        tot = 0
        for e in range(4):
            ref, mask = workloads.decided(params[e], hill_map, pbs[e], 65, 30)
            tot += _check_decided(short[e], ref, mask, 65, ("env", e))[0]
        print("precision 65, mixed environments at 30 evaluations: %d of %d trajectories decided" % (tot, mixed.B))
        assert tot >= mixed.B // 2, tot


def _in_env(pb, e):
    from uneven_planner_b200 import problems
    return problems.concat([pb], [e])


# ------------------------------------------------------------------ D: ualm_set_params' limits
@pytest.mark.parametrize("prec", [64, 32])
def test_set_params_limits(gpu, bumps_map, prec):
    from uneven_planner_b200 import _lib, problems
    pb = problems.generate(bumps_map, 2, seed=5)
    limits = [("mem_size", 1, True), ("mem_size", 1024, True), ("mem_size", 0, False), ("mem_size", 1025, False),
              ("past", 0, True), ("past", 16, True), ("past", -1, False), ("past", 17, False)]
    if prec == 32:
        limits += [("int_K", 127, True), ("int_K", 128, False)]
    for field, value, ok in limits:
        opt = gpu.BatchALMTrajOpt(precision=prec)
        if ok:
            opt.init(workloads._p(**{field: value})).set_environment(bumps_map)
            res = opt.optimize(pb)[0]
            assert all(r.ret_code in (0, 1, 2) and r.n_evals > 0 for r in res), (field, value)
        else:
            with pytest.raises(gpu.UalmError, match="error %d" % _lib.UALM_ELIMIT):
                opt.init(workloads._p(**{field: value}))
        opt.close()
