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
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import budget_oracle as bo  # noqa: E402

THREADS = min(32, os.cpu_count() or 1)

# lbfgs return codes (oracle/oracle.cpp)
LBFGS_CONVERGENCE, LBFGS_STOP, LBFGS_CANCELED = 0, 1, 2
LBFGSERR_MINIMUMSTEP, LBFGSERR_MAXIMUMITERATION = -1011, -1008

DISCRETE = ("ret_code", "outer_iters", "n_evals", "n_lbfgs_iters", "last_lbfgs_ret", "max_bound")
CONTINUOUS = ("inner_cost", "jerk_cost", "total_T", "res_h", "res_g", "scale_fx")
RECORD = DISCRETE + CONTINUOUS + ("rho_final",)

# the per-trajectory rule of the throughput path against the oracle (test_gpu_solver_control.py says what was measured):
# relative perturbation of the inputs that decides a trajectory, and the bound on its continuous fields and coefficients
EPS = {65: 1e-11, 32: 1e-5}
TOLC = {65: 1e-7, 32: 1e-3}
BUDGETS = {65: [1, 2, 3, 5, 8, 13, 21, 34], 32: [1, 2, 3]}


def _p(**kw):
    from uneven_planner_b200 import _lib
    p = _lib.default_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _any(pred):
    return lambda rs: any(pred(r) for r in rs)


def _all(pred):
    return lambda rs: all(pred(r) for r in rs)


# name -> (overrides of default_params(), what the oracle's records must show over the case problems)
CASES = {
    # the history ring wraps: a full ring (max_bound == mem_size) in inner solves of more than 2 mem_size iterations each
    "ring_m2": (dict(mem_size=2, past=0, g_epsilon=1e-12, inner_max_iter=40),
                _any(lambda r: r.max_bound == 2 and r.n_lbfgs_iters >= 40 * (r.outer_iters + 1) - 1)),
    "ring_m3": (dict(mem_size=3, past=0, g_epsilon=1e-12, inner_max_iter=60),
                _any(lambda r: r.max_bound == 3 and r.n_lbfgs_iters >= 60 * (r.outer_iters + 1) - 1)),
    "ring_m17": (dict(mem_size=17, past=0, g_epsilon=1e-12, inner_max_iter=80),
                 _any(lambda r: r.max_bound == 17 and r.n_lbfgs_iters >= 80 * (r.outer_iters + 1) - 1)),
    # the accepted maxima: more history than the yaml's 256 slots, and the 16-slot pf ring past its first wrap ending in LBFGS_STOP
    "max_mem_past": (dict(mem_size=1024, past=16),
                     lambda rs: any(r.max_bound > 256 for r in rs) and any(r.last_lbfgs_ret == LBFGS_STOP for r in rs)),
    # past 0: neither delta test (never LBFGS_STOP)
    "past0": (dict(past=0, inner_max_iter=300),
              lambda rs: all(r.last_lbfgs_ret != LBFGS_STOP for r in rs) and any(r.last_lbfgs_ret == LBFGS_CONVERGENCE for r in rs)),
    # past 1: the line search's early exit at delta / 1 and the one-slot pf ring
    "past1": (dict(past=1), _any(lambda r: r.last_lbfgs_ret == LBFGS_STOP)),
    # LBFGSERR_MAXIMUMITERATION, then the ALM loop goes on
    "inner1": (dict(inner_max_iter=1), _any(lambda r: r.last_lbfgs_ret == LBFGSERR_MAXIMUMITERATION and r.outer_iters >= 1)),
    "inner2": (dict(inner_max_iter=2), _any(lambda r: r.last_lbfgs_ret == LBFGSERR_MAXIMUMITERATION and r.outer_iters >= 1 and r.max_bound == 1)),
    # ret_code 2 after the first / second inner solve
    "max_iter0": (dict(max_iter=0), lambda rs: all(r.outer_iters <= 1 for r in rs) and any(r.ret_code == 2 and r.outer_iters == 1 for r in rs)),
    "max_iter1": (dict(max_iter=1), lambda rs: all(r.outer_iters <= 2 for r in rs) and any(r.ret_code == 2 and r.outer_iters == 2 for r in rs)),
    "max_iter0_inner1": (dict(max_iter=0, inner_max_iter=1),
                         _all(lambda r: r.outer_iters <= 1 and r.n_lbfgs_iters <= 1 and r.ret_code in (0, 2))),
    # every inner solve converges at its first evaluation (no line search at all)
    "g_eps_large": (dict(g_epsilon=1e3), _any(lambda r: r.n_lbfgs_iters == 0 and r.n_evals == r.outer_iters and r.ret_code == 2)),
    # converged at the first dual update (after a two-iteration inner solve, so that the outcome does not hinge on the trajectory)
    "eps_con_large": (dict(epsilon_con=1e6, inner_max_iter=2),_all(lambda r: r.ret_code == 0 and r.outer_iters == 0)),
    # rho reaches the cap beta
    "beta_cap": (dict(beta=3.0), _any(lambda r: r.rho_final == 3.0 and r.outer_iters >= 2)),
    # a hard line-search error: ret_code 1 before any dual update
    "min_step_large": (dict(min_step=1e3),
                       _all(lambda r: r.ret_code == 1 and r.last_lbfgs_ret == LBFGSERR_MINIMUMSTEP and r.outer_iters == 0 and r.rho_final == 1.0)),
    # LBFGS_STOP within a few iterations of every inner solve
    "delta_large": (dict(delta=0.5), _any(lambda r: r.last_lbfgs_ret == LBFGS_STOP and r.n_lbfgs_iters <= 5 * (r.outer_iters + 1))),
}
# the cases whose outcome is fixed by their structure rather than by the trajectory: the only ones precision 32 is compared at
STRUCTURAL = ("max_iter0_inner1", "g_eps_large", "eps_con_large")
# evaluation budget of the cases where the throughput path is compared with the oracle at precision 65: long enough for the case to
# reach its branch (ring_m17 fills its ring, max_mem_past wraps its pf ring), short enough that most trajectories stay decided
CASE_BUDGET = dict({c: 40 for c in CASES}, ring_m2=20, ring_m3=20)


def case_budget(name, prec):
    return CASE_BUDGET[name] if prec == 65 else 0


def case_params(name):
    return _p(**CASES[name][0])


def case_problems(bumps, hill):
    """[(label, map, batch)]: generated problems on the bumps map and on the hill terrain, and the edge shapes on the bumps map"""
    from test_gpu_tp_shapes import CASES as SHAPES
    from uneven_planner_b200 import configs, problems
    shapes = problems.concat([SHAPES[k]() for k in ("N1_M1", "N64_M128", "off_map")], [0, 0, 0])
    shapes.env = None
    gb = problems.generate(bumps, 6, seed=7)
    gh = problems.generate(hill, 6, seed=11, **configs.gen_kwargs("hill"))
    both = problems.concat([gb, shapes], [0, 0])
    both.env = None
    return [("bumps", bumps, both), ("hill", hill, gh)]


def bench_problems(hill, B):
    """the first B problems of the bench's workload (BASELINE config 2, hill parameters, seed 0)"""
    from uneven_planner_b200 import configs, problems
    return problems.generate(hill, B, seed=0, **configs.gen_kwargs("hill"))


def perturb(pb, eps, seed):
    """pb with its inner waypoints and total time moved by a relative eps in a seeded random direction"""
    import copy
    rng = np.random.default_rng(seed)
    out = copy.copy(pb)
    for f in ("inner_xy", "inner_yaw", "total_time"):
        a = np.asarray(getattr(pb, f), np.float64)
        setattr(out, f, a + eps * np.maximum(np.abs(a), 1.0) * rng.choice([-1.0, 1.0], a.shape))
    return out


def oracle(params, mapdata, pb, max_evals=0):
    """budget_oracle (max_evals 0: the oracle's own solve) of every problem: [(record, c_xy, c_yaw)]"""
    import pyoracle as po
    out = bo.solve_batch(po.params_from(params), po.OracleMap(mapdata), pb, max_evals, threads=THREADS)
    return [(r, cxy, cyaw) for r, cxy, cyaw, _ in out]


def _rel(a, b, floor):
    return abs(float(a) - float(b)) / max(abs(float(b)), floor)


def trajectory_error(got, want):
    """(discrete fields and rho_final all equal, worst relative error of the continuous fields and coefficients) of one trajectory.
    A residual is measured against max(|oracle|, 1e-6) (near zero it is a cancellation), everything else against its own size."""
    g, gx, gy = got
    w, wx, wy = want
    same = all(getattr(g, f) == getattr(w, f) for f in DISCRETE) and g.rho_final == w.rho_final
    err = max(_rel(getattr(g, f), getattr(w, f), 1e-6 if f in ("res_h", "res_g") else 1e-300) for f in CONTINUOUS)
    for a, b in ((gx, wx), (gy, wy)):
        err = max(err, float(np.linalg.norm(np.asarray(a) - b) / max(np.linalg.norm(b), 1e-300)))
    if not np.isfinite(err):
        err = np.inf
    return same, err


def agrees(got, want, prec):
    same, err = trajectory_error(got, want)
    return same and err <= TOLC[prec]


def decided(params, mapdata, pb, prec, max_evals=0):
    """(oracle solves, boolean mask of the decided trajectories): three runs from seeded perturbations of the inputs by EPS[prec]
    all agree with the unperturbed run under the same rule the GPU is held to"""
    ref = oracle(params, mapdata, pb, max_evals)
    mask = np.ones(pb.B, bool)
    for s in range(3):
        alt = oracle(params, mapdata, perturb(pb, EPS[prec], 1000 + s), max_evals)
        mask &= np.array([agrees(alt[i], ref[i], prec) for i in range(pb.B)])
    return ref, mask


# ------------------------------------------------------------------ the guards (no GPU)
@pytest.fixture(scope="module")
def sets(bumps_map, hill_map):
    return case_problems(bumps_map, hill_map)


@pytest.mark.parametrize("case", list(CASES))
def test_case_reaches_its_branch(built, sets, case):
    """the oracle's own records show each case forcing what it is meant to force"""
    p = case_params(case)
    recs = [r for _, m, pb in sets for r, _, _ in oracle(p, m, pb)]
    assert CASES[case][1](recs), (case, [tuple(getattr(r, f) for f in DISCRETE) + (r.rho_final,) for r in recs])


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
    names = list(CASES) if prec == 65 else list(STRUCTURAL)
    fr = {}
    for c in names:
        p = case_params(c)
        masks = [decided(p, m, pb, prec, case_budget(c, prec))[1] for _, m, pb in sets]
        fr[c] = float(np.concatenate(masks).mean())
    print("precision %d, decided fraction per case: %s" % (prec, {k: round(v, 3) for k, v in fr.items()}))
    low = {c: v for c, v in fr.items() if v < FLOOR_CASE[prec]}
    assert not low, low
