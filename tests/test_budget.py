"""Evaluation budget of a solve (include/ualm.h, UALM_RET_STOPPED) on the CPU: its reference (tests/stop_oracle.cpp, the oracle's
solve with the stop predicate), and the C ABI entry points that need no device."""
import os
import sys

import numpy as np
import pytest

import pyoracle as po
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stop_oracle as so  # noqa: E402
from uneven_planner_b200 import configs, problems

from harness import solve_diff

NAMES = ["hill", "desert", "volcano", "forest"]
STOPPED = 3


def _golden_problems(terrain, golden, name):
    m = terrain(name)
    gold = golden(name, m)
    pb = problems.generate(m, int(gold["B"]), seed=int(gold["seed"]), **configs.gen_kwargs(name))
    return m, gold, pb, po.params_from(configs.params_for(name))


@pytest.mark.parametrize("name", NAMES)
def test_no_budget_and_large_budget_match_golden(terrain, golden, name):
    m, gold, pb, prm = _golden_problems(terrain, golden, name)
    om = po.OracleMap(m)
    free = po.solve_batch(prm, om, pb, threads=4)
    for max_evals in (0, int(gold["n_evals"].max()) + 1):
        out = so.budget_batch(prm, om, pb, max_evals, threads=4)
        for o, f in zip(out, free):
            assert not solve_diff(o, f), solve_diff(o, f)          # the oracle's orc_solve
        assert np.array_equal(np.array([r[0].ret_code for r in out]), gold["ret_code"]), max_evals
        assert np.array_equal(np.array([r[0].n_evals for r in out]), gold["n_evals"]), max_evals
        assert np.array_equal(np.array([r[0].outer_iters for r in out]), gold["outer_iters"]), max_evals
        assert np.array_equal(np.array([r[0].inner_cost for r in out]), gold["inner_cost"]), max_evals
        assert np.array_equal(np.concatenate([r[1] for r in out]), gold["c_xy"]), max_evals
        assert np.array_equal(np.concatenate([r[2] for r in out]), gold["c_yaw"]), max_evals


@pytest.mark.parametrize("name", ["hill", "volcano"])
def test_small_budgets(terrain, golden, name):
    m, gold, pb, prm = _golden_problems(terrain, golden, name)
    om = po.OracleMap(m)
    free = po.solve_batch(prm, om, pb, threads=4)
    n_stopped = 0
    for max_evals in (1, 20, 100):
        out = so.budget_batch(prm, om, pb, max_evals, threads=4)
        for i, (o, f) in enumerate(zip(out, free)):
            r = o[0]
            if r.ret_code != STOPPED:
                assert not solve_diff(o, f), solve_diff(o, f)          # no stop acted on it: the unbudgeted result
                continue
            n_stopped += 1
            assert max_evals <= r.n_evals <= max_evals + 64, (max_evals, i, r.n_evals)
            assert r.n_evals <= f[0].n_evals     # the same path as the unbudgeted solve up to the stop
            if r.last_lbfgs_ret == 2:    # CANCELED at the earlyExit point: the accepted point was the last one evaluated
                ev = po.eval_one(prm, om, pb, i, o[3])
                assert np.array_equal(ev["c_xy"], o[1]) and np.array_equal(ev["c_yaw"], o[2]), (max_evals, i)
    assert n_stopped > 0


def test_budget_entry_points_exported_and_reject_null_context(built):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    assert hasattr(L, "ualm_set_budget") and hasattr(L, "ualm_wait_batch_for")
    assert L.ualm_set_budget(None, 10) == _lib.UALM_EINVAL
    assert L.ualm_wait_batch_for(None, 0, 1.0, None, None, None) == _lib.UALM_EINVAL
    assert _lib.UALM_RET_STOPPED == STOPPED
