"""Cancelling problems of a batch in flight (include/ualm.h: ualm_cancel_problems) on the CPU: the reference a cancelled parity-path
solve is checked against (tests/cancel_oracle.cpp: the oracle's solve with a stop predicate that holds from its s-th stop test on),
and the argument checks of the Python wrapper that need no device."""
import os
import sys

import numpy as np
import pytest

import pyoracle as po
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import budget_oracle as bo  # noqa: E402
import cancel_oracle as co  # noqa: E402
from uneven_planner_b200 import configs, problems

from harness import solve_diff

STOPPED = 3


def _golden_problems(terrain, golden, name):
    m = terrain(name)
    gold = golden(name, m)
    pb = problems.generate(m, int(gold["B"]), seed=int(gold["seed"]), **configs.gen_kwargs(name))
    return m, gold, pb, po.params_from(configs.params_for(name))


@pytest.mark.parametrize("name", ["hill", "volcano"])
def test_stop_from_the_first_test_is_a_budget_of_one(terrain, golden, name):
    m, _, pb, prm = _golden_problems(terrain, golden, name)
    om = po.OracleMap(m)
    for i in range(pb.B):
        c = co.solve_one(prm, om, pb, i, 1)
        d = solve_diff(c, bo.solve_one(prm, om, pb, i, 1))
        assert not d, d
        assert c[0].ret_code == STOPPED and c[0].n_lbfgs_iters == 1, i


@pytest.mark.parametrize("name", ["hill", "desert", "volcano", "forest"])
def test_stop_past_the_last_test_is_the_free_solve(terrain, golden, name):
    m, gold, pb, prm = _golden_problems(terrain, golden, name)
    om = po.OracleMap(m)
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        ne, site = co.stop_tests(prm, om, pb, i)
        assert ne.size > 0 and np.all(np.diff(ne) >= 0) and set(site.tolist()) <= {0, 1}
        out = co.solve_one(prm, om, pb, i, ne.size + 1)
        d = solve_diff(out, po.solve_one(prm, om, pb, i))
        assert not d, d
        r = out[0]
        assert r.ret_code == gold["ret_code"][i] and r.n_evals == gold["n_evals"][i] and r.inner_cost == gold["inner_cost"][i]
        assert r.n_evals == ne[-1]
        assert np.array_equal(out[1], gold["c_xy"][ocx[i]:ocx[i + 1]]) and np.array_equal(out[2], gold["c_yaw"][ocy[i]:ocy[i + 1]])


def test_every_stop_is_found_again_from_its_record(terrain, golden):
    """match_stopped, the search the GPU test makes, recovers s from the record of the stop-from-test-s solve"""
    m, _, pb, prm = _golden_problems(terrain, golden, "hill")
    om = po.OracleMap(m)
    n = 0
    for i in range(min(pb.B, 6)):
        ne, _ = co.stop_tests(prm, om, pb, i)
        for s in sorted({1, 2, ne.size // 2, ne.size}):
            if s < 1:
                continue
            r, cxy, cyaw, _ = co.solve_one(prm, om, pb, i, s)
            assert r.ret_code == STOPPED and r.n_evals == ne[s - 1]
            s2 = co.match_stopped(prm, om, pb, i, r, cxy, cyaw)
            assert s2 is not None
            d = solve_diff(co.solve_one(prm, om, pb, i, s2), (r, cxy, cyaw, co.solve_one(prm, om, pb, i, s)[3]))
            assert not d, d
            n += 1
    assert n > 0


class _NoDevice:
    """what cancel() would call once its checks pass: records the call instead of reaching a device"""
    def __init__(self):
        self.calls = []

    def ualm_cancel_problems(self, h, ticket, n, idx):
        self.calls.append((ticket, n, [idx[k] for k in range(n)]))
        return 0


def test_wrapper_argument_checks():
    from uneven_planner_b200 import api
    opt = object.__new__(api.BatchALMTrajOpt)
    opt.L, opt.h = _NoDevice(), None
    pb = problems.ProblemBatch(np.full(5, 2, np.int32), np.full(5, 2, np.int32), np.zeros((5, 18)), np.ones(5), np.zeros(10), np.zeros(5))
    opt._tickets = {3: (pb, None)}
    for ticket in (0, -1, "3", None):
        with pytest.raises(ValueError):
            opt.cancel(ticket, [0])
    for idx in ([0, 5], [-1], [[0, 1]], [0.5], np.array([1.0])):
        with pytest.raises(ValueError):
            opt.cancel(3, idx)
    assert opt.L.calls == []                    # a refused call reaches nothing
    opt.cancel(3, [])
    opt.cancel(3, np.array([4, 0, 4], np.int64))
    opt.cancel(3, range(5))
    assert opt.L.calls == [(3, 0, []), (3, 3, [4, 0, 4]), (3, 5, [0, 1, 2, 3, 4])]


def test_cancel_entry_point_exported_and_refuses_without_context(built):
    from uneven_planner_b200 import _lib
    L = _lib.lib()
    assert hasattr(L, "ualm_cancel_problems")
    assert L.ualm_cancel_problems(None, 0, 0, None) == _lib.UALM_EINVAL
