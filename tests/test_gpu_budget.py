"""Evaluation budgets and deadline-bounded waits (include/ualm.h: ualm_set_budget, ualm_wait_batch_for, UALM_RET_STOPPED) on the
GPU: the parity path against the budgeted oracle (tests/stop_oracle.cpp) bit for bit, the throughput path against its own unbudgeted solve, and
the deadline on both paths.  Workload: the bench's (BASELINE config 2: 1024 problems on the hill terrain or its stand-in)."""
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stop_oracle as so  # noqa: E402
from harness import RECORD, ctx, gpu, same_problem  # noqa: F401, E402


pytestmark = pytest.mark.gpu

STOPPED = 3


@pytest.fixture(scope="module")
def work(hill_map):
    from uneven_planner_b200 import configs, problems
    return hill_map, configs.params_for("hill"), problems.generate(hill_map, 1024, seed=0, **configs.gen_kwargs("hill"))


@pytest.fixture(scope="module")
def free(gpu, work):
    """unbudgeted solve of the workload per precision: (res, c_xy, c_yaw)"""
    cache = {}

    def get(precision):
        if precision not in cache:
            opt = ctx(gpu, precision, work[1], work[0])
            cache[precision] = opt.optimize(work[2])
            opt.close()
        return cache[precision]
    return get


def _check_budgeted(pb, out, ref, max_evals):
    """stopped problems within the evaluation bound, every other problem exactly its unbudgeted result"""
    n_stop = 0
    for i in range(pb.B):
        r = out[0][i]
        if r.ret_code == STOPPED:
            n_stop += 1
            assert max_evals <= r.n_evals <= max_evals + 64, (i, r.n_evals)
        else:
            assert same_problem(pb, out, ref, i, values=True), i
    return n_stop


@pytest.mark.parametrize("max_evals", [1, 50, 200])
def test_parity_budget_matches_oracle(gpu, work, max_evals):
    import pyoracle as po
    m, params, pb = work
    opt = ctx(gpu, 64, work[1], work[0]).set_budget(max_evals)
    res, cxy, cyaw = opt.optimize(pb)
    opt.close()
    ores = so.budget_batch(po.params_from(params), po.OracleMap(m), pb, max_evals, threads=min(32, os.cpu_count()))
    _, _, ocx, ocy = pb.offsets()
    for i in range(pb.B):
        g, (r, ocxy, ocyaw, _) = res[i], ores[i]
        assert all(getattr(g, f) == getattr(r, f) for f in RECORD), (i, [(f, getattr(g, f), getattr(r, f)) for f in RECORD])
        assert np.array_equal(cxy[ocx[i]:ocx[i + 1]], ocxy) and np.array_equal(cyaw[ocy[i]:ocy[i + 1]], ocyaw), i
    rc = np.array([r.ret_code for r in res])
    assert (rc == STOPPED).any()
    print("max_evals %d: %d of %d problems stopped" % (max_evals, int((rc == STOPPED).sum()), pb.B))


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_budget_above_every_problem_changes_nothing(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0]).set_budget(max(r.n_evals for r in ref[0]) + 1)
    out = opt.optimize(pb)
    opt.close()
    assert all(same_problem(pb, out, ref, i, values=True) for i in range(pb.B))


@pytest.mark.parametrize("precision", [32, 65])
def test_throughput_budget_50(gpu, work, free, precision):
    pb = work[2]
    opt = ctx(gpu, precision, work[1], work[0]).set_budget(50)
    out = opt.optimize(pb)
    opt.close()
    assert _check_budgeted(pb, out, free(precision), 50) > 0


@pytest.mark.parametrize("precision", [64, 32])
def test_deadline(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0])
    t0 = time.perf_counter()
    out = opt.wait(opt.submit(pb, depth=1), timeout_ms=0)
    ms0 = (time.perf_counter() - t0) * 1e3
    n_stop = 0
    for i in range(pb.B):
        if out[0][i].ret_code == STOPPED:
            n_stop += 1
            assert out[0][i].n_lbfgs_iters >= 1
        else:
            assert same_problem(pb, out, ref, i, values=True), i
    assert n_stop > 0
    # the post-solve scan and the MPC hand-over work on the stopped batch (lane 0)
    opt.pb = pb
    assert opt.feasibility(0.01).shape == (pb.B, 10)
    assert opt.mpc_export(pb.N, pb.M)["c_mpc_xy"].size == 12 * int(pb.N.sum())
    # the lane is reusable and its next batch starts without a stop request
    out2 = opt.wait(opt.submit(pb, depth=1))
    assert all(same_problem(pb, out2, ref, i, values=True) for i in range(pb.B))
    # a generous deadline is ualm_wait_batch
    t0 = time.perf_counter()
    out3 = opt.wait(opt.submit(pb, depth=1), timeout_ms=600000.0)
    ms3 = (time.perf_counter() - t0) * 1e3
    assert all(same_problem(pb, out3, ref, i, values=True) for i in range(pb.B))
    opt.close()
    print("precision %d: wait_batch_for(0) %.1f ms (%d of %d stopped), generous deadline %.1f ms" % (precision, ms0, n_stop, pb.B, ms3))


@pytest.mark.parametrize("precision", [64, 32])
def test_budget_argument_and_state_checks(gpu, work, precision):
    from uneven_planner_b200 import _lib
    pb = work[2].select(np.arange(8))
    opt = ctx(gpu, precision, work[1], work[0])
    with pytest.raises(gpu.UalmError, match="error %d" % _lib.UALM_EINVAL):
        opt.set_budget(-1)
    t = opt.submit(pb, depth=1)
    with pytest.raises(gpu.UalmError, match="error %d" % _lib.UALM_ESTATE):
        opt.set_budget(5)
    assert opt.L.ualm_wait_batch_for(opt.h, t, -1.0, None, None, None) == _lib.UALM_EINVAL
    opt.wait(t)
    opt.set_budget(5)
    opt.close()
