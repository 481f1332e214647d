"""The throughput path advances a submitted batch on the device: its group loops run after ualm_submit_batch returns, publish into
the mailbox and take cancels and deadlines with no further library call (include/ualm.h, DESIGN 3g).  Precision 64 (the parity
path, which always worked this way) is the control.  Every result is compared byte for byte with the same batch solved by
optimize.  Workload: 1024 problems on the hill terrain or its stand-in with hill parameters."""
import time

import numpy as np
import pytest

from harness import ctx, gpu, same_bytes, same_problem  # noqa: F401


pytestmark = pytest.mark.gpu

STOPPED = 3


@pytest.fixture(scope="module")
def work(hill_map):
    from uneven_planner_b200 import configs, problems
    return hill_map, configs.params_for("hill"), problems.generate(hill_map, 1024, seed=0, **configs.gen_kwargs("hill"))


@pytest.fixture(scope="module")
def free(gpu, work):
    """optimize of the workload per precision: (res, c_xy, c_yaw)"""
    cache = {}

    def get(precision):
        if precision not in cache:
            opt = ctx(gpu, precision, work[1], work[0])
            cache[precision] = opt.optimize(work[2])
            opt.close()
        return cache[precision]
    return get


def _wait_time(opt, pb):
    """seconds of one submit + wait of the batch (its first run warms the context up)"""
    opt.wait(opt.submit(pb, depth=1))
    t0 = time.perf_counter()
    opt.wait(opt.submit(pb, depth=1))
    return time.perf_counter() - t0


def _idle(T):
    """how long a test leaves the batch alone: far longer than it needs on the device"""
    return max(20.0 * T, 2.0)


@pytest.mark.parametrize("precision", [32, 65, 64])
def test_batch_completes_without_host_calls(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0])
    T = _wait_time(opt, pb)
    t = opt.submit(pb, depth=1)
    time.sleep(_idle(T))
    out = opt.outputs(pb)
    idx, pending = opt.poll(t, out, 0.0)
    assert idx.size == pb.B and pending == 0, (idx.size, pending)
    assert same_bytes(out, ref)
    assert same_bytes(opt.wait(t), ref)
    opt.close()
    print("precision %d: wait %.1f ms; all %d problems published during a sleep of %.1f s" % (precision, 1e3 * T, pb.B, _idle(T)))


@pytest.mark.parametrize("precision", [32, 64])
def test_eight_tickets_complete_without_host_calls(gpu, work, precision):
    pb = work[2]
    parts = [pb.select(np.arange(k * 128, (k + 1) * 128)) for k in range(8)]
    opt = ctx(gpu, precision, work[1], work[0])
    refs = [opt.optimize(p) for p in parts]
    T = _wait_time(opt, pb)
    tickets = [opt.submit(p, depth=8) for p in parts]
    assert sorted(tickets) == list(range(8))
    time.sleep(_idle(T))
    for t, p, r in zip(tickets, parts, refs):
        out = opt.outputs(p)
        idx, pending = opt.poll(t, out, 0.0)
        assert idx.size == p.B and pending == 0, (t, idx.size, pending)
        assert same_bytes(out, r), t
    for t, r in zip(tickets, refs):
        assert same_bytes(opt.wait(t), r), t
    for t, p, r in zip(tickets, parts, refs):         # every lane takes its next batch
        t2 = opt.submit(p, depth=8)
        assert t2 == t
        assert same_bytes(opt.wait(t2), r)
    opt.close()


@pytest.mark.parametrize("precision", [32, 64])
def test_mixed_environment_batch_completes_without_host_calls(gpu, work, terrain, precision):
    from uneven_planner_b200 import configs, problems
    m0, p0, pb = work
    names = ["volcano", "forest", "desert"]
    maps = [m0] + [terrain(n) for n in names]
    params = [p0] + [configs.params_for(n) for n in names]
    parts = [pb.select(np.arange(200))] + [problems.generate(maps[k + 1], 200, seed=7 + k, **configs.gen_kwargs(n)) for k, n in enumerate(names)]
    mixed = problems.concat(parts, [0, 1, 2, 3])
    opt = gpu.BatchALMTrajOpt(precision=precision)
    for e in range(4):
        opt.init(params[e], env=e).set_environment(maps[e], env=e)
    ref = opt.optimize(mixed)
    T = _wait_time(opt, mixed)
    t = opt.submit(mixed, depth=1)
    time.sleep(_idle(T))
    out = opt.outputs(mixed)
    idx, pending = opt.poll(t, out, 0.0)
    assert idx.size == mixed.B and pending == 0, (idx.size, pending)
    assert same_bytes(out, ref) and same_bytes(opt.wait(t), ref)
    t = opt.submit(mixed, depth=1)
    assert same_bytes(opt.wait(t), ref)
    opt.close()


@pytest.mark.parametrize("precision", [32, 65, 64])
def test_cancel_reaches_a_running_batch(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0])
    T = _wait_time(opt, pb)
    t = opt.submit(pb, depth=1)
    time.sleep(T / 4)
    t0 = time.perf_counter()
    opt.cancel(t, np.arange(pb.B))
    time.sleep(max(0.0, _idle(T) - (time.perf_counter() - t0)))
    out = opt.outputs(pb)
    idx, pending = opt.poll(t, out, 0.0)
    assert idx.size == pb.B and pending == 0, (idx.size, pending)
    assert same_bytes(out, opt.wait(t))
    stopped = [i for i in range(pb.B) if out[0][i].ret_code == STOPPED]
    for i in range(pb.B):
        if out[0][i].ret_code != STOPPED:
            assert same_problem(pb, out, ref, i), i
    assert stopped
    assert all(out[0][i].n_lbfgs_iters >= 1 for i in stopped)
    assert np.mean([r.n_evals for r in out[0]]) < np.mean([r.n_evals for r in ref[0]])
    opt.close()
    print("precision %d: %d of %d stopped by a cancel %.1f ms after submit" % (precision, len(stopped), pb.B, 250 * T))


@pytest.mark.parametrize("precision", [32, 65])
def test_budget_and_deadline_under_the_device_loop(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0])
    opt.set_budget(50)
    budget_ref = opt.optimize(pb)
    assert same_bytes(opt.wait(opt.submit(pb, depth=1)), budget_ref)
    opt.set_budget(0)
    out = opt.wait(opt.submit(pb, depth=1), timeout_ms=0)
    rc = np.array([r.ret_code for r in out[0]])
    assert (rc == STOPPED).any()
    for i in np.flatnonzero(rc != STOPPED):
        assert same_problem(pb, out, ref, i), i
    assert same_bytes(opt.wait(opt.submit(pb, depth=1)), ref)         # the lane is reusable
    opt.close()


@pytest.mark.parametrize("precision", [32, 65])
def test_phase_entry_points_run_through_the_device_loop(gpu, work, precision):
    """eval_batch (at the uploaded initial guesses) and init_scaling_batch repeat byte for byte, and around them the resident
    batch solves to optimize's bytes"""
    pb = work[2].select(np.arange(256))
    opt = ctx(gpu, precision, work[1], work[0])
    ref = opt.optimize(pb)
    opt.upload(pb)
    ev = [opt.eval_batch() for _ in range(2)]
    sc = [opt.init_scaling_batch() for _ in range(2)]
    for k in ev[0]:
        assert ev[0][k].tobytes() == ev[1][k].tobytes(), k
    assert sc[0][0].tobytes() == sc[1][0].tobytes() and sc[0][1].tobytes() == sc[1][1].tobytes()
    opt.solve_resident()
    opt.sync()
    assert same_bytes(opt.download(), ref)
    # and in the other order on the same lane: the solve leaves nothing the phase calls see
    again = opt.eval_batch(), opt.init_scaling_batch()
    for k in ev[0]:
        assert again[0][k].tobytes() == ev[0][k].tobytes(), k
    assert again[1][0].tobytes() == sc[0][0].tobytes() and again[1][1].tobytes() == sc[0][1].tobytes()
    opt.close()
