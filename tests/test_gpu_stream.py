"""Results of a batch in flight as its problems finish (include/ualm.h: ualm_poll_batch) on both paths: every problem comes back
exactly once, bit for bit what ualm_wait_batch returns for it (and, on the parity path, what the oracle computes), tickets do not
mix, problems over the limits come back at once, and budgets and deadlines keep their meaning.  Workload: BASELINE configs[1]'s
recipe (hill terrain or its stand-in, hill parameters)."""
import ctypes as C
import struct
import subprocess
import time

import numpy as np
import pytest

from harness import build_driver, ctx, gpu, same_bytes, same_problem  # noqa: F401


pytestmark = pytest.mark.gpu

STOPPED = 3
ip = C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def work(hill_map):
    from uneven_planner_b200 import configs, problems
    return hill_map, configs.params_for("hill"), problems.generate(hill_map, 256, seed=0, **configs.gen_kwargs("hill"))


def _poll_all(opt, ticket, pb, wait_ms=1.0, limit_s=600.0):
    """poll until nothing is pending: (filled outputs, [(number returned, pending after) per poll]); every index exactly once"""
    out = opt.outputs(pb)
    seen = np.zeros(pb.B, np.int64)
    polls, pending = [], pb.B
    t0 = time.perf_counter()
    while pending:
        idx, pending = opt.poll(ticket, out, wait_ms)
        assert idx.size == 0 or (idx.min() >= 0 and idx.max() < pb.B)
        np.add.at(seen, idx, 1)
        polls.append((idx.size, pending))
        assert pending == pb.B - int(seen.sum())
        assert time.perf_counter() - t0 < limit_s
    assert (seen == 1).all()
    return out, polls


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_polled_equals_waited(gpu, work, golden, precision):
    m, _, pb = work
    opt = ctx(gpu, precision, work[1], work[0])
    t = opt.submit(pb, depth=1)
    polled, polls = _poll_all(opt, t, pb)
    waited = opt.wait(t)
    assert same_bytes(polled, waited)
    if precision == 64:
        # the batch starts with the committed golden problems (same generator, seed and terrain): bit for bit the oracle's
        gold = golden("hill", m)
        gB = int(gold["B"])
        _, _, ocx, ocy = pb.offsets()
        assert np.array_equal(np.array([r.ret_code for r in polled[0][:gB]]), gold["ret_code"])
        assert np.array_equal(np.array([r.n_evals for r in polled[0][:gB]]), gold["n_evals"])
        assert np.array_equal(np.array([r.inner_cost for r in polled[0][:gB]]), gold["inner_cost"])
        assert np.array_equal(polled[1][:ocx[gB]], gold["c_xy"]) and np.array_equal(polled[2][:ocy[gB]], gold["c_yaw"])
    opt.close()
    print("precision %d: %d polls, %d returned problems" % (precision, len(polls), sum(1 for n, _ in polls if n > 0)))


@pytest.mark.parametrize("precision", [64, 32])
def test_three_tickets_polled_interleaved(gpu, work, precision):
    pb = work[2]
    parts = [pb.select(np.arange(0, 96)), pb.select(np.arange(96, 160)), pb.select(np.arange(160, 256))]
    ref = []
    opt = ctx(gpu, precision, work[1], work[0])
    for p in parts:
        ref.append(opt.optimize(p))
    tickets = [opt.submit(p, depth=3) for p in parts]
    assert len(set(tickets)) == 3
    outs = [opt.outputs(p) for p in parts]
    seen = [np.zeros(p.B, np.int64) for p in parts]
    pending = [p.B for p in parts]
    t0 = time.perf_counter()
    while any(pending):
        for k, t in enumerate(tickets):
            if pending[k]:
                idx, pending[k] = opt.poll(t, outs[k], 1.0)
                assert idx.size == 0 or (idx.min() >= 0 and idx.max() < parts[k].B)    # never another ticket's problem
                np.add.at(seen[k], idx, 1)
        assert time.perf_counter() - t0 < 600.0
    for k, t in enumerate(tickets):
        assert (seen[k] == 1).all()
        assert same_bytes(outs[k], opt.wait(t))
        assert same_bytes(outs[k], ref[k])
    opt.close()


def _spread_batch(m):
    """32 short problems (at most 6 pieces) and four long ones (start and goal at least 11 m apart: about 40 pieces), all resident
    at once"""
    from uneven_planner_b200 import configs, problems
    kw = configs.gen_kwargs("hill")
    short = problems.generate(m, 32, seed=11, n_max=6, min_dist=1.0, **kw)
    long_ = problems.generate(m, 4, seed=12, min_dist=11.0, **kw)
    assert long_.N.min() >= 5 * short.N.max()
    pb = problems.concat([short, long_], [0, 0])
    pb.env = None
    return pb


@pytest.mark.parametrize("precision", [64, 32])
def test_short_problems_come_back_before_the_long_ones(gpu, work, precision):
    pb = _spread_batch(work[0])
    opt = ctx(gpu, precision, work[1], work[0])
    ref = opt.optimize(pb)
    t = opt.submit(pb, depth=1)
    polled, polls = _poll_all(opt, t, pb)
    assert any(n > 0 and pend > 0 for n, pend in polls), polls
    assert same_bytes(polled, opt.wait(t))
    assert same_bytes(polled, ref)
    opt.close()
    print("precision %d: polls (returned, pending) %s" % (precision, [p for p in polls if p[0] > 0]))


def _with_oversized(pb, at):
    """pb with a problem of 65 xy pieces (over UALM_NMAX = 64) inserted at index `at`"""
    from uneven_planner_b200 import problems
    oxy, oyaw, _, _ = pb.offsets()
    N = 65
    start, end = pb.bnd[0][0:2], pb.bnd[0][6:8]
    inner = np.stack([start + (end - start) * (k + 1) / N for k in range(N - 1)]).reshape(-1)
    big = problems.ProblemBatch(np.array([N], np.int32), pb.M[:1].copy(), pb.bnd[:1].copy(), pb.total_time[:1] * 4.0, inner,
                                pb.inner_yaw[oyaw[0]:oyaw[1]].copy())
    head, tail = pb.select(np.arange(at)), pb.select(np.arange(at, pb.B))
    out = problems.concat([head, big, tail], [0, 0, 0])
    out.env = None
    return out


@pytest.mark.parametrize("precision", [64, 32])
def test_problem_over_the_limits_comes_back_first(gpu, work, precision):
    from uneven_planner_b200 import _lib
    base = work[2].select(np.arange(24))
    at = 9
    pb = _with_oversized(base, at)
    opt = ctx(gpu, precision, work[1], work[0])
    ref = opt.optimize(base)
    t = opt.submit(pb, depth=1)
    out = opt.outputs(pb)
    idx, pending = opt.poll(t, out, 0.0)
    assert at in idx and pending == pb.B - idx.size
    _, _, ocx, ocy = pb.offsets()
    assert out[0][at].ret_code == _lib.UALM_ELIMIT and not out[1][ocx[at]:ocx[at + 1]].any() and not out[2][ocy[at]:ocy[at + 1]].any()
    seen = np.zeros(pb.B, np.int64)
    np.add.at(seen, idx, 1)
    t0 = time.perf_counter()
    while pending:
        idx, pending = opt.poll(t, out, 1.0)
        assert at not in idx
        np.add.at(seen, idx, 1)
        assert time.perf_counter() - t0 < 600.0
    assert (seen == 1).all()
    waited = opt.wait(t)
    assert same_bytes(out, waited)
    for i in range(pb.B):                       # the rest of the batch is unaffected
        if i != at:
            j = i if i < at else i - 1
            _, _, bcx, bcy = base.offsets()
            assert bytes(out[0][i]) == bytes(ref[0][j])
            assert out[1][ocx[i]:ocx[i + 1]].tobytes() == ref[1][bcx[j]:bcx[j + 1]].tobytes()
            assert out[2][ocy[i]:ocy[i + 1]].tobytes() == ref[2][bcy[j]:bcy[j + 1]].tobytes()
    opt.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_polls_then_a_deadline(gpu, work, precision):
    pb = work[2]
    opt = ctx(gpu, precision, work[1], work[0])
    free = opt.optimize(pb)
    t = opt.submit(pb, depth=1)
    out = opt.outputs(pb)
    seen = np.zeros(pb.B, np.int64)
    t0 = time.perf_counter()
    while seen.sum() < pb.B // 8:             # poll until an eighth of the batch is back, then stop the rest at a deadline
        idx, _ = opt.poll(t, out, 5.0)
        np.add.at(seen, idx, 1)
        assert time.perf_counter() - t0 < 600.0
    assert (seen <= 1).all()
    polled = np.flatnonzero(seen)
    waited = opt.wait(t, timeout_ms=1.0)
    n_stop = 0
    for i in range(pb.B):
        if i in polled:
            assert same_problem(pb, out, waited, i), i
        if waited[0][i].ret_code == STOPPED:
            n_stop += 1
        else:
            assert same_problem(pb, waited, free, i), i
    # the lane's next batch starts without a stop request and streams again
    t = opt.submit(pb, depth=1)
    again, _ = _poll_all(opt, t, pb)
    assert same_bytes(again, opt.wait(t)) and same_bytes(again, free)
    opt.close()
    print("precision %d: %d problems returned by the polls, %d stopped by the deadline" % (precision, polled.size, n_stop))


@pytest.mark.parametrize("precision", [64, 32])
def test_budget_stopped_problems_stream(gpu, work, precision):
    pb = work[2]
    opt = ctx(gpu, precision, work[1], work[0]).set_budget(50)
    ref = opt.optimize(pb)
    t = opt.submit(pb, depth=1)
    polled, _ = _poll_all(opt, t, pb)
    assert same_bytes(polled, opt.wait(t)) and same_bytes(polled, ref)
    assert any(r.ret_code == STOPPED for r in polled[0])
    opt.close()


def _raw_poll(opt, ticket, wait_ms=0.0, idx=True, n_new=True, n_pending=True):
    a = np.zeros(1024, np.int32)
    n, p = C.c_int(), C.c_int()
    return opt.L.ualm_poll_batch(opt.h, ticket, wait_ms, a.ctypes.data_as(ip) if idx else None, C.byref(n) if n_new else None,
                                 C.byref(p) if n_pending else None, None, None, None)


@pytest.mark.parametrize("precision", [64, 32])
def test_poll_refusals(gpu, work, precision):
    from uneven_planner_b200 import _lib
    EINVAL, ESTATE = _lib.UALM_EINVAL, _lib.UALM_ESTATE
    pb = work[2].select(np.arange(16))
    opt = ctx(gpu, precision, work[1], work[0])
    t = opt.submit(pb, depth=1)
    assert _raw_poll(opt, -1) == EINVAL and _raw_poll(opt, _lib.lib().ualm_max_lanes()) == EINVAL
    assert _raw_poll(opt, 5) == ESTATE                       # never submitted
    assert _raw_poll(opt, t, -1.0) == EINVAL and _raw_poll(opt, t, float("nan")) == EINVAL
    assert _raw_poll(opt, t, idx=False) == EINVAL and _raw_poll(opt, t, n_new=False) == EINVAL and _raw_poll(opt, t, n_pending=False) == EINVAL
    assert _raw_poll(opt, t) == 0
    opt.wait(t)
    assert _raw_poll(opt, t) == ESTATE                       # already waited
    # a batch of the three-step path is not a ticket
    opt.upload(pb)
    opt.solve_resident()
    assert _raw_poll(opt, 0) == ESTATE
    opt.sync()
    opt.close()


def _write_case(path, m, pb):
    oxy, oyaw, _, _ = pb.offsets()
    with open(path, "wb") as f:
        f.write(struct.pack("<4i", *m.shape, pb.B))
        f.write(m.cells.tobytes())
        f.write(np.ascontiguousarray(pb.N, np.int32).tobytes())
        f.write(np.ascontiguousarray(pb.M, np.int32).tobytes())
        f.write(np.ascontiguousarray(pb.bnd, np.float64).tobytes())
        f.write(np.ascontiguousarray(pb.total_time, np.float64).tobytes())
        f.write(np.ascontiguousarray(pb.inner_xy, np.float64).tobytes())
        f.write(np.ascontiguousarray(pb.inner_yaw, np.float64).tobytes())


@pytest.mark.parametrize("precision", [64, 32])
def test_cpp_poll_batch(gpu, work, tmp_path, precision):
    """pollBatch through include/ualm_traj_opt.hpp: the union of the polled results equals waitBatch (checked by the driver)"""
    m, _, pb = work
    exe = build_driver("stream_driver", tmp_path)
    case = str(tmp_path / "case.bin")
    _write_case(case, m, pb.select(np.arange(64)))
    r = subprocess.run([exe, case, str(precision)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
