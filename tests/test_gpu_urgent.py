"""Urgent work (include/ualm.h: ualm_set_urgent) on both paths: an urgent ticket, check or replan goes ahead of the batches in flight and
changes no result bit of any ticket.  Workload: the 1024-problem hill workload of tests/test_gpu_cancel.py (more than the 528 resident
parity slots), and 4096-problem background batches where the order of work is measured."""
import ctypes as C
import os
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stop_oracle as so  # noqa: E402
from harness import build_driver, ctx, gpu, part, pending, same_bytes, same_problem  # noqa: F401, E402


pytestmark = pytest.mark.gpu

STOPPED = 3
DEPTH = {64: 3, 32: 8, 65: 8}


@pytest.fixture(scope="module")
def work(hill_map, golden):
    from uneven_planner_b200 import configs, problems
    kw = configs.gen_kwargs("hill")
    gold = golden("hill", hill_map)
    return dict(m=hill_map, params=configs.params_for("hill"), pb=problems.generate(hill_map, 1024, seed=0, **kw), gold=gold,
                gold_pb=problems.generate(hill_map, int(gold["B"]), seed=int(gold["seed"]), **kw),
                big=problems.generate(hill_map, 4096, seed=11, **kw), small=problems.generate(hill_map, 16, seed=12, **kw))


@pytest.fixture(scope="module")
def free(gpu, work):
    """(precision, batch name, budget) -> the batch solved alone on a fresh context"""
    cache = {}

    def get(precision, name, budget=0):
        key = (precision, name, budget)
        if key not in cache:
            opt = ctx(gpu, precision, work["params"], work["m"])
            if budget:
                opt.set_budget(budget)
            cache[key] = opt.optimize(work[name])
            opt.close()
        return cache[key]
    return get


def _drain(opt, t, pb, limit_s=600.0):
    """poll until the ticket is complete; returns the seconds it took"""
    out = opt.outputs(pb)
    t0 = time.perf_counter()
    pending = pb.B
    while pending:
        pending = opt.poll(t, out, 1.0)[1]
        assert time.perf_counter() - t0 < limit_s
    return time.perf_counter() - t0


@pytest.mark.parametrize("precision", [64, 32, 65])
def test_urgent_ticket_bits(gpu, work, free, precision):
    opt = ctx(gpu, precision, work["params"], work["m"])
    d = DEPTH[precision]
    t0, t1 = opt.submit(work["pb"], depth=d), opt.submit(work["pb"], depth=d)
    tu = opt.submit(work["gold_pb"], depth=d, urgent=True)
    outs = [opt.wait(tu), opt.wait(t0), opt.wait(t1)]
    opt.close()
    assert same_bytes(outs[0], free(precision, "gold_pb"))
    assert same_bytes(outs[1], free(precision, "pb")) and same_bytes(outs[2], free(precision, "pb"))
    if precision == 64:
        g = work["gold"]
        res, cxy, cyaw = outs[0]
        assert np.array_equal([r.ret_code for r in res], g["ret_code"]) and np.array_equal([r.n_evals for r in res], g["n_evals"])
        assert np.array_equal([r.inner_cost for r in res], g["inner_cost"])
        assert np.array_equal(cxy, g["c_xy"]) and np.array_equal(cyaw, g["c_yaw"])


def _race(opt, work, urgent):
    """two 4096-problem background tickets, then 16 problems (urgent or not): the pending count of background ticket 1 when the third
    ticket is complete, and the third ticket's submit-to-complete time.  (Ticket 1, not 0: submitting ticket 1 behind a full device
    returns only once ticket 0's slots start to free, so ticket 0 is mostly done before the third ticket exists.)"""
    big, small = work["big"], work["small"]
    t0, t1 = opt.submit(big, depth=3), opt.submit(big, depth=3)
    s = time.perf_counter()
    tu = opt.submit(small, depth=3, urgent=urgent)
    _drain(opt, tu, small)
    ms = 1e3 * (time.perf_counter() - s)
    left = pending(opt, t1, big)
    outs = [opt.wait(tu), opt.wait(t0), opt.wait(t1)]
    return left, ms, outs


def test_urgent_ticket_goes_ahead(gpu, work, free):
    opt = ctx(gpu, 64, work["params"], work["m"])
    left_n, ms_n, _ = _race(opt, work, False)
    left_u, ms_u, outs = _race(opt, work, True)
    opt.close()
    print("16 problems behind two 4096-problem tickets: urgent complete after %.1f ms with %d of background ticket 1 pending; "
          "not urgent %.1f ms with %d pending (background ticket 1)" % (ms_u, left_u, ms_n, left_n))
    assert left_u > work["big"].B // 2
    assert same_bytes(outs[0], free(64, "small"))


def test_urgent_ticket_that_grows_its_lane(gpu, work, free):
    """an urgent ticket larger than its lane's previous batch, submitted behind two 4096-problem tickets: the lane's buffers grow (which
    waits for the device) before the hold is raised, so no launch is held while the call waits, and nothing waits for the hold's 2 s
    bound.  Urgent against not urgent, each on a fresh context whose three lanes last held 16 problems"""
    big, pb, small = work["big"], work["pb"], work["small"]

    def run(urgent):
        opt = ctx(gpu, 64, work["params"], work["m"])
        for _ in range(3):
            opt.wait(opt.submit(small, depth=3))
        t0, t1 = opt.submit(big, depth=3), opt.submit(big, depth=3)
        s = time.perf_counter()
        tu = opt.submit(pb, depth=3, urgent=urgent)
        call = time.perf_counter() - s
        _drain(opt, tu, pb)
        done_u = time.perf_counter() - s
        _drain(opt, t1, big)
        done_all = time.perf_counter() - s
        outs = [opt.wait(tu), opt.wait(t0), opt.wait(t1)]
        opt.close()
        return call, done_u, done_all, outs
    n, u = run(False), run(True)
    print("1024 urgent problems into a lane that held 16, behind two 4096-problem tickets: call %.1f ms, complete %.1f ms, everything %.1f ms; "
          "not urgent: call %.1f ms, complete %.1f ms, everything %.1f ms" % tuple(1e3 * x for x in u[:3] + n[:3]))
    assert u[2] < n[2] + 0.5
    assert u[1] - u[0] < 1.0
    assert same_bytes(u[3][0], free(64, "pb")) and same_bytes(u[3][1], n[3][1]) and same_bytes(u[3][2], n[3][2])


def test_urgent_check_and_replan_in_flight(gpu, work, free):
    pb, big = work["gold_pb"], work["big"]
    held = free(64, "gold_pb")
    rows, tf = np.arange(pb.B), np.full(pb.B, 0.5)
    opt = ctx(gpu, 64, work["params"], work["m"])
    chk_idle = opt.check_results(pb, held)
    tr, new_idle = opt.submit_replan(pb, held, rows, tf, depth=3)
    rep_idle = opt.wait(tr)
    t0, t1 = opt.submit(big, depth=3), opt.submit(big, depth=3)
    chk = opt.check_results(pb, held, urgent=True)
    left_c = pending(opt, t1, big)
    tr, new = opt.submit_replan(pb, held, rows, tf, depth=3, urgent=True)
    left_r = pending(opt, t1, big)
    rep = opt.wait(tr)
    opt.cancel(t0, np.arange(big.B))
    opt.cancel(t1, np.arange(big.B))
    opt.wait(t0), opt.wait(t1)
    opt.close()
    print("background ticket 1 pending after the urgent check: %d, after the urgent replan: %d of %d" % (left_c, left_r, big.B))
    assert left_c > big.B // 2 and left_r > big.B // 2
    assert chk.tobytes() == chk_idle.tobytes()
    for a in ("N", "M", "bnd", "total_time", "inner_xy", "inner_yaw"):
        assert np.asarray(getattr(new, a)).tobytes() == np.asarray(getattr(new_idle, a)).tobytes(), a
    assert same_bytes(rep, rep_idle)


def test_interplay_with_cancel_deadline_and_budget(gpu, work, free):
    import pyoracle as po
    pb, small = work["pb"], work["small"]
    ref, ref_small = free(64, "pb"), free(64, "small")
    opt = ctx(gpu, 64, work["params"], work["m"])
    # cancels of a held ticket and of the urgent ticket
    t0 = opt.submit(pb, depth=3)
    tu = opt.submit(small, depth=3, urgent=True)
    cut0 = np.argsort(pb.N, kind="stable")[:40]
    cutu = np.arange(0, small.B, 4)
    opt.cancel(t0, cut0)
    opt.cancel(tu, cutu)
    outu, out0 = opt.wait(tu), opt.wait(t0)
    # a deadline on a ticket while an urgent ticket holds it back
    t1 = opt.submit(pb, depth=3)
    tu2 = opt.submit(small, depth=3, urgent=True)
    out1 = opt.wait(t1, timeout_ms=5.0)
    outu2 = opt.wait(tu2)
    opt.close()
    assert same_bytes(outu2, ref_small)
    stopped = []
    for out, b, r, cut in ((out0, pb, ref, cut0), (outu, small, ref_small, cutu), (out1, pb, ref, np.arange(pb.B))):
        for i in range(b.B):
            if i in cut and out[0][i].ret_code == STOPPED:
                stopped.append((b, out, i))
            else:
                assert same_problem(b, out, r, i), i
    assert any(o is out1 for _, o, _ in stopped)
    prm, om = po.params_from(work["params"]), po.OracleMap(work["m"])
    so.lib()
    rng = np.random.default_rng(3)
    pick = [stopped[k] for k in rng.choice(len(stopped), min(24, len(stopped)), replace=False)]
    for b, out, i in pick:
        r, cxy, cyaw = part(b, out, i)
        assert so.match_stopped(prm, om, b, i, r, cxy, cyaw) is not None, i
    # a budget: the urgent ticket and the held ones, each bit for bit its free solve under the same budget
    budget = 40
    opt = ctx(gpu, 64, work["params"], work["m"])
    opt.set_budget(budget)
    t0 = opt.submit(pb, depth=3)
    tu = opt.submit(small, depth=3, urgent=True)
    outu, out0 = opt.wait(tu), opt.wait(t0)
    opt.close()
    assert same_bytes(outu, free(64, "small", budget)) and same_bytes(out0, free(64, "pb", budget))
    assert any(r.ret_code == STOPPED for r in out0[0])


def test_no_leaked_hold(gpu, work, free):
    from uneven_planner_b200 import _lib, problems
    L = _lib.lib()
    big, small, gold_pb = work["big"], work["small"], work["gold_pb"]
    held = free(64, "gold_pb")
    opt = ctx(gpu, 64, work["params"], work["m"])
    opt.wait(opt.submit(big, depth=1))                          # warm-up
    alone = _drain(opt, opt.submit(big, depth=1), big)
    opt.wait(0)
    assert L.ualm_set_urgent(opt.h, 2) == _lib.UALM_EINVAL and L.ualm_set_urgent(opt.h, -1) == _lib.UALM_EINVAL
    assert L.ualm_set_urgent(None, 1) == _lib.UALM_EINVAL
    t = opt.submit(big, depth=1)
    with pytest.raises(RuntimeError):
        opt.submit(small, depth=1, urgent=True)                 # the next lane is in flight
    opt.cancel(t, np.arange(big.B))
    opt.wait(t)
    # a replan refused after its build: a trajectory resting at its goal has a polyline of zero length
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    one = np.ones(1, np.int32)
    pt, cxy, cyaw, bnd, tf = np.ones(2), np.zeros(12), np.zeros(6), np.zeros(18), np.zeros(1)
    No, Mo, bo, To = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(18), np.zeros(1)
    tk = C.c_int(-1)
    P = lambda a, t=dp: a.ctypes.data_as(t)
    assert L.ualm_set_urgent(opt.h, 1) == 0
    rc = L.ualm_submit_replan(opt.h, 1, P(one, ip), P(one, ip), P(pt), P(cxy), P(cyaw), P(bnd), None, P(tf), 0.01, None, 2, C.byref(tk), P(No, ip),
                              P(Mo, ip), P(bo), P(To), None, None)
    assert L.ualm_set_urgent(opt.h, 0) == 0
    assert rc == _lib.UALM_EINVAL, rc
    # urgent tickets with nothing to solve: B = 0, and only problems over the compiled limits
    empty = gold_pb.select(np.arange(0))
    opt.wait(opt.submit(empty, depth=2, urgent=True))
    over = problems.ProblemBatch(np.array([65], np.int32), np.array([3], np.int32), gold_pb.bnd[:1].copy(), gold_pb.total_time[:1].copy(),
                                 np.zeros(2 * 64), np.zeros(2))
    res, _, _ = opt.wait(opt.submit(over, depth=2, urgent=True))
    assert res[0].ret_code == _lib.UALM_ELIMIT
    # successful urgent work in between
    opt.wait(opt.submit(small, depth=2, urgent=True))
    opt.check_results(gold_pb, held, urgent=True)
    opt.wait(opt.submit_replan(gold_pb, held, np.arange(gold_pb.B), 0.5, depth=2, urgent=True)[0])
    after = _drain(opt, opt.submit(big, depth=1), big)
    out = opt.wait(0)
    opt.close()
    print("4096 problems alone: %.1f ms before the urgent calls, %.1f ms after" % (1e3 * alone, 1e3 * after))
    assert after < 1.5 * alone
    assert out[0][0].ret_code in (0, 1, 2)


@pytest.mark.parametrize("precision", [64, 32])
def test_cpp_set_urgent(gpu, work, tmp_path, precision):
    """setUrgent through include/ualm_traj_opt.hpp around submitBatch / checkTrajectories / submitReplan (checked by the driver)"""
    from uneven_planner_b200 import maps
    exe = build_driver("urgent_driver", tmp_path)
    g0 = maps.stand_in_terrain("hill")
    pb = work["pb"].select(np.arange(0, 1024, 32))
    tf = np.full(pb.B, 0.5)
    case = str(tmp_path / "urgent.bin")
    with open(case, "wb") as f:
        f.write(struct.pack("<5i", *g0.shape, pb.B, 16))
        f.write(g0.cells.tobytes())
        for a in (pb.N, pb.M):
            f.write(np.ascontiguousarray(a, np.int32).tobytes())
        for a in (pb.bnd, pb.total_time, pb.inner_xy, pb.inner_yaw, tf):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, case, str(precision)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
    print(r.stdout.strip())
