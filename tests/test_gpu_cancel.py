"""Cancelling problems of a batch in flight (include/ualm.h: ualm_cancel_problems) on both paths.  The parity path is checked bit for
bit: a problem not cancelled is its uncancelled solve, and a cancelled one is either its uncancelled result (it was final first) or
the oracle's solve with a stop predicate that holds from its s-th stop test on (tests/stop_oracle.cpp, tests/stop_oracle.py).
The throughput path keeps every problem not cancelled bit for bit.  Cancels do not reach other tickets or the lane's next batch.
Workload: 1024 problems on the hill terrain or its stand-in with hill parameters (more than the 528 resident parity slots, so the
smallest problems start last)."""
import os
import struct
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stop_oracle as so  # noqa: E402
from harness import build_driver, ctx, gpu, part, same_bytes, same_problem  # noqa: F401, E402


pytestmark = pytest.mark.gpu

STOPPED = 3


@pytest.fixture(scope="module")
def work(hill_map):
    from uneven_planner_b200 import configs, problems
    return hill_map, configs.params_for("hill"), problems.generate(hill_map, 1024, seed=0, **configs.gen_kwargs("hill"))


@pytest.fixture(scope="module")
def free(gpu, work):
    """uncancelled solve of the workload per precision: (res, c_xy, c_yaw)"""
    cache = {}

    def get(precision):
        if precision not in cache:
            opt = ctx(gpu, precision, work[1], work[0])
            cache[precision] = opt.optimize(work[2])
            opt.close()
        return cache[precision]
    return get


class Poller:
    """polls one ticket into its own outputs; every problem must come back exactly once"""

    def __init__(self, opt, ticket, pb):
        self.opt, self.t, self.pb = opt, ticket, pb
        self.out = opt.outputs(pb)
        self.seen = np.zeros(pb.B, np.int64)
        self.pending = pb.B

    def poll(self, wait_ms=2.0):
        idx, self.pending = self.opt.poll(self.t, self.out, wait_ms)
        assert idx.size == 0 or (idx.min() >= 0 and idx.max() < self.pb.B)
        np.add.at(self.seen, idx, 1)
        assert (self.seen <= 1).all() and self.pending == self.pb.B - int(self.seen.sum())
        return idx

    def drain(self, limit_s=600.0):
        t0 = time.perf_counter()
        while self.pending:
            self.poll()
            assert time.perf_counter() - t0 < limit_s
        assert (self.seen == 1).all()
        return self.out


def _run_three_groups(opt, pb, seed):
    """(a) the ~100 smallest problems right after submit, (b) a spread of ~100 not yet returned after polls returned ~300, (c) 20
    problems a poll already returned; then drain.  Returns (polled outputs, waited outputs, a, b, c, (c)'s records before)."""
    rng = np.random.default_rng(seed)
    t = opt.submit(pb, depth=1)
    a = np.argsort(pb.N, kind="stable")[:100]
    opt.cancel(t, a)
    p = Poller(opt, t, pb)
    t0 = time.perf_counter()
    while p.pending and p.seen.sum() < 300:
        p.poll()
        assert time.perf_counter() - t0 < 600.0
    back = np.flatnonzero(p.seen)
    rest = np.setdiff1d(np.flatnonzero(p.seen == 0), a)
    b = np.sort(rng.choice(rest, min(100, rest.size), replace=False))
    c = np.sort(rng.choice(back, min(20, back.size), replace=False))
    before = [bytes(p.out[0][i]) for i in c]
    opt.cancel(t, b)
    opt.cancel(t, c)
    opt.cancel(t, np.concatenate([a[:10], a[:10]]))     # duplicates and repeats are harmless
    polled = p.drain()
    waited = opt.wait(t)
    return polled, waited, a, b, c, before


def test_parity_cancel_matches_oracle(gpu, work, free):
    import pyoracle as po
    m, params, pb = work
    ref = free(64)
    opt = ctx(gpu, 64, work[1], work[0])
    polled, waited, a, b, c, before = _run_three_groups(opt, pb, seed=1)
    opt.close()
    assert same_bytes(polled, waited)
    cancelled = np.union1d(np.union1d(a, b), c)
    for i in np.setdiff1d(np.arange(pb.B), cancelled):
        assert same_problem(pb, polled, ref, i), i
    for k, i in enumerate(c):                     # already final: unchanged
        assert bytes(polled[0][i]) == before[k] and same_problem(pb, polled, ref, i), i
    stopped = [int(i) for i in cancelled if polled[0][i].ret_code == STOPPED]
    for i in cancelled:
        if polled[0][i].ret_code != STOPPED:
            assert same_problem(pb, polled, ref, i), i
    prm, om = po.params_from(params), po.OracleMap(m)
    so.lib()                                      # compiled once, before the threads use it

    def check(i):
        r, cxy, cyaw = part(pb, polled, i)
        return i, so.match_stopped(prm, om, pb, i, r, cxy, cyaw)
    with ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as ex:
        found = list(ex.map(check, stopped))
    assert all(s is not None for _, s in found), [i for i, s in found if s is None]
    iters = np.array([polled[0][i].n_lbfgs_iters for i in stopped])
    assert (iters == 1).any() and (iters > 1).any(), iters
    print("parity: %d cancelled, %d stopped (%d at the first stop test), %d final first" %
          (cancelled.size, len(stopped), int((iters == 1).sum()), cancelled.size - len(stopped)))


@pytest.mark.parametrize("precision", [32, 65])
def test_throughput_cancel(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0])
    polled, waited, a, b, c, before = _run_three_groups(opt, pb, seed=2)
    opt.close()
    assert same_bytes(polled, waited)
    cancelled = np.union1d(np.union1d(a, b), c)
    n_stop = 0
    for i in range(pb.B):
        r = polled[0][i]
        if i in cancelled and r.ret_code == STOPPED:
            assert r.n_lbfgs_iters >= 1, i
            n_stop += 1
        else:
            assert same_problem(pb, polled, ref, i), i
    for k, i in enumerate(c):
        assert bytes(polled[0][i]) == before[k]
    assert n_stop > 0
    print("precision %d: %d cancelled, %d stopped" % (precision, cancelled.size, n_stop))


@pytest.mark.parametrize("precision", [64, 32])
def test_other_ticket_and_next_batch_unaffected(gpu, work, precision):
    pb = work[2]
    A, B2 = pb.select(np.arange(0, 256)), pb.select(np.arange(256, 512))
    opt = ctx(gpu, precision, work[1], work[0])
    refA, refB = opt.optimize(A), opt.optimize(B2)
    ta, tb = opt.submit(A, depth=2), opt.submit(B2, depth=2)
    assert ta != tb
    opt.cancel(ta, np.arange(0, A.B, 2))
    pa, pbp = Poller(opt, ta, A), Poller(opt, tb, B2)
    t0 = time.perf_counter()
    while pa.pending or pbp.pending:
        for p in (pa, pbp):
            if p.pending:
                p.poll(1.0)
        assert time.perf_counter() - t0 < 600.0
    assert same_bytes(pa.out, opt.wait(ta)) and same_bytes(pbp.out, opt.wait(tb))
    assert same_bytes(pbp.out, refB)                           # the other ticket, bit for bit
    for i in range(A.B):
        if i % 2 or pa.out[0][i].ret_code != STOPPED:
            assert same_problem(A, pa.out, refA, i), i
    # the next batch on the cancelled ticket's lane, without cancels: no word carries over
    t = opt.submit(A, depth=2)
    assert t == ta
    again = Poller(opt, t, A).drain()
    assert same_bytes(again, opt.wait(t)) and same_bytes(again, refA)
    opt.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_cancel_everything_right_after_submit(gpu, work, free, precision):
    pb = work[2]
    ref = free(precision)
    opt = ctx(gpu, precision, work[1], work[0])
    t = opt.submit(pb, depth=1)        # warm-up: the free drain time
    t0 = time.perf_counter()
    assert same_bytes(Poller(opt, t, pb).drain(), ref)
    free_s = time.perf_counter() - t0
    opt.wait(t)
    t = opt.submit(pb, depth=1)
    t0 = time.perf_counter()
    opt.cancel(t, np.arange(pb.B))
    out = Poller(opt, t, pb).drain()
    drain_s = time.perf_counter() - t0
    assert same_bytes(out, opt.wait(t))
    rc = np.array([r.ret_code for r in out[0]])
    for i in range(pb.B):
        if rc[i] != STOPPED:
            assert same_problem(pb, out, ref, i), i
    assert (rc == STOPPED).any()
    opt.close()
    print("precision %d: %d of %d stopped; drained in %.1f ms after cancelling all, %.1f ms without cancels" %
          (precision, int((rc == STOPPED).sum()), pb.B, 1e3 * drain_s, 1e3 * free_s))


@pytest.mark.parametrize("precision", [64, 32])
def test_cancel_in_a_mixed_environment_batch(gpu, work, terrain, precision):
    from uneven_planner_b200 import configs, problems
    m0, p0, pb = work
    m1 = terrain("volcano")
    p1 = configs.params_for("volcano")
    one = problems.generate(m1, 300, seed=5, **configs.gen_kwargs("volcano"))
    mixed = problems.concat([pb.select(np.arange(300)), one], [0, 1])
    opt = gpu.BatchALMTrajOpt(precision=precision).init(p0, env=0).set_environment(m0, env=0).init(p1, env=1).set_environment(m1, env=1)
    ref = opt.optimize(mixed)
    t = opt.submit(mixed, depth=1)
    cut = []
    for e in (0, 1):
        ids = np.flatnonzero(mixed.env == e)
        cut.append(ids[np.argsort(mixed.N[ids], kind="stable")[:40]])
    cut = np.concatenate(cut)
    opt.cancel(t, cut)
    out = Poller(opt, t, mixed).drain()
    assert same_bytes(out, opt.wait(t))
    stops = [0, 0]
    for i in range(mixed.B):
        if i in cut and out[0][i].ret_code == STOPPED:
            stops[int(mixed.env[i])] += 1
        else:
            assert same_problem(mixed, out, ref, i), i
    assert stops[0] > 0 and stops[1] > 0, stops
    opt.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_cancel_refusals(gpu, work, precision):
    import ctypes as C
    from uneven_planner_b200 import _lib
    EINVAL, ESTATE = _lib.UALM_EINVAL, _lib.UALM_ESTATE
    pb = work[2].select(np.arange(64))
    opt = ctx(gpu, precision, work[1], work[0])
    ref = opt.optimize(pb)
    L, h = opt.L, opt.h
    ip = C.POINTER(C.c_int32)

    def raw(ticket, idx, n=None, null=False):
        a = np.ascontiguousarray(idx, np.int32)
        return L.ualm_cancel_problems(h, ticket, a.size if n is None else n, None if null else a.ctypes.data_as(ip))
    t = opt.submit(pb, depth=1)
    assert L.ualm_cancel_problems(None, t, 1, np.zeros(1, np.int32).ctypes.data_as(ip)) == EINVAL
    assert raw(-1, [0]) == EINVAL and raw(_lib.lib().ualm_max_lanes(), [0]) == EINVAL
    assert raw(t, [0], n=-1) == EINVAL and raw(t, [0], n=1, null=True) == EINVAL
    assert raw(t, [0, pb.B]) == EINVAL and raw(t, [3, -1]) == EINVAL      # a valid index next to an invalid one: nothing raised
    assert raw(5, [0]) == ESTATE                                          # never submitted
    assert raw(t, [], n=0, null=True) == 0 and raw(t, []) == 0
    out = Poller(opt, t, pb).drain()
    assert same_bytes(out, opt.wait(t)) and same_bytes(out, ref)                    # the refused calls raised nothing
    assert raw(t, [0]) == ESTATE                                          # already waited
    opt.upload(pb)                                                        # a batch of the three-step path is not a ticket
    opt.solve_resident()
    assert raw(0, [0]) == ESTATE
    opt.sync()
    opt.close()


def _write_case(path, m, pb):
    with open(path, "wb") as f:
        f.write(struct.pack("<4i", *m.shape, pb.B))
        f.write(m.cells.tobytes())
        for a, t in ((pb.N, np.int32), (pb.M, np.int32), (pb.bnd, np.float64), (pb.total_time, np.float64), (pb.inner_xy, np.float64),
                     (pb.inner_yaw, np.float64)):
            f.write(np.ascontiguousarray(a, t).tobytes())


@pytest.mark.parametrize("precision", [64, 32])
def test_cpp_cancel_problems(gpu, work, tmp_path, precision):
    """cancelProblems through include/ualm_traj_opt.hpp (checked by the driver)"""
    m, _, pb = work
    exe = build_driver("cancel_driver", tmp_path)
    case = str(tmp_path / "case.bin")
    _write_case(case, m, pb.select(np.arange(128)))
    r = subprocess.run([exe, case, str(precision)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
    print(r.stdout.strip())
